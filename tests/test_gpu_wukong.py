"""WuKong on the H100: the layer (FM row kernel, the FMB's MLP, the field-axis GEMM, the combine row kernel and back)
against the reference's goldens and against the float64 oracle over the row kernels' launch-plan branches in every
matmul mode, stacked so that the (B D, fp) layout and its one gradient buffer are crossed; the operand copies both row
kernels write, bit for bit; eval against dropout 0; zoo.WuKong with the fused optimizer along the reference's
training trajectories; a CUDA-graph-captured training step against the eager one; and two virtual ranks with
row-sharded tables against the unsharded model."""
import sys

import pytest
import torch

from conftest import Golden, ROOT, close, rel_err

sys.path.insert(0, ROOT)
import wukong_oracle as WO  # noqa: E402

pytestmark = pytest.mark.gpu

RTOL = 1e-5
# single-pass modes: Frobenius bars on the output and on the gradients (the row kernels are fp32 in every mode; the
# field-axis and MLP GEMMs round their operands)
FRO = {"tf32": (1e-2, 6e-2), "bf16": (3e-2, 1.5e-1)}
# ... and on a whole model's y_pred and losses and its gradients: a stack of layers (and fc's BatchNorm over a 32-row
# batch) compounds the layer's rounding
FRO_MODEL = {"tf32": (2e-2, 4e-1), "bf16": (5e-2, 4e-1)}


@pytest.fixture(scope="module", autouse=True)
def _built():
    import __graft_entry__
    __graft_entry__.build()
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"


@pytest.fixture
def mode_of():
    from fuxictr_b200 import functional as F2
    yield F2.set_matmul_precision
    F2.set_matmul_precision("fp32")
    F2.set_x3_inline(True)


def fro(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def noise_only(grads, key):
    """A parameter whose exact gradient is zero (residual_proj.bias before the output LayerNorm(D); the last
    LayerNorm's bias before fc's BatchNorm1d): below 1e-6 of the largest gradient, rounding noise in every
    implementation, which Adam turns into steps of lr.  Trajectories compare the other parameters."""
    scale = max(float(v.abs().max()) for v in grads.values())
    return key not in grads or float(grads[key].abs().max()) <= 1e-6 * scale


# ------------------------------------------------------------------ the reference's goldens
@pytest.mark.parametrize("mode", ["fp32", "tf32x3", "tf32", "bf16"])
@pytest.mark.parametrize("c", ["proj", "identity", "noln"])
def test_layer_matches_reference_golden(c, mode, mode_of):
    from fuxictr_b200 import layers
    g = Golden("next_WuKongLayer")
    _, nf, lcb, fmb, D, k, units, ln = [q for q in g.meta["cases"] if q[0] == c][0]
    layer = layers.WuKongLayer(nf, lcb, fmb, D, k, units, "relu", 0.0, ln)
    layer.load_state_dict(g["w_" + c])
    layer = layer.cuda()
    mode_of(mode)
    x = g["in"]["x_" + c].cuda().requires_grad_(True)
    out = layer(x)
    out.backward(g["in"]["gout_" + c].cuda())
    named = dict(layer.named_parameters())
    want = g["g_" + c]
    if mode in ("fp32", "tf32x3"):
        assert close(out, g["out"]["y_" + c], RTOL), rel_err(out, g["out"]["y_" + c])
        assert close(x.grad, g["gin"]["x_" + c], RTOL, atol=RTOL * float(g["gin"]["x_" + c].abs().max()))
        scale = max(float(v.abs().max()) for v in want.values())
        for key, ref in want.items():
            assert close(named[key].grad, ref, RTOL, atol=RTOL * scale), (key, rel_err(named[key].grad, ref))
        return
    tol_y, tol = FRO[mode]
    assert fro(out, g["out"]["y_" + c]) <= tol_y
    assert fro(x.grad, g["gin"]["x_" + c]) <= tol
    for key, ref in want.items():
        assert noise_only(want, key) or fro(named[key].grad, ref) <= tol, key


# ------------------------------------------------------------------ float64 oracle over the launch-plan branches
def make_stack(nf, lcb, fmb, D, k, units, ln, nlayers, seed):
    from fuxictr_b200 import layers
    torch.manual_seed(seed)
    net = [layers.WuKongLayer(nf if i == 0 else lcb + fmb, lcb, fmb, D, k, units, "relu", 0.0, ln)
           for i in range(nlayers)]
    with torch.no_grad():
        for m in net:
            for mod in m.modules():
                if isinstance(mod, torch.nn.LayerNorm):     # away from the initial 1 and 0
                    mod.weight.uniform_(0.5, 1.5)
                    mod.bias.uniform_(-0.3, 0.3)
            m.fmb.proj_Y.mul_(0.3)
    return [m.cuda() for m in net]


# (B, F, lcb, fmb, D, k, layers, LayerNorm): WuKong_default's layer 0 and 1 (F 39 -> 80, D 64, k 8: the pitch-40 X'_0,
# tensor-core GEMMs where the mode has them); the widest FM (F 128, k 8; F 32, k 32) and D 128; F 1, 2, 5 (projection,
# scalar staging of X at D 3, SIMT GEMMs); F 40 and 80 identity stacks; D 1 (without LayerNorm, which would make the
# layer a constant) and 4; no LayerNorm; B 0, 1, odd, 4096
CASES = [
    (257, 39, 40, 40, 64, 8, 2, True), (4096, 39, 40, 40, 64, 8, 1, True), (33, 128, 64, 64, 16, 8, 2, True),
    (17, 32, 48, 80, 128, 32, 1, True), (5, 1, 1, 1, 3, 1, 2, True), (9, 2, 3, 1, 4, 3, 2, False),
    (31, 5, 8, 8, 16, 8, 3, True), (63, 40, 20, 20, 16, 3, 2, True), (3, 80, 40, 40, 1, 8, 2, False),
    (1, 39, 40, 40, 64, 8, 2, False), (0, 39, 40, 40, 64, 8, 2, True),
]


@pytest.mark.parametrize("mode", ["fp32", "tf32x3", "tf32", "bf16"])
@pytest.mark.parametrize("case", CASES, ids=lambda c: "B%d_F%d_l%d_f%d_D%d_k%d_L%d_ln%d" % c)
def test_stack_matches_float64_oracle(mode, case, mode_of):
    from fuxictr_b200 import layers
    B, nf, lcb, fmb, D, k, nl, ln = case
    units = [24]
    net = make_stack(nf, lcb, fmb, D, k, units, ln, nl, seed=B + nf)
    mode_of(mode)
    x = clear_of_relu_kinks(net, B, nf, D, nl, units, ln).cuda().requires_grad_(True)
    gen = torch.Generator().manual_seed(5)
    out = layers.wukong_stack(net, x)
    gout = torch.randn(out.shape, generator=gen).cuda()
    out.backward(gout)
    st = {}
    for i, m in enumerate(net):
        for key, v in m.state_dict().items():
            st["%d.%s" % (i, key)] = v.detach().double().cpu().requires_grad_(True)
    xr = x.detach().double().cpu().requires_grad_(True)
    y = xr
    for i in range(nl):
        y = WO.wukong_layer(y, st, "%d." % i, len(units), ln)
    y = y.flatten(start_dim=1)
    (y * gout.double().cpu()).sum().backward()
    if B == 0:
        assert out.shape == (0, (lcb + fmb) * D) and x.grad.shape == x.shape
        return
    got = {"%d.%s" % (i, key): p.grad for i, m in enumerate(net) for key, p in m.named_parameters()}
    want = {key: v.grad for key, v in st.items()}
    # Relative Frobenius errors.  The bar in fp32 and 3xTF32 is the larger of a fixed one and four times the error of
    # the reference's ops in fp32 eager on the same inputs (the stacked FM LayerNorms amplify rounding).  The
    # single-pass modes get the layer's bars per stacked layer.
    e32 = eager_fp32_errors(net, x, gout, nl, units, ln, y.detach(), xr.grad, want)
    if mode in ("fp32", "tf32x3"):
        base = 1e-6 if mode == "fp32" else 3e-6
        assert fro(out, y) <= max(base, 4 * e32["out"]), (fro(out, y), e32["out"])
        assert fro(x.grad, xr.grad) <= max(base, 4 * e32["x"]), (fro(x.grad, xr.grad), e32["x"])
        for key, ref in want.items():
            assert noise_only(want, key) or fro(got[key], ref) <= max(10 * base, 4 * e32[key]), \
                (key, fro(got[key], ref), e32[key])
        return
    tol_y, tol = FRO[mode]
    assert fro(out, y) <= tol_y * nl
    assert fro(x.grad, xr.grad) <= tol * nl
    for key, ref in want.items():
        assert noise_only(want, key) or fro(got[key], ref) <= tol * nl, (key, fro(got[key], ref))


def clear_of_relu_kinks(net, B, nf, D, nl, units, ln, margin=1e-5):
    """B samples (B, F, D) on which no ReLU of any layer's FMB MLP has a float64 pre-activation within `margin` of
    zero.  A pre-activation within rounding of zero flips that ReLU, and with it its sample's gradient, in any
    arithmetic but float64's; such samples say nothing about the kernels."""
    st = {"%d.%s" % (i, key): v.detach().double().cpu() for i, m in enumerate(net) for key, v in m.state_dict().items()}
    gen = torch.Generator().manual_seed(5)
    keep = [torch.zeros(0, nf, D)]
    while sum(len(k) for k in keep) < B:
        x = torch.randn(B + B // 4 + 8, nf, D, generator=gen) * 0.7
        y, margins = x.double(), []
        for i in range(nl):
            y = WO.wukong_layer(y, st, "%d." % i, len(units), ln, margins=margins)
        ok = torch.stack(margins).amin(dim=0) > margin
        keep.append(x[ok])
    return torch.cat(keep)[:B].contiguous()


def eager_fp32_errors(net, x, gout, nl, units, ln, y64, gx64, grads64):
    """Relative Frobenius errors against float64 of the reference's ops (the float64 oracle's code) run in fp32 on the
    GPU, TF32 off: the output, the input gradient and each parameter gradient."""
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        st = {"%d.%s" % (i, key): v.detach().float().clone().requires_grad_(True)
              for i, m in enumerate(net) for key, v in m.state_dict().items()}
        xf = x.detach().float().clone().requires_grad_(True)
        y = xf
        for i in range(nl):
            y = WO.wukong_layer(y, st, "%d." % i, len(units), ln)
        y = y.flatten(start_dim=1)
        (y * gout).sum().backward()
    finally:
        torch.backends.cuda.matmul.allow_tf32 = prev
    errs = {"out": fro(y, y64), "x": fro(xf.grad, gx64)}
    for key, ref in grads64.items():
        errs[key] = fro(st[key].grad, ref)
    return errs


@pytest.mark.parametrize("mode", ["bf16", "tf32x3"])
def test_operand_copies_are_bit_exact(mode, mode_of):
    """The copies the row kernels hand on: the FMB MLP's input (FM kernel) and X'_1 (the combine kernel), against the
    copies b2_to_bf16 / b2_split_tf32 make of the fp32 tensors (3xTF32 in the form with small parts in HBM)."""
    from fuxictr_b200 import functional as F2
    mode_of(mode)
    F2.set_x3_inline(False)
    net = make_stack(39, 40, 40, 64, 8, [64], True, 2, seed=1)
    seen = []
    hook = net[0].fmb.mlp.register_forward_hook(lambda m, i, o: seen.append(i[0]))
    x = (torch.randn(300, 39, 64) * 0.5).cuda()
    xp1 = net[0].run(x, last=False, want_aux=True)
    hook.remove()
    for t in (seen[0], xp1):
        hint = t._b2_aux
        ref = F2.split_tf32(t.contiguous()) if mode == "tf32x3" else t.to(torch.bfloat16)
        assert hint[0] == mode and torch.equal(hint[1].float(), ref.float()), tuple(t.shape)


def test_eval_mode_is_bit_equal_to_dropout_zero():
    from fuxictr_b200 import layers
    torch.manual_seed(9)
    a = layers.WuKongLayer(39, 40, 40, 64, 8, [64, 32], "relu", 0.4, True).cuda().eval()
    torch.manual_seed(9)
    b = layers.WuKongLayer(39, 40, 40, 64, 8, [64, 32], "relu", 0.0, True).cuda()
    x = (torch.randn(65, 39, 64) * 0.5).cuda()
    assert torch.equal(a(x), b(x))


# ------------------------------------------------------------------ zoo.WuKong
def build_golden_model(g):
    from fuxictr_b200 import zoo
    from fuxictr_b200.schema import FeatureMap
    fm = FeatureMap.from_specs(g.meta["specs"], labels=g.meta["labels"], embedding_dim=g.meta["kwargs"]["embedding_dim"])
    model = zoo.WuKong(fm, gpu=-1, **g.meta["kwargs"])
    model.load_state_dict(g["w"])
    model.device = torch.device("cuda:0")
    model.model_to_device()
    model.compile("adam", "binary_crossentropy", 1e-3)
    model.train()
    model.use_fused_optimizer()
    return fm, model


@pytest.mark.parametrize("mode", ["fp32", "tf32x3", "tf32", "bf16"])
@pytest.mark.parametrize("name", ["bn", "nobn", "noln"])
def test_model_with_fused_adam_matches_reference_trajectory(name, mode, mode_of):
    """y_pred, loss and every gradient on batch 0, then three fused_train_steps (fused logit + BCE, arena clip + Adam)
    against the reference's train_step()s: losses, gradients and the state after three steps to 1e-5 in fp32 and
    3xTF32; Frobenius bars on y_pred, the losses and the gradients in TF32 and bf16."""
    mode_of(mode)
    g = Golden("model_WuKong_" + name)
    fm, model = build_golden_model(g)
    B = g.meta["batch"]
    mat = g["in"]["matrix"].cuda()
    batches = [fm.batch_dict(mat[i * B:(i + 1) * B]) for i in range(3)]
    exact = mode in ("fp32", "tf32x3")
    tol_y, tol = FRO_MODEL.get(mode, (RTOL, RTOL))
    ret = model.forward(batches[0])
    assert close(ret["y_pred"], g["out"]["y_pred"], RTOL) if exact else fro(ret["y_pred"], g["out"]["y_pred"]) <= tol_y
    loss = model.compute_loss(ret, model.get_labels(batches[0]))
    model._fused_optimizer.zero_grad()
    loss.backward()
    named = dict(model.named_parameters())
    # With fc's BatchNorm1d (the "bn" case) the single-pass modes' embedding gradients are 0.57 (TF32) and 0.59
    # (bf16) off the reference's in Frobenius norm on an H100; the BatchNorm backward over 32 rows subtracts column
    # means of nearly the same size.  There only y_pred and the losses are held to the bars.
    check_grads = exact or not g.meta["kwargs"]["mlp_batch_norm"]
    for key, ref in g["g"].items():
        if noise_only(g["g"], key) or not check_grads:
            continue
        if exact:
            assert close(named[key].grad, ref, RTOL, atol=RTOL * float(ref.abs().max()) + 1e-9), \
                (key, rel_err(named[key].grad, ref))
        else:
            assert fro(named[key].grad, ref) <= tol, key
    model._arena.zero_grads()
    losses = [float(model.fused_train_step(b)) for b in batches]
    want = g["out"]["step_losses"]
    assert close(torch.tensor(losses), want, RTOL) if exact else fro(torch.tensor(losses), want) <= tol_y
    if not exact:       # Adam's steps are sign-like where a gradient is small: the state is compared in 1e-5 modes
        return
    sd = model.state_dict()
    for key, ref in g["w3"].items():
        if noise_only(g["g"], key):
            continue
        assert close(sd[key], ref, 2e-5), (key, rel_err(sd[key], ref))


def _fm_and_batches(n, B, seed, dim):
    import test_gpu_sharded_models as S
    from fuxictr_b200.schema import FeatureMap
    fm = FeatureMap.from_specs(S._CAT, embedding_dim=dim)
    gen = torch.Generator().manual_seed(seed)
    mats = []
    for _ in range(n):
        ids = torch.cat([torch.randint(0, s["vocab_size"], (B, 1), generator=gen) for _, s in S._CAT], 1)
        mats.append(torch.cat([ids.double(), (torch.rand(B, 1, generator=gen) < 0.4).double()], 1).cuda())
    return fm, mats


def make_model(fm, kw, seed=123, **extra):
    from fuxictr_b200 import zoo
    torch.manual_seed(seed)
    m = zoo.WuKong(fm, gpu=0, **dict(kw, **extra))
    with torch.no_grad():
        for mod in m.modules():
            if isinstance(mod, torch.nn.Embedding):
                mod.weight[1:].normal_(0, 0.3)
    return m


# WuKong_test's and WuKong_default's hyperparameters (at a smaller embedding and batch for the test's sake)
CONFIGS = {
    "test": dict(embedding_dim=64, num_wukong_layers=3, lcb_features=8, fmb_features=8, fmb_mlp_units=[32, 32],
                 fmp_rank_k=8, mlp_hidden_units=[32, 32], mlp_batch_norm=True),
    "default": dict(embedding_dim=64, num_wukong_layers=3, lcb_features=40, fmb_features=40,
                    fmb_mlp_units=[512, 256], fmp_rank_k=8, mlp_hidden_units=[512, 256], mlp_batch_norm=False),
}


@pytest.mark.parametrize("mode", ["fp32", "tf32x3", "tf32", "bf16"])
@pytest.mark.parametrize("name", sorted(CONFIGS))
def test_configs_train(name, mode, mode_of):
    """Ten fused_train_steps on one batch at the YAML configurations' hyperparameters: finite and falling losses."""
    mode_of(mode)
    kw = CONFIGS[name]
    fm, mats = _fm_and_batches(1, 512, seed=3, dim=kw["embedding_dim"])
    model = make_model(fm, kw)
    model.train()
    model.use_fused_optimizer()
    losses = [float(model.fused_train_step(fm.batch_dict(mats[0]))) for _ in range(10)]
    assert all(l == l for l in losses) and losses[-1] < losses[0], losses


# ------------------------------------------------------------------ CUDA graph capture
@pytest.mark.parametrize("drop", [0.0, 0.2])
@pytest.mark.parametrize("mode", ["tf32x3", "bf16"])
def test_graph_captured_step_matches_eager(drop, mode, mode_of):
    """Five eager fused_train_steps against three warm-up steps and two replays of the captured step.  With dropout
    the replays draw the masks the eager steps drew (the device RNG state advances inside the graph)."""
    from fuxictr_b200.pipeline import TrainPipeline
    from fuxictr_b200 import functional as F2
    mode_of(mode)
    kw = dict(embedding_dim=16, num_wukong_layers=3, lcb_features=8, fmb_features=8, fmb_mlp_units=[32],
              fmp_rank_k=4, mlp_hidden_units=[32, 16], mlp_batch_norm=False)
    fm, mats = _fm_and_batches(1, 512, seed=4, dim=kw["embedding_dim"])
    mat = mats[0]
    eager = make_model(fm, kw, net_dropout=drop)
    graphed = make_model(fm, kw, net_dropout=drop)
    for m in (eager, graphed):
        m.train()
        m.use_fused_optimizer()
    torch.manual_seed(11)
    F2._DROPOUT.clear()
    F2.dropout_state(mat.device)
    ref = [float(eager.fused_train_step(fm.batch_dict(mat))) for _ in range(5)]
    torch.manual_seed(11)
    F2._DROPOUT.clear()
    F2.dropout_state(mat.device)
    pipe = TrainPipeline(graphed, mat.shape[0], mat.shape[1], graph=False)
    pipe.prime(mat)
    pipe.capture(warmup=3)
    got = [float(pipe.step_device(mat)) for _ in range(2)]
    torch.cuda.synchronize()
    # the row kernels sum dY, dgamma, dbeta and b_res's gradient with float atomics, so eager steps and replays agree
    # to rounding, not bit for bit; residual_proj.bias (exact gradient zero before the LayerNorm) is left out
    # (in bf16 a last-bit difference can move an operand's bf16 rounding: a looser bar there)
    tol = 5e-5 if mode == "tf32x3" else 2e-3
    for a, b in zip(got, ref[3:]):
        assert abs(a - b) <= tol * abs(b), (got, ref)
    if drop:
        assert ref[3] != ref[4]
    sd, want = graphed.state_dict(), eager.state_dict()
    for key, v in want.items():
        if key.endswith("residual_proj.bias"):
            continue
        if mode == "tf32x3":
            assert close(sd[key], v, 1e-4), (key, rel_err(sd[key], v))
        else:
            assert fro(sd[key], v) <= 2e-2, (key, fro(sd[key], v))


# ------------------------------------------------------------------ row-sharded tables, two virtual ranks
def test_two_sharded_ranks_train_like_the_unsharded_model():
    """test_gpu_sharded_models.py's lock-step harness: two virtual ranks on one GPU, each with half of every table's
    rows, three fused_train_steps against the unsharded model with torch's clip + Adam on the global batches."""
    import test_gpu_sharded_models as S
    from fuxictr_b200.schema import FeatureMap
    world = 2
    fm = FeatureMap.from_specs(S._CAT, embedding_dim=S.D)
    kw = dict(embedding_dim=S.D, num_wukong_layers=2, lcb_features=4, fmb_features=4, fmb_mlp_units=[16],
              fmp_rank_k=4, mlp_hidden_units=[16], mlp_batch_norm=False, layer_norm=False)    # every gradient nonzero

    def make():
        return make_model(fm, kw)
    ref = make()
    ref.fm_ = fm
    models = S._ranks(make, world, fm)
    gen = torch.Generator().manual_seed(21)
    batches = []
    for _ in range(3):
        ids = torch.cat([torch.randint(0, s["vocab_size"], (S.B_L * world, 1), generator=gen) for _, s in S._CAT], 1)
        batches.append(torch.cat([ids.double(), (torch.rand(S.B_L * world, 1, generator=gen) < 0.4).double()],
                                 1).cuda())
    losses = []
    for mat in batches:
        mats = [mat[r * S.B_L:(r + 1) * S.B_L].contiguous() for r in range(world)]
        losses.append(sum(S._lockstep_train_step(models, mats, fm)) / world)
    ref_losses = S._reference_steps(ref, batches, world, False)
    for a, b in zip(losses, ref_losses):
        assert abs(a - b) <= 1e-5 * abs(b), (losses, ref_losses)
    S._check_states(models, ref, world)

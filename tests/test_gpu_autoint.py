"""AutoInt on the H100: the self-attention layer (pack, GEMM, row kernel and back) against the float64 oracle over the
row kernels' launch-plan branches in every matmul mode; the operand copy the forward hands on, bit for bit; the
attention dropout masks against a host restatement of the Philox counter; zoo.AutoInt with the fused optimizer along
the float64 oracle's training trajectory; a CUDA-graph-captured training step against the eager one; and two virtual
ranks with row-sharded tables against the unsharded model."""
import sys
from collections import OrderedDict

import pytest
import torch

from conftest import Golden, ROOT, close, rel_err

sys.path.insert(0, ROOT)
import autoint_oracle as AO  # noqa: E402
from oracle import fuxictr_oracle as O  # noqa: E402

pytestmark = pytest.mark.gpu

RTOL = 1e-5
# single-pass modes: Frobenius bars on the output and on the gradients (the row kernel is fp32 in every mode; only
# the projection GEMMs round their operands)
FRO = {"tf32": (1e-2, 6e-2), "bf16": (3e-2, 1.5e-1)}


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


def make_layer(din, A, H, use_residual, use_scale, layer_norm, seed, dropout=0.0):
    from fuxictr_b200 import layers
    torch.manual_seed(seed)
    layer = layers.MultiHeadSelfAttention(din, A, H, dropout_rate=dropout, use_residual=use_residual,
                                          use_scale=use_scale, layer_norm=layer_norm)
    if layer_norm:      # away from the initial 1 and 0, so that a dropped gamma or beta shows
        with torch.no_grad():
            layer.layer_norm.weight.uniform_(0.5, 1.5)
            layer.layer_norm.bias.uniform_(-0.3, 0.3)
    return layer.cuda()


# ------------------------------------------------------------------ the reference's goldens
@pytest.mark.parametrize("mode", ["fp32", "tf32x3", "tf32", "bf16"])
@pytest.mark.parametrize("c", ["wres", "h3_scale", "ln"])
def test_layer_matches_reference_golden(c, mode, mode_of):
    from fuxictr_b200 import layers
    g = Golden("next_MultiHeadSelfAttention")
    _, din, A, H, res, scale, ln = [k for k in g.meta["cases"] if k[0] == c][0]
    layer = layers.MultiHeadSelfAttention(din, A, H, use_residual=res, use_scale=scale, layer_norm=ln)
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
        scale_ = max(float(v.abs().max()) for v in want.values())
        for k, ref in want.items():
            assert close(named[k].grad, ref, RTOL, atol=RTOL * scale_), (k, rel_err(named[k].grad, ref))
        return
    tol_y, tol = FRO[mode]
    assert fro(out, g["out"]["y_" + c]) <= tol_y
    assert fro(x.grad, g["gin"]["x_" + c]) <= tol
    for k, ref in want.items():
        assert fro(named[k].grad, ref) <= tol, k


def build_golden_model(g):
    from fuxictr_b200 import zoo
    from fuxictr_b200.schema import FeatureMap
    fm = FeatureMap.from_specs(g.meta["specs"], labels=g.meta["labels"], embedding_dim=g.meta["kwargs"]["embedding_dim"])
    model = zoo.AutoInt(fm, gpu=-1, **g.meta["kwargs"])
    model.load_state_dict(g["w"])
    model.device = torch.device("cuda:0")
    model.model_to_device()
    model.compile("adam", "binary_crossentropy", 1e-3)
    model.train()
    model.use_fused_optimizer()
    return fm, model


@pytest.mark.parametrize("mode", ["fp32", "tf32x3"])
@pytest.mark.parametrize("name", ["test", "wide", "nodnn"])
def test_model_with_fused_adam_matches_reference_trajectory(name, mode, mode_of):
    """y_pred, loss and every gradient on batch 0, then three fused_train_steps (fused logit + BCE, arena clip + Adam)
    against the reference's train_step()s."""
    mode_of(mode)
    g = Golden("model_AutoInt_" + name)
    fm, model = build_golden_model(g)
    B = g.meta["batch"]
    mat = g["in"]["matrix"].cuda()
    batches = [fm.batch_dict(mat[i * B:(i + 1) * B]) for i in range(3)]
    ret = model.forward(batches[0])
    assert close(ret["y_pred"], g["out"]["y_pred"], RTOL)
    loss = model.compute_loss(ret, model.get_labels(batches[0]))
    assert close(loss, g["out"]["loss"], RTOL)
    model._fused_optimizer.zero_grad()
    loss.backward()
    named = dict(model.named_parameters())
    for k, ref in g["g"].items():
        assert close(named[k].grad, ref, RTOL, atol=RTOL * float(ref.abs().max()) + 1e-9), \
            (k, rel_err(named[k].grad, ref))
    model._arena.zero_grads()
    losses = []
    for i in range(3):
        losses.append(float(model.fused_train_step(batches[i])))
        if i == 0:
            sd = model.state_dict()
            for k, ref in g["w1"].items():
                assert close(sd[k], ref, RTOL), (k, rel_err(sd[k], ref))
    assert close(torch.tensor(losses), g["out"]["step_losses"], RTOL)
    sd = model.state_dict()
    for k, ref in g["w3"].items():
        assert close(sd[k], ref, 2e-5), (k, rel_err(sd[k], ref))


# (B, F, d_in, A, H, use_residual, use_scale, layer_norm): AutoInt_default's layer (F 39, A 40, H 2: d_h 20, float4
# staging, tensor-core GEMM where the mode has one); W_res at d_in 16 and at AutoInt_test's d_in 4 (SIMT GEMM); the
# widest tile (F 64, A 64) at d_h 32 and at d_h 1; the scalar staging path (A 10, d_h 5; A 12, H 3); F 1 and F 2;
# no residual; B 0, 1, odd B and B over many CTAs per SM
CASES = [
    (37, 39, 40, 40, 2, True, False, False),
    (37, 39, 16, 40, 2, True, True, True),
    (33, 39, 4, 8, 2, True, False, False),
    (5, 64, 64, 64, 2, True, True, True),
    (7, 64, 64, 64, 64, True, False, True),
    (33, 2, 10, 10, 2, True, True, True),
    (3, 5, 12, 12, 3, True, True, False),
    (1, 1, 8, 20, 4, True, True, False),
    (1, 2, 20, 20, 1, True, False, True),
    (33, 39, 40, 40, 2, False, True, False),
    (2000, 39, 40, 40, 2, True, True, True),
    (0, 39, 40, 40, 2, True, False, True),
    # the backward's shared memory just under 48 KiB, where its static part makes the opt-in necessary
    (9, 47, 40, 40, 2, True, False, True),
    (9, 43, 48, 48, 4, True, True, False),
    (9, 62, 17, 17, 1, True, False, True),
]


@pytest.mark.parametrize("mode", ["fp32", "tf32x3", "tf32", "bf16"])
@pytest.mark.parametrize("case", CASES, ids=lambda c: "B%d_F%d_din%d_A%d_H%d_r%d_s%d_ln%d" % c)
def test_layer_matches_float64_oracle(mode, case, mode_of):
    B, F, din, A, H, use_res, use_scale, ln = case
    layer = make_layer(din, A, H, use_res, use_scale, ln, seed=B + F + A)
    state = {k: v.detach().double().requires_grad_(True) for k, v in layer.state_dict().items()}
    gen = torch.Generator().manual_seed(F * 7 + B)
    x = torch.randn(B, F, din, generator=gen) * 0.5
    gout = torch.randn(B, F, A, generator=gen)
    xr = x.double().cuda().requires_grad_(True)
    yr = AO.self_attention(xr, state, "", H, use_res, use_scale, ln)
    yr.backward(gout.double().cuda())
    mode_of(mode)
    xg = x.cuda().requires_grad_(True)
    yg = layer(xg)
    assert yg.shape == (B, F, A)
    yg.backward(gout.cuda())
    named = dict(layer.named_parameters())
    if B == 0:
        assert xg.grad.shape == xg.shape
        assert all(float(p.grad.abs().sum()) == 0 for p in named.values())
        return
    if mode in ("fp32", "tf32x3"):
        assert close(yg, yr, RTOL), rel_err(yg, yr)
        assert close(xg.grad, xr.grad, RTOL, atol=RTOL * float(xr.grad.abs().max())), rel_err(xg.grad, xr.grad)
        for k, ref in state.items():
            assert close(named[k].grad, ref.grad, RTOL, atol=RTOL * float(ref.grad.abs().max())), \
                (k, rel_err(named[k].grad, ref.grad))
        return
    tol_y, tol = FRO[mode]
    assert fro(yg, yr) <= tol_y
    assert fro(xg.grad, xr.grad) <= tol
    for k, ref in state.items():
        assert fro(named[k].grad, ref.grad) <= tol, k


@pytest.mark.parametrize("mode", ["bf16", "tf32x3"])
def test_operand_copy_is_bit_exact(mode, mode_of):
    """The next layer's GEMM operand that the row kernel writes beside out: its bf16 rounding, or (3xTF32 with the
    small parts in HBM) its small part, equal to what the standalone conversion makes of out."""
    from fuxictr_b200 import functional as F2
    mode_of(mode)
    F2.set_x3_inline(False)
    layer = make_layer(40, 40, 2, True, True, True, seed=5)
    x = (torch.randn(129, 39, 40) * 0.5).cuda()
    out = F2.self_attention_layer(x, layer.W_q.weight, layer.W_k.weight, layer.W_v.weight, num_heads=2,
                                  use_scale=True, gamma=layer.layer_norm.weight, beta=layer.layer_norm.bias,
                                  want_aux=True)
    hint = out._b2_aux
    assert hint[0] == mode
    flat = out.view(-1, 40)
    want = flat.to(torch.bfloat16) if mode == "bf16" else F2.split_tf32(flat)
    assert torch.equal(hint[1], want)


# ------------------------------------------------------------------ attention dropout
def keep_weights(snap, layer, B, H, F, p):
    """The keep mask of the (B, H, F, F) attention weights: element ((b H + h) F + i) F + j of the dropout layer at
    counter offset snapshot offset + layer."""
    from test_mlp_dropout_host import keep_mask
    seed, off = [int(v) for v in snap.cpu()]
    return torch.from_numpy(keep_mask(seed, off + layer, B * H * F, F, p)).view(B, H, F, F)


@pytest.mark.parametrize("case", [(37, 39, 40, 40, 2, True, True, True), (9, 7, 10, 10, 5, True, False, False),
                                  (5, 64, 16, 64, 4, True, True, True)])
def test_dropout_masks_match_the_host_philox(case, mode_of):
    from fuxictr_b200 import functional as F2
    B, F, din, A, H, use_res, use_scale, ln = case
    p = 0.3
    layer = make_layer(din, A, H, use_res, use_scale, ln, seed=3, dropout=p).train()
    state = {k: v.detach().double().requires_grad_(True) for k, v in layer.state_dict().items()}
    x = torch.randn(B, F, din) * 0.5
    gout = torch.randn(B, F, A)
    snap = F2.dropout_snapshot("cuda", 2)
    keep = keep_weights(snap, 1, B, H, F, p).cuda()
    assert 0.5 < float(keep.float().mean()) < 0.9
    xg = x.cuda().requires_grad_(True)
    yg = layer(xg, snapshot=snap, layer=1)
    yg.backward(gout.cuda())
    xr = x.double().cuda().requires_grad_(True)
    yr = AO.self_attention(xr, state, "", H, use_res, use_scale, ln, keep=keep, p=p)
    yr.backward(gout.double().cuda())
    assert close(yg, yr, RTOL), rel_err(yg, yr)
    assert close(xg.grad, xr.grad, RTOL, atol=RTOL * float(xr.grad.abs().max())), rel_err(xg.grad, xr.grad)
    named = dict(layer.named_parameters())
    for k, ref in state.items():
        assert close(named[k].grad, ref.grad, RTOL, atol=RTOL * float(ref.grad.abs().max())), k


def test_eval_mode_is_bit_equal_to_dropout_zero():
    a = make_layer(40, 40, 2, True, True, True, seed=9, dropout=0.4).eval()
    b = make_layer(40, 40, 2, True, True, True, seed=9, dropout=0.0)
    x = (torch.randn(65, 39, 40) * 0.5).cuda()
    assert torch.equal(a(x), b(x))


# ------------------------------------------------------------------ zoo.AutoInt
def _fm_and_batches(n, B, seed, dim):
    import test_gpu_sharded_models as S
    from fuxictr_b200.schema import FeatureMap
    fm = FeatureMap.from_specs(S._CAT, embedding_dim=dim)
    gen = torch.Generator().manual_seed(seed)
    mats = []
    for _ in range(n):
        ids = torch.cat([torch.randint(0, s["vocab_size"], (B, 1), generator=gen) for _, s in S._CAT], 1)
        mats.append(torch.cat([ids.double(), (torch.rand(B, 1, generator=gen) < 0.4).double()], 1).cuda())
    return fm, OrderedDict(S._CAT), mats


# AutoInt_test-like (D 4 != A 8: layer 0 has W_res, K 4), use_wide + layer_norm + use_scale, and no DNN
MODELS = {
    "test": dict(embedding_dim=4, attention_dim=8, num_heads=2, attention_layers=3, dnn_hidden_units=[64, 32]),
    "wide_ln_scale": dict(embedding_dim=16, attention_dim=16, num_heads=2, attention_layers=2,
                          dnn_hidden_units=[32], use_wide=True, layer_norm=True, use_scale=True),
    "no_dnn": dict(embedding_dim=8, attention_dim=12, num_heads=3, attention_layers=2, dnn_hidden_units=[]),
}


def make_model(fm, kw, seed=123, **extra):
    from fuxictr_b200 import zoo
    torch.manual_seed(seed)
    m = zoo.AutoInt(fm, gpu=0, **dict(kw, **extra))
    with torch.no_grad():
        for mod in m.modules():
            if isinstance(mod, torch.nn.Embedding):
                mod.weight[1:].normal_(0, 0.3)
    return m


def oracle_pred(specs, kw):
    nh = len(kw["dnn_hidden_units"]) if kw["dnn_hidden_units"] else None
    return lambda s, X: torch.sigmoid(AO.autoint_logit(
        specs, s, X, kw["attention_layers"], kw["num_heads"], nh, use_scale=kw.get("use_scale", False),
        layer_norm=kw.get("layer_norm", False), use_wide=kw.get("use_wide", False)))


def oracle_step(tr, batch):
    """OracleTrainer.train_step in float64 (the labels cast to the oracle's dtype)."""
    tr.optimizer.zero_grad()
    y_pred, y = tr.forward(batch)
    loss = O.bce_mean(y_pred, y.to(y_pred.dtype))
    loss.backward()
    torch.nn.utils.clip_grad_norm_(tr.params, tr.max_norm)
    tr.optimizer.step()
    return float(loss)


@pytest.mark.parametrize("mode", ["fp32", "tf32x3"])
@pytest.mark.parametrize("name", sorted(MODELS))
def test_model_with_fused_adam_matches_oracle_trajectory(name, mode, mode_of):
    """y_pred and every gradient on batch 0 against the float64 oracle, then three fused_train_steps (fused logit +
    BCE, arena clip + Adam) against the oracle's clip + Adam steps."""
    mode_of(mode)
    kw = MODELS[name]
    fm, specs, mats = _fm_and_batches(3, 256, seed=len(name), dim=kw["embedding_dim"])
    model = make_model(fm, kw)
    model.train()
    tr = O.OracleTrainer({k: v.double() for k, v in model.state_dict().items()}, oracle_pred(specs, kw), specs,
                         fm.labels)
    model.use_fused_optimizer()
    batches = [fm.batch_dict(m) for m in mats]
    ret = model.forward(batches[0])
    y_ref, y = tr.forward(batches[0])
    assert close(ret["y_pred"], y_ref, RTOL), rel_err(ret["y_pred"], y_ref)
    loss = model.compute_loss(ret, model.get_labels(batches[0]))
    model._fused_optimizer.zero_grad()
    loss.backward()
    O.bce_mean(y_ref, y.double()).backward()
    named = dict(model.named_parameters())
    for k, p in named.items():
        ref = tr.state[k].grad
        assert close(p.grad, ref, RTOL, atol=RTOL * float(ref.abs().max()) + 1e-9), (k, rel_err(p.grad, ref))
    model._arena.zero_grads()
    tr.optimizer.zero_grad()
    losses = [float(model.fused_train_step(b)) for b in batches]
    ref_losses = [oracle_step(tr, b) for b in batches]
    assert close(torch.tensor(losses), torch.tensor(ref_losses), RTOL), (losses, ref_losses)
    sd = model.state_dict()
    for k, v in tr.state.items():
        assert close(sd[k], v, 2e-5), (k, rel_err(sd[k], v))


# ------------------------------------------------------------------ CUDA graph capture
@pytest.mark.parametrize("drop", [0.0, 0.2])
@pytest.mark.parametrize("mode", ["tf32x3", "bf16"])
def test_graph_captured_step_matches_eager(drop, mode, mode_of):
    """Five eager fused_train_steps against three warm-up steps and two replays of the captured step.  With dropout
    the replays draw the masks the eager steps drew (the device RNG state advances inside the graph)."""
    from fuxictr_b200.pipeline import TrainPipeline
    from fuxictr_b200 import functional as F2
    mode_of(mode)
    kw = dict(embedding_dim=16, attention_dim=16, num_heads=2, attention_layers=3, dnn_hidden_units=[32, 16],
              layer_norm=True, use_scale=True, use_wide=True)
    fm, _, mats = _fm_and_batches(1, 512, seed=4, dim=kw["embedding_dim"])
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
    for a, b in zip(got, ref[3:]):
        assert abs(a - b) <= 1e-5 * abs(b), (got, ref)
    sd, want = graphed.state_dict(), eager.state_dict()
    for k, v in want.items():
        assert close(sd[k], v, 1e-5), (k, rel_err(sd[k], v))


# ------------------------------------------------------------------ row-sharded tables, two virtual ranks
@pytest.mark.parametrize("use_wide", [False, True])
def test_two_sharded_ranks_train_like_the_unsharded_model(use_wide):
    """test_gpu_sharded_models.py's lock-step harness: two virtual ranks on one GPU, each with half of every table's
    rows, three fused_train_steps against the unsharded model with torch's clip + Adam on the global batches.  With
    use_wide the sharded front's logit is the LR term alone (no FM)."""
    import test_gpu_sharded_models as S
    from fuxictr_b200.schema import FeatureMap
    world = 2
    fm = FeatureMap.from_specs(S._CAT, embedding_dim=S.D)
    kw = dict(embedding_dim=S.D, attention_dim=8, num_heads=2, attention_layers=2, dnn_hidden_units=[16, 8],
              use_wide=use_wide)

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

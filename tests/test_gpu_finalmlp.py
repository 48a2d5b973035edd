"""FinalMLP on the H100: the gating kernel and the interaction aggregation (pack, GEMM, row kernels and back) against
the reference's goldens and against the float64 oracle over the kernels' launch-plan branches in every matmul mode;
the GEMM operand copies the row kernels write (bf16, and 3xTF32 small parts in HBM) against the values they copy;
zoo.FinalMLP (without and with context features, without feature selection) and zoo.DualMLP with the fused optimizer
along the reference's training trajectories (within the Frobenius bars in TF32 and bf16); a CUDA-graph-captured training step against the eager one; and two
virtual ranks with row-sharded tables against the unsharded model."""
import sys

import pytest
import torch

from conftest import Golden, ROOT, close, rel_err

sys.path.insert(0, ROOT)
import finalmlp_oracle as FO  # noqa: E402

pytestmark = pytest.mark.gpu

RTOL = 1e-5
# single-pass modes: the Frobenius bars of test_gpu_gdcn.py
FRO = {"tf32": (1e-2, 6e-2), "bf16": (3e-2, 1.5e-1)}
MODEL_CASES = ["FinalMLP", "FinalMLP_ctx", "FinalMLP_nofs", "DualMLP"]


@pytest.fixture(scope="module", autouse=True)
def _built():
    import __graft_entry__
    __graft_entry__.build()
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"


@pytest.fixture
def mode_of():
    """Sets a matmul mode; "tf32x3_hbm" is 3xTF32 with the small parts in HBM (set_x3_inline(False)), the layout in
    which the producers of GEMM operands also write their small parts."""
    from fuxictr_b200 import functional as F2

    def set_mode(mode):
        F2.set_x3_inline(mode != "tf32x3_hbm")
        F2.set_matmul_precision("tf32x3" if mode == "tf32x3_hbm" else mode)
    yield set_mode
    F2.set_matmul_precision("fp32")
    F2.set_x3_inline(True)


def operand_copy(t):
    """What the current matmul mode's GEMMs read of t besides t itself: its bf16 rounding, or its 3xTF32 small part
    (b2_split_tf32) in the HBM small-part layout."""
    from fuxictr_b200 import functional as F2
    return t.bfloat16() if F2.get_matmul_precision() == "bf16" else F2.split_tf32(t.contiguous())


def fro(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def check(mode, got, want, what, cond):
    """fp32-class modes: |got - want| <= 1e-5 * cond elementwise, cond the same gradient with every term replaced by
    its magnitude (the float64 oracle on absolute values), the scale of fp32 summation error in a sum that cancels.
    Single-pass modes: the Frobenius bar."""
    if mode in ("fp32", "tf32x3"):
        err = (got.detach().double().cpu() - want.detach().double().cpu()).abs()
        assert (err <= RTOL * cond.detach().double().cpu() + 1e-12).all(), (what, rel_err(got, want))
    else:
        assert fro(got, want) <= FRO[mode][1], (what, fro(got, want))


# ------------------------------------------------------------------ the layers against the reference's goldens
@pytest.mark.parametrize("mode", ["fp32", "tf32x3"])
@pytest.mark.parametrize("tag", ["h1", "h2", "h3", "h2w"])
def test_aggregation_matches_reference_golden(mode, tag, mode_of):
    from fuxictr_b200 import layers
    g = Golden("next_InteractionAggregation")
    _, dx, dy, heads = next(c for c in g.meta["configs"] if c[0] == tag)
    agg = layers.InteractionAggregation(dx, dy, num_heads=heads)
    agg.load_state_dict(g["w_" + tag])
    agg = agg.cuda()
    mode_of(mode)
    x = g["in"]["x_" + tag].cuda().requires_grad_(True)
    y = g["in"]["y_" + tag].cuda().requires_grad_(True)
    out = agg(x, y)
    assert close(out, g["out"][tag], RTOL), rel_err(out, g["out"][tag])
    (out * g["in"]["gout_" + tag].cuda()).sum().backward()
    assert close(x.grad, g["gin"]["x_" + tag], RTOL) and close(y.grad, g["gin"]["y_" + tag], RTOL)
    named = dict(agg.named_parameters())
    for k, ref in g["g_" + tag].items():
        assert close(named[k].grad, ref, RTOL), (k, rel_err(named[k].grad, ref))


@pytest.mark.parametrize("mode", ["fp32", "tf32x3"])
@pytest.mark.parametrize("tag", ["noctx", "ctx"])
def test_feature_selection_matches_reference_golden(mode, tag, mode_of):
    from fuxictr_b200 import layers
    from fuxictr_b200.schema import FeatureMap
    g = Golden("next_FeatureSelection")
    fm = FeatureMap.from_specs(g.meta["specs"], labels=g.meta["labels"], embedding_dim=g.meta["embedding_dim"])
    c1, c2 = g.meta["contexts"][tag]
    D = g.meta["embedding_dim"]
    fs = layers.FeatureSelection(fm, D * fm.num_fields, D, g.meta["fs_hidden_units"], c1, c2)
    fs.load_state_dict(g["w_" + tag])
    fs = fs.cuda()
    mode_of(mode)
    batch = fm.batch_dict(g["in"]["matrix"].cuda())
    X = {k: v for k, v in batch.items() if k not in fm.labels}
    emb = g["in"]["emb_" + tag].cuda().requires_grad_(True)
    f1, f2 = fs(X, emb)
    assert close(f1, g["out"]["f1_" + tag], RTOL) and close(f2, g["out"]["f2_" + tag], RTOL)
    ((f1 * g["in"]["gout1_" + tag].cuda()).sum() + (f2 * g["in"]["gout2_" + tag].cuda()).sum()).backward()
    assert close(emb.grad, g["gin"]["emb_" + tag], RTOL), rel_err(emb.grad, g["gin"]["emb_" + tag])
    named = dict(fs.named_parameters())
    for k, ref in g["g_" + tag].items():
        assert close(named[k].grad, ref, RTOL, atol=RTOL * float(ref.abs().max())), (k, rel_err(named[k].grad, ref))


# ------------------------------------------------------------------ the kernels against the float64 oracle
# (B, d): the float4 gate kernels (d 624, 40) and the scalar ones (d 39, 13, 1); B 0, below one CTA's rows, not a
# multiple of them, and 8192 (many CTAs adding into a broadcast gate's column sums)
GATE_SHAPES = [(0, 40), (5, 40), (37, 40), (8192, 624), (5, 39), (37, 13), (8192, 39), (1, 1), (37, 1)]


@pytest.mark.parametrize("mode", ["fp32", "tf32x3", "tf32", "bf16"])
@pytest.mark.parametrize("rows", [(False, False), (True, False), (True, True)])
@pytest.mark.parametrize("B,d", GATE_SHAPES)
def test_gate_matches_float64_oracle(mode, rows, B, d, mode_of):
    """The gating products alone: a broadcast gate (one row) or a per-row one for each stream.  The kernel is fp32
    in every mode (the mode only decides which operand copies it writes)."""
    from fuxictr_b200 import functional as F2
    mode_of(mode)
    gen = torch.Generator().manual_seed(B * 7 + d)
    e = torch.randn(B, d, generator=gen)
    g1 = torch.rand(B if rows[0] else 1, d, generator=gen)
    g2 = torch.rand(B if rows[1] else 1, d, generator=gen)
    d1, d2 = torch.randn(B, d, generator=gen), torch.randn(B, d, generator=gen)
    leaves = [t.double().cuda().requires_grad_(True) for t in (e, g1, g2)]
    ref1, ref2 = leaves[0] * (2 * leaves[1]), leaves[0] * (2 * leaves[2])
    ((ref1 * d1.double().cuda()).sum() + (ref2 * d2.double().cuda()).sum()).backward()
    ins = [t.cuda().requires_grad_(True) for t in (e, g1, g2)]
    f1, f2 = F2.fs_gate(*ins)
    ((f1 * d1.cuda()).sum() + (f2 * d2.cuda()).sum()).backward()
    for got, want in ((f1, ref1), (f2, ref2)) + tuple((a.grad, b.grad) for a, b in zip(ins, leaves)):
        assert got.shape == want.shape
        if want.numel():
            assert close(got, want, RTOL, atol=RTOL * float(want.abs().max())), rel_err(got, want)


@pytest.mark.parametrize("mode", ["bf16", "tf32x3_hbm"])
@pytest.mark.parametrize("rows", [(False, False), (True, True)])
@pytest.mark.parametrize("B,d", [(5, 40), (37, 40), (8192, 624), (37, 13), (5, 39), (37, 1)])
def test_gate_writes_the_operand_copies_the_towers_read(mode, rows, B, d, mode_of):
    """In bf16 mode and in the HBM small-part 3xTF32 layout the gate kernel also writes f1's and f2's GEMM operand
    copies, which the towers' first layers take (make_aux finds them on the tensors): each must be exactly the bf16
    rounding (round to nearest even), or the small part b2_split_tf32 gives, of its own stream."""
    from fuxictr_b200 import functional as F2
    mode_of(mode)
    gen = torch.Generator().manual_seed(B * 5 + d)
    e = torch.randn(B, d, generator=gen).cuda()
    g1 = torch.rand(B if rows[0] else 1, d, generator=gen).cuda()
    g2 = torch.rand(B if rows[1] else 1, d, generator=gen).cuda()
    f1, f2 = F2.fs_gate(e, g1, g2)
    for f in (f1, f2):
        hint = f._b2_aux
        assert hint[0] == F2.get_matmul_precision() and hint[2] == f._version
        assert F2.make_aux(f).data_ptr() == hint[1].data_ptr()          # what the tower's first GEMM takes
        want = operand_copy(f)
        assert hint[1].dtype == want.dtype and hint[1].shape == want.shape
        assert torch.equal(hint[1], want)
    assert not torch.equal(operand_copy(f1), operand_copy(f2))


@pytest.mark.parametrize("mode", ["bf16", "tf32x3_hbm"])
@pytest.mark.parametrize("B,dy", [(37, 8), (4096, 256), (37, 14), (5, 18)])
def test_aggregation_backward_writes_the_operand_copy_the_gemms_read(mode, B, dy, mode_of):
    """b2_agg_bwd's ys = [g y | g | 0], and its operand copy (the dgrad's and wgrad's A): the bf16 rounding or the
    3xTF32 small part of ys, at the padded row pitch the GEMMs read (float4 path: dy 8, 256; scalar: dy 14, 18)."""
    from fuxictr_b200 import _lib, functional as F2
    mode_of(mode)
    n = (dy + 4) // 4 * 4
    gen = torch.Generator().manual_seed(B + dy)
    Q, y, g = (torch.randn(B, n, generator=gen).cuda(), torch.randn(B, dy, generator=gen).cuda(),
               torch.randn(B, 1, generator=gen).cuda())
    gy, ys = torch.empty(B, dy, device="cuda"), torch.empty(B, n, device="cuda")
    aux = F2.empty_aux(B, n, "cuda")
    gw_y, gb_x, gb_y = torch.zeros(dy, device="cuda"), torch.zeros(1, device="cuda"), torch.zeros(1, device="cuda")
    _lib.call("b2_agg_bwd", F2._ptr(Q), F2._ptr(y), F2._ptr(g), B, dy, F2._ptr(gy), F2._ptr(ys), *F2._aux_args(aux),
              F2._ptr(gw_y), F2._ptr(gb_x), F2._ptr(gb_y), F2._stream())
    want = torch.cat([g * y, g, torch.zeros(B, n - dy - 1, device="cuda")], dim=1)
    assert torch.equal(ys, want) and torch.equal(gy, g * Q[:, :dy])
    assert torch.equal(aux, operand_copy(ys))
    # column sums by per-CTA partials and float atomics: fp32 summation error, bounded by the sum of magnitudes (the
    # two biases' sums arrive in their own atomic order, so they need not agree bit for bit)
    assert ((gw_y.double() - want[:, :dy].double().sum(0)).abs() <= RTOL * (g * y).abs().double().sum(0)).all()
    for gb in (gb_x, gb_y):
        assert abs(float(gb) - float(g.double().sum())) <= RTOL * float(g.abs().double().sum())


# (B, dx, dy, H): tensor-core GEMMs with the float4 row kernels (20 | 12, 64 | 32, 512 | 256 at H 2 and 16),
# the SIMT GEMM with scalar row kernels (26 | 14, 30 | 18: dx % 4 != 0), the SIMT GEMM with float4 row kernels
# (W_aug under 16 rows: dy 8), and B 0
AGG_SHAPES = [(5, 20, 12, 1), (37, 64, 32, 2), (4096, 512, 256, 2), (1000, 512, 512, 16), (37, 26, 14, 2),
              (4096, 30, 18, 3), (37, 64, 8, 2), (0, 64, 32, 2)]


@pytest.mark.parametrize("mode", ["fp32", "tf32x3", "tf32", "bf16"])
@pytest.mark.parametrize("B,dx,dy,heads", AGG_SHAPES)
def test_aggregation_matches_float64_oracle(mode, B, dx, dy, heads, mode_of):
    from fuxictr_b200 import layers
    torch.manual_seed(B + dx + dy)
    agg = layers.InteractionAggregation(dx, dy, num_heads=heads)
    with torch.no_grad():
        agg.w_x.bias.fill_(0.3)
        agg.w_y.bias.fill_(-0.2)
    state = {k: v.detach().double().cuda().requires_grad_(True) for k, v in agg.state_dict().items()}
    gen = torch.Generator().manual_seed(dx * 7 + B)
    x, y = torch.rand(B, dx, generator=gen), torch.rand(B, dy, generator=gen)       # ReLU outputs are >= 0
    gout = torch.randn(B, 1, generator=gen)
    xr, yr = x.double().cuda().requires_grad_(True), y.double().cuda().requires_grad_(True)
    outr = FO.interaction_aggregation(state, "", xr, yr, heads)
    outr.backward(gout.double().cuda())
    cond_state = {k: v.detach().abs().requires_grad_(True) for k, v in state.items()}
    xa, ya = xr.detach().abs().requires_grad_(True), yr.detach().abs().requires_grad_(True)
    FO.interaction_aggregation(cond_state, "", xa, ya, heads).backward(gout.double().abs().cuda())
    agg = agg.cuda()
    mode_of(mode)
    xg, yg = x.cuda().requires_grad_(True), y.cuda().requires_grad_(True)
    out = agg(xg, yg)
    out.backward(gout.cuda())
    assert out.shape == (B, 1)
    named = dict(agg.named_parameters())
    if B == 0:
        for k, ref in state.items():
            assert float(named[k].grad.abs().max()) == 0.0, k
        return
    if mode in ("fp32", "tf32x3"):
        assert close(out, outr, RTOL), rel_err(out, outr)
    else:
        assert fro(out, outr) <= FRO[mode][0]
    check(mode, xg.grad, xr.grad, "x", xa.grad)
    check(mode, yg.grad, yr.grad, "y", ya.grad)
    for k, ref in state.items():
        check(mode, named[k].grad, ref.grad, k, cond_state[k].grad)


# ------------------------------------------------------------------ the models along the golden trajectories
def build_model(case, g):
    from fuxictr_b200 import zoo
    from fuxictr_b200.schema import FeatureMap
    fm = FeatureMap.from_specs(g.meta["specs"], labels=g.meta["labels"], embedding_dim=g.meta["kwargs"]["embedding_dim"])
    model = getattr(zoo, g.meta["model"])(fm, gpu=-1, **g.meta["kwargs"])
    model.load_state_dict(g["w"])
    model.device = torch.device("cuda:0")
    model.model_to_device()
    model.compile("adam", "binary_crossentropy", 1e-3)
    model.train()
    model.use_fused_optimizer()
    return fm, model


@pytest.mark.parametrize("mode", ["fp32", "tf32x3", "tf32x3_hbm"])
@pytest.mark.parametrize("case", MODEL_CASES)
def test_model_with_fused_adam_matches_reference_trajectory(case, mode, mode_of):
    """test_gpu_gdcn.py's model recipe with the fused optimizer: y_pred, loss and every gradient on batch 0, then
    three fused_train_steps (fused logit + BCE, arena clip + Adam) against the reference's train_step()s.
    tf32x3_hbm: the gate kernel, the aggregation's row kernel and the MLP chain hand their operands' small parts on
    through HBM."""
    mode_of(mode)
    g = Golden("model_" + case)
    fm, model = build_model(case, g)
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
        assert close(named[k].grad, ref, RTOL), (k, rel_err(named[k].grad, ref))
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


@pytest.mark.parametrize("mode", ["tf32", "bf16"])
@pytest.mark.parametrize("case", MODEL_CASES)
def test_model_in_single_pass_modes_matches_reference_within_frobenius_bars(case, mode, mode_of):
    """y_pred, all gradients on batch 0 taken together, and the losses of three fused_train_steps against the
    reference's.  In bf16 the towers' first GEMMs multiply the bf16 copies the gate kernel wrote, and the aggregation's
    dgrad and wgrad the copy of ys its row kernel wrote.  The gradients are judged as one vector: single parameters of
    these small models can have gradients that cancel, and exact bf16 operand rounding alone (restated on the CPU)
    leaves up to 0.43 relative Frobenius error in one gate bias of FinalMLP_ctx, but 0.054 at most over all of a
    model's gradients."""
    mode_of(mode)
    g = Golden("model_" + case)
    fm, model = build_model(case, g)
    B = g.meta["batch"]
    mat = g["in"]["matrix"].cuda()
    batches = [fm.batch_dict(mat[i * B:(i + 1) * B]) for i in range(3)]
    ret = model.forward(batches[0])
    tol_y, tol = FRO[mode]
    assert fro(ret["y_pred"], g["out"]["y_pred"]) <= tol_y
    loss = model.compute_loss(ret, model.get_labels(batches[0]))
    model._fused_optimizer.zero_grad()
    loss.backward()
    named = dict(model.named_parameters())
    keys = list(g["g"])
    got = torch.cat([named[k].grad.detach().flatten().cpu() for k in keys])
    assert fro(got, torch.cat([g["g"][k].flatten() for k in keys])) <= tol
    model._arena.zero_grads()
    losses = torch.tensor([float(model.fused_train_step(b)) for b in batches])
    assert fro(losses, g["out"]["step_losses"]) <= tol_y


# ------------------------------------------------------------------ CUDA graph capture
@pytest.mark.parametrize("mode", ["tf32x3", "bf16"])
@pytest.mark.parametrize("case", ["FinalMLP", "FinalMLP_ctx", "DualMLP"])
def test_graph_captured_step_matches_eager(case, mode, mode_of):
    """Five eager fused_train_steps against three warm-up steps and two replays of the captured step (the gate MLPs,
    the gating kernel, the aggregation's pack, GEMMs and row kernels, and the operand copies they hand on are all
    in the graph)."""
    from fuxictr_b200.pipeline import TrainPipeline
    mode_of(mode)
    g = Golden("model_" + case)
    fm, eager = build_model(case, g)
    _, graphed = build_model(case, g)
    mat = g["in"]["matrix"][:g.meta["batch"]].cuda()
    ref = [float(eager.fused_train_step(fm.batch_dict(mat))) for _ in range(5)]
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
@pytest.mark.parametrize("name", ["FinalMLP", "DualMLP"])
def test_two_sharded_ranks_train_like_the_unsharded_model(name):
    """test_gpu_sharded_models.py's lock-step harness: two virtual ranks on one GPU, each with half of every table's
    rows, three fused_train_steps against the unsharded model with torch's clip + Adam on the global batches."""
    import test_gpu_sharded_models as S
    from fuxictr_b200 import zoo
    from fuxictr_b200.schema import FeatureMap
    world = 2
    fm = FeatureMap.from_specs(S._CAT, embedding_dim=S.D)

    def make():
        torch.manual_seed(123)
        m = getattr(zoo, name)(fm, gpu=0, embedding_dim=S.D, mlp1_hidden_units=[16, 8], mlp2_hidden_units=[16, 12],
                               fs_hidden_units=[16], num_heads=2)
        with torch.no_grad():
            for mod in m.modules():
                if isinstance(mod, torch.nn.Embedding):
                    mod.weight[1:].normal_(0, 0.3)
        return m
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

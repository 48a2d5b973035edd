"""MaskNet on the H100: the mask block and the embedding LayerNorm against the reference's golden and against the float64
oracle over the row kernels' and GEMMs' branches in every matmul mode; the operand copies the row kernel writes; the
dropout masks against the host restatement; zoo.MaskNet (serial, parallel, no LayerNorm) with the fused optimizer
along the reference's training trajectory; eval against dropout 0; a CUDA-graph-captured step against the eager one;
and two virtual ranks with row-sharded tables against the unsharded model."""
import sys

import pytest
import torch

from conftest import Golden, ROOT, close, rel_err

sys.path.insert(0, ROOT)
import masknet_oracle as MO  # noqa: E402

pytestmark = pytest.mark.gpu

RTOL = 1e-5
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


def near(got, ref, tol=RTOL):
    return close(got, ref, tol, atol=tol * max(float(ref.detach().abs().max()), 1e-30))


@pytest.mark.parametrize("mode", ["fp32", "tf32x3"])
@pytest.mark.parametrize("n", [20, 13])
def test_block_matches_reference_golden(mode, n, mode_of):
    from fuxictr_b200 import layers
    g = Golden("next_MaskBlock")
    blk = layers.MaskBlock(g.meta["input_dim"], g.meta["hidden_dim"], n, g.meta["widths"][str(n)],
                           g.meta["reduction_ratio"], 0, True)
    blk.load_state_dict(g["w_n%d" % n])
    blk = blk.cuda()
    mode_of(mode)
    emb = g["in"]["emb_n%d" % n].cuda().requires_grad_(True)
    hid = g["in"]["hid_n%d" % n].cuda().requires_grad_(True)
    out = blk(emb, hid)
    assert close(out, g["out"]["y_n%d" % n], RTOL), rel_err(out, g["out"]["y_n%d" % n])
    (out * g["in"]["gout_n%d" % n].cuda()).sum().backward()
    assert near(emb.grad, g["gin"]["emb_n%d" % n]), rel_err(emb.grad, g["gin"]["emb_n%d" % n])
    assert near(hid.grad, g["gin"]["hid_n%d" % n]), rel_err(hid.grad, g["gin"]["hid_n%d" % n])
    named = dict(blk.named_parameters())
    for k, ref in g["g_n%d" % n].items():
        assert near(named[k].grad, ref), (k, rel_err(named[k].grad, ref))


def _blocks(nb, d, hd, n, act, ln, seed):
    from fuxictr_b200 import layers
    torch.manual_seed(seed)
    blks = [layers.MaskBlock(d, hd, n, act, 1.0, 0, ln) for _ in range(nb)]
    gen = torch.Generator().manual_seed(seed)
    for b in blks:
        if ln:
            with torch.no_grad():
                b.hidden_layer[1].weight.copy_(1 + 0.4 * torch.randn(n, generator=gen))
                b.hidden_layer[1].bias.copy_(0.3 * torch.randn(n, generator=gen))
    return blks


# (B, d, hd, n, nb): the float4 row kernel (n % 4 == 0) on its register tier (n <= 256) and its wide one (n 400,
# 1024), the scalar row kernel (n 1, 13, 1023), tensor-core GEMMs (d, hd >= 16, % 4) and SIMT ones (d 13, hd 13);
# B 0, 1, 37 and 4096 (many CTAs adding into the LayerNorm gradients); nb 3: three blocks into one concatenation
SHAPES = [(37, 64, 64, 20, 1), (1, 64, 64, 20, 1), (0, 64, 64, 20, 1), (4096, 624, 624, 64, 3), (37, 64, 32, 13, 1),
          (37, 64, 32, 1, 1), (37, 13, 13, 7, 2), (4096, 160, 400, 400, 1), (37, 64, 64, 1024, 1),
          (37, 64, 64, 1023, 1), (37, 48, 48, 8, 3)]


@pytest.mark.parametrize("mode", ["fp32", "tf32x3", "tf32", "bf16"])
@pytest.mark.parametrize("B,d,hd,n,nb", SHAPES)
@pytest.mark.parametrize("act,ln", [("relu", True), ("sigmoid", False)])
def test_blocks_match_float64_oracle(mode, B, d, hd, n, nb, act, ln, mode_of):
    from fuxictr_b200 import layers
    blks = _blocks(nb, d, hd, n, act, ln, B + n + nb)
    states = [{k: v.detach().double().cuda().requires_grad_(True) for k, v in b.state_dict().items()} for b in blks]
    gen = torch.Generator().manual_seed(d + hd + B)
    emb = torch.randn(B, d, generator=gen) * 0.5 + 0.1
    hid = torch.randn(B, hd, generator=gen) * 0.5 + 0.2
    gout = torch.randn(B, nb * n, generator=gen)
    er, hr = emb.double().cuda().requires_grad_(True), hid.double().cuda().requires_grad_(True)
    yr = torch.cat([MO.mask_block(s, "", er, hr, act, ln) for s in states], dim=1)
    yr.backward(gout.double().cuda())
    # torch fp32 on the same inputs: where a ReLU input lies within fp32 rounding of 0, fp32 arithmetic and float64
    # take different branches; err(ours, fp64) <= max(1e-5, 3 err(torch fp32, fp64)) (test_gpu_kernel_sweep.py's bar)
    states32 = [{k: v.detach().float().requires_grad_(True) for k, v in s.items()} for s in states]
    e32, h32 = emb.cuda().requires_grad_(True), hid.cuda().requires_grad_(True)
    y32 = torch.cat([MO.mask_block(s, "", e32, h32, act, ln) for s in states32], dim=1)
    y32.backward(gout.cuda())
    blks = [b.cuda() for b in blks]
    mode_of(mode)
    eg, hg = emb.cuda().requires_grad_(True), hid.cuda().requires_grad_(True)
    yg = layers._run_mask_blocks(blks, eg, hg, want_aux=nb > 1)
    yg.backward(gout.cuda())
    if B == 0:
        assert yg.shape == (0, nb * n)
        return
    pairs = [(yg, yr, y32), (eg.grad, er.grad, e32.grad), (hg.grad, hr.grad, h32.grad)]
    for b, s, s32 in zip(blks, states, states32):
        named = dict(b.named_parameters())
        pairs += [(named[k].grad, s[k].grad, s32[k].grad) for k in s]
    if mode in ("fp32", "tf32x3"):
        for i, (got, ref, t32) in enumerate(pairs):
            assert near(got, ref) or rel_err(got, ref) <= 3 * rel_err(t32, ref), (i, rel_err(got, ref))
        return
    assert fro(yg, yr) <= FRO[mode][0]
    for got, ref, _ in pairs[1:3]:
        assert fro(got, ref) <= FRO[mode][1]
    flat = lambda ts: torch.cat([t.detach().double().flatten().cpu() for t in ts])  # noqa: E731
    assert fro(flat(p[0] for p in pairs[3:]), flat(p[1] for p in pairs[3:])) <= FRO[mode][1]


@pytest.mark.parametrize("mode,inline", [("bf16", True), ("tf32x3", False)])
@pytest.mark.parametrize("n", [8, 13])
def test_operand_copies_are_bit_exact(mode, inline, n, mode_of):
    """The copy of the concatenation the row kernel writes for the MLP's GEMM: the bf16 rounding, or the 3xTF32
    small part, of exactly the values it wrote."""
    from fuxictr_b200 import layers, functional as F2
    blks = [b.cuda() for b in _blocks(3, 32, 32, n, "relu", True, 5)]
    mode_of(mode)
    F2.set_x3_inline(inline)
    emb = torch.randn(300, 32, device="cuda")
    out = layers._run_mask_blocks(blks, emb, emb, want_aux=True)
    aux = out._b2_aux[1]
    want = out.to(torch.bfloat16) if mode == "bf16" else F2.split_tf32(out)
    assert torch.equal(aux, want)


@pytest.mark.parametrize("mode", ["fp32", "tf32x3", "tf32", "bf16"])
@pytest.mark.parametrize("B,F,D", [(37, 39, 40), (4096, 39, 40), (1, 5, 13), (37, 3, 1), (37, 2, 1024),
                                   (37, 2, 1021), (0, 4, 8), (4096, 26, 16)])
def test_embedding_layernorm_matches_float64_oracle(mode, B, F, D, mode_of):
    """All F fields in one launch each way (float4 and scalar paths, widths 1 to 1024) with the parameters at their
    stride; the input gradient adds into the shared buffer."""
    from fuxictr_b200 import functional as F2
    norms = torch.nn.ModuleList(torch.nn.LayerNorm(D) for _ in range(F)).cuda()
    gen = torch.Generator().manual_seed(B + F + D)
    with torch.no_grad():
        for m in norms:
            m.weight.copy_(1 + 0.3 * torch.randn(D, generator=gen))
            m.bias.copy_(0.2 * torch.randn(D, generator=gen))
    F2.pack_field_params(norms)
    state = {"%d.%s" % (f, k): getattr(m, k).detach().double().requires_grad_(True)
             for f, m in enumerate(norms) for k in ("weight", "bias")}
    x = (torch.randn(B, F * D, generator=gen) * 2 + 5).cuda()         # mean large against the spread
    g = torch.randn(B, F * D, generator=gen).cuda()
    xr = x.double().requires_grad_(True)
    yr = MO.field_layernorm(state, "", xr, F)
    yr.backward(g.double())
    mode_of(mode)
    xg = x.clone().requires_grad_(True)
    v, sink = F2.shared_grad(xg)
    yg = F2.field_layernorm(v, sink, [m.weight for m in norms], [m.bias for m in norms])
    yg.backward(g)
    if B == 0:
        return
    assert near(yg, yr), rel_err(yg, yr)
    assert near(xg.grad, xr.grad), rel_err(xg.grad, xr.grad)
    for f, m in enumerate(norms):
        assert near(m.weight.grad, state["%d.weight" % f].grad, 2e-5)
        assert near(m.bias.grad, state["%d.bias" % f].grad, 2e-5)


@pytest.mark.parametrize("n", [20, 13])
def test_dropout_masks_match_host_restatement(n, mode_of):
    """Training-mode blocks draw keep(seed, offset + k, row, column) over each block's (B, n) output; the output and
    every gradient then match the oracle given those masks."""
    import test_mlp_dropout_host as H
    from fuxictr_b200 import layers, functional as F2
    p, B, nb = 0.3, 64, 2
    torch.manual_seed(7)
    blks = [layers.MaskBlock(24, 24, n, "relu", 1, p, True).cuda() for _ in range(nb)]
    states = [{k: v.detach().double().requires_grad_(True) for k, v in b.state_dict().items()} for b in blks]
    mode_of("tf32x3")
    emb = torch.randn(B, 24, device="cuda")
    eg = emb.clone().requires_grad_(True)
    state = F2.dropout_state(eg.device)
    seed, off = [int(v) for v in state.cpu()]
    out = layers._run_mask_blocks(blks, eg, eg)
    gout = torch.randn_like(out)
    out.backward(gout)
    scale = F2.dropout_consts(p)[1]
    keeps = [torch.from_numpy(H.keep_mask(seed, off + k, B, n, p).astype("float64")).cuda() for k in range(nb)]
    er = emb.double().requires_grad_(True)
    yr = torch.cat([MO.mask_block(s, "", er, er, "relu", True, keeps[k], scale) for k, s in enumerate(states)], 1)
    yr.backward(gout.double())
    assert bool((out[torch.cat(keeps, 1) == 0] == 0).all())
    assert near(out, yr) and near(eg.grad, er.grad)
    for b, s in zip(blks, states):
        named = dict(b.named_parameters())
        for k in s:
            assert near(named[k].grad, s[k].grad), k


# ------------------------------------------------------------------ zoo.MaskNet along the golden trajectory
def build_model(g, **over):
    from fuxictr_b200 import zoo
    from fuxictr_b200.schema import FeatureMap
    fm = FeatureMap.from_specs(g.meta["specs"], labels=g.meta["labels"], embedding_dim=g.meta["kwargs"]["embedding_dim"])
    model = zoo.MaskNet(fm, gpu=-1, **dict(g.meta["kwargs"], **over))
    # a Dropout in ParallelMaskNet's MLP shifts the MLP's child indices: the golden weights go over in order
    model.load_state_dict(dict(zip(model.state_dict().keys(), g["w"].values())))
    model.device = torch.device("cuda:0")
    model.model_to_device()
    model.compile("adam", "binary_crossentropy", 1e-3)
    model.train()
    model.use_fused_optimizer()
    return fm, model


@pytest.mark.parametrize("mode", ["fp32", "tf32x3", "tf32", "bf16"])
@pytest.mark.parametrize("case", ["serial", "parallel", "noln"])
def test_model_with_fused_adam_matches_reference_trajectory(case, mode, mode_of):
    mode_of(mode)
    g = Golden("model_MaskNet_" + case)
    fm, model = build_model(g)
    B = g.meta["batch"]
    mat = g["in"]["matrix"].cuda()
    batches = [fm.batch_dict(mat[i * B:(i + 1) * B]) for i in range(3)]
    ret = model.forward(batches[0])
    loss = model.compute_loss(ret, model.get_labels(batches[0]))
    model._fused_optimizer.zero_grad()
    loss.backward()
    named = dict(model.named_parameters())
    exact = mode in ("fp32", "tf32x3")
    if exact:
        assert close(ret["y_pred"], g["out"]["y_pred"], RTOL)
        for k, ref in g["g"].items():
            assert near(named[k].grad, ref), (k, rel_err(named[k].grad, ref))
    else:
        assert fro(ret["y_pred"], g["out"]["y_pred"]) <= FRO[mode][0]
        got = torch.cat([named[k].grad.flatten().cpu() for k in g["g"]])
        assert fro(got, torch.cat([v.flatten() for v in g["g"].values()])) <= FRO[mode][1]
    model._arena.zero_grads()
    losses = []
    for i in range(3):
        losses.append(float(model.fused_train_step(batches[i])))
        if i == 0 and exact:
            sd = model.state_dict()
            for k, ref in g["w1"].items():
                assert close(sd[k], ref, RTOL), (k, rel_err(sd[k], ref))
    if exact:
        assert close(torch.tensor(losses), g["out"]["step_losses"], RTOL)
        sd = model.state_dict()
        for k, ref in g["w3"].items():
            assert close(sd[k], ref, 2e-5), (k, rel_err(sd[k], ref))
    else:
        assert fro(torch.tensor(losses), g["out"]["step_losses"]) <= FRO[mode][0]


@pytest.mark.parametrize("case", ["serial", "parallel"])
def test_eval_is_bit_equal_to_dropout_zero(case, mode_of):
    mode_of("tf32x3")
    g = Golden("model_MaskNet_" + case)
    fm, dropped = build_model(g, net_dropout=0.3)
    _, plain = build_model(g)
    mat = g["in"]["matrix"][:g.meta["batch"]].cuda()
    dropped.fused_train_step(fm.batch_dict(mat))            # a training step draws masks and moves the weights
    plain.load_state_dict(dict(zip(plain.state_dict().keys(), dropped.state_dict().values())))
    dropped.eval()
    plain.eval()
    with torch.no_grad():
        a = dropped.forward(fm.batch_dict(mat))["y_pred"]
        b = plain.forward(fm.batch_dict(mat))["y_pred"]
    assert torch.equal(a, b)


# ------------------------------------------------------------------ CUDA graph capture
@pytest.mark.parametrize("mode", ["tf32x3", "bf16"])
@pytest.mark.parametrize("case,drop", [("serial", 0.0), ("parallel", 0.0), ("serial", 0.2), ("parallel", 0.2)])
def test_graph_captured_step_matches_eager(case, drop, mode, mode_of):
    """Five eager fused_train_steps against three warm-up steps and two replays of the captured step.  With dropout
    the replays draw the masks the eager steps drew (the device RNG state advances inside the graph)."""
    from fuxictr_b200.pipeline import TrainPipeline
    from fuxictr_b200 import functional as F2
    mode_of(mode)
    g = Golden("model_MaskNet_" + case)
    fm, eager = build_model(g, net_dropout=drop)
    _, graphed = build_model(g, net_dropout=drop)
    mat = g["in"]["matrix"][:g.meta["batch"]].cuda()
    torch.manual_seed(11)
    F2._DROPOUT.clear()             # a state left by an earlier test under the same seed would be reused
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
@pytest.mark.parametrize("model_type", ["SerialMaskNet", "ParallelMaskNet"])
def test_two_sharded_ranks_train_like_the_unsharded_model(model_type):
    import test_gpu_sharded_models as S
    from fuxictr_b200 import zoo
    from fuxictr_b200.schema import FeatureMap
    world = 2
    fm = FeatureMap.from_specs(S._CAT, embedding_dim=S.D)

    def make():
        torch.manual_seed(123)
        m = zoo.MaskNet(fm, gpu=0, embedding_dim=S.D, dnn_hidden_units=[16, 8], model_type=model_type,
                        parallel_num_blocks=2, parallel_block_dim=8)
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

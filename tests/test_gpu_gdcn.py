"""GDCN on the H100: the gated cross layer (pack, GEMM, row kernel and back) against the reference's golden and
against the float64 oracle over the kernels' launch-plan branches in every matmul mode; zoo.GDCN and zoo.GDCNP with
the fused optimizer along the reference's training trajectory; a CUDA-graph-captured training step against the eager
one; and two virtual ranks with row-sharded tables against the unsharded model."""
import sys

import pytest
import torch

from conftest import Golden, ROOT, close, rel_err

sys.path.insert(0, ROOT)
import gdcn_oracle as GO  # noqa: E402

pytestmark = pytest.mark.gpu

RTOL = 1e-5
# single-pass modes: the Frobenius bars of test_gpu_crossnet_mix.py
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


def fro(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


@pytest.mark.parametrize("mode", ["fp32", "tf32x3"])
@pytest.mark.parametrize("d", [20, 13])
def test_layer_matches_reference_golden(mode, d, mode_of):
    from fuxictr_b200 import layers
    g = Golden("next_GateCorssLayer")
    layer = layers.GateCorssLayer(d, g.meta["cn_layers"])
    layer.load_state_dict(g["w_d%d" % d])
    layer = layer.cuda()
    mode_of(mode)
    x = g["in"]["x_d%d" % d].cuda().requires_grad_(True)
    out = layer(x)
    assert close(out, g["out"]["y_d%d" % d], RTOL), rel_err(out, g["out"]["y_d%d" % d])
    (out * g["in"]["gout_d%d" % d].cuda()).sum().backward()
    assert close(x.grad, g["gin"]["x_d%d" % d], RTOL), rel_err(x.grad, g["gin"]["x_d%d" % d])
    named = dict(layer.named_parameters())
    want = g["g_d%d" % d]
    scale = max(float(v.abs().max()) for v in want.values())
    for k, ref in want.items():
        assert close(named[k].grad, ref, RTOL, atol=RTOL * scale), (k, rel_err(named[k].grad, ref))


# (B, d): the float4 row kernels with the tensor-core GEMM (d 20, 624), the float4 row kernels with the SIMT GEMM
# (d 12 < 16), the scalar row kernels with the SIMT GEMM (d 13, 1); B below one CTA's rows (5 < 8 rows of 32 slots
# at d 20, 13, 12; 1), B not a multiple of them (37), and B 8192 (many CTAs adding into db)
SHAPES = [(5, 20), (37, 20), (8192, 20), (5, 12), (37, 12), (5, 13), (37, 13), (8192, 13), (1, 1), (37, 1),
          (5, 624), (37, 624), (8192, 624)]


@pytest.mark.parametrize("mode", ["fp32", "tf32x3", "tf32", "bf16"])
@pytest.mark.parametrize("B,d", SHAPES)
def test_layer_matches_float64_oracle(mode, B, d, mode_of):
    from fuxictr_b200 import layers
    nl = 3
    torch.manual_seed(B + d)
    layer = layers.GateCorssLayer(d, nl)
    state = {k: v.detach().double().cuda().requires_grad_(True) for k, v in layer.state_dict().items()}
    gen = torch.Generator().manual_seed(d * 7 + B)
    x = torch.randn(B, d, generator=gen) * 0.5
    gout = torch.randn(B, d, generator=gen)
    xr = x.double().cuda().requires_grad_(True)
    yr = GO.gate_cross_net(xr, state, "", nl)
    yr.backward(gout.double().cuda())
    layer = layer.cuda()
    mode_of(mode)
    xg = x.cuda().requires_grad_(True)
    yg = layer(xg)
    yg.backward(gout.cuda())
    named = dict(layer.named_parameters())
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


# ------------------------------------------------------------------ zoo.GDCN / zoo.GDCNP along the golden trajectory
def build_model(name, g):
    from fuxictr_b200 import zoo
    from fuxictr_b200.schema import FeatureMap
    fm = FeatureMap.from_specs(g.meta["specs"], labels=g.meta["labels"], embedding_dim=g.meta["kwargs"]["embedding_dim"])
    model = getattr(zoo, name)(fm, gpu=-1, **g.meta["kwargs"])
    model.load_state_dict(g["w"])
    model.device = torch.device("cuda:0")
    model.model_to_device()
    model.compile("adam", "binary_crossentropy", 1e-3)
    model.train()
    model.use_fused_optimizer()
    return fm, model


@pytest.mark.parametrize("mode", ["fp32", "tf32x3"])
@pytest.mark.parametrize("name", ["GDCN", "GDCNP"])
def test_model_with_fused_adam_matches_reference_trajectory(name, mode, mode_of):
    """test_gpu_parity.py's model recipe with the fused optimizer: y_pred, loss and every gradient on batch 0, then
    three fused_train_steps (fused logit + BCE, arena clip + Adam) against the reference's train_step()s."""
    mode_of(mode)
    g = Golden("model_" + name)
    fm, model = build_model(name, g)
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


# ------------------------------------------------------------------ CUDA graph capture
@pytest.mark.parametrize("mode", ["tf32x3", "bf16"])
@pytest.mark.parametrize("name", ["GDCN", "GDCNP"])
def test_graph_captured_step_matches_eager(name, mode, mode_of):
    """Five eager fused_train_steps against three warm-up steps and two replays of the captured step (the layer's
    pack, GEMMs, row kernels and the operand copies they hand on are all in the graph)."""
    from fuxictr_b200.pipeline import TrainPipeline
    mode_of(mode)
    g = Golden("model_" + name)
    fm, eager = build_model(name, g)
    _, graphed = build_model(name, g)
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
@pytest.mark.parametrize("name", ["GDCN", "GDCNP"])
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
        m = getattr(zoo, name)(fm, gpu=0, embedding_dim=S.D, dnn_hidden_units=[16, 8], num_cross_layers=2)
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

"""CrossNetMix on the H100: the layer (pack, GEMM1, row kernel, GEMM2 and back) against the reference's
golden and against the oracle in float64 across the kernels' branches in every matmul mode; a DCNv2 with
the mixture composed from mirror layers along the reference's training trajectory; and the unmodified
reference DCNv2 (use_low_rank_mixture=True) on cuda:0 under patch.enable() against itself on CPU."""
import logging
import os
import sys
import tempfile

import pytest
import torch

from conftest import Golden, ROOT, close, rel_err

sys.path.insert(0, ROOT)
from oracle import fuxictr_oracle as O  # noqa: E402
from baseline import refenv  # noqa: E402

pytestmark = pytest.mark.gpu

RTOL = 1e-5
# single-pass modes: the Frobenius bars of test_gpu_parity.py::test_mlp_chain_matches_torch_autograd
FRO = {"tf32": (1e-2, 6e-2), "bf16": (3e-2, 1.5e-1)}


@pytest.fixture(scope="module", autouse=True)
def _built():
    import __graft_entry__
    __graft_entry__.build()
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"


@pytest.fixture
def mode_of():
    from fuxictr_b200 import functional as F2

    def set_mode(mode):
        F2.set_matmul_precision(mode)
    yield set_mode
    F2.set_matmul_precision("fp32")


def fro(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


@pytest.mark.parametrize("mode", ["fp32", "tf32x3"])
def test_layer_matches_reference_golden(mode, mode_of):
    from fuxictr_b200 import layers
    g = Golden("next_CrossNetMix")
    m = g.meta
    layer = layers.CrossNetMix(g["in"]["x"].shape[1], m["layer_num"], m["low_rank"], m["num_experts"])
    layer.load_state_dict(g["w"])
    layer = layer.cuda()
    mode_of(mode)
    x = g["in"]["x"].cuda().requires_grad_(True)
    out = layer(x)
    assert close(out, g["out"]["y"], RTOL), rel_err(out, g["out"]["y"])
    (out * g["in"]["gout"].cuda()).sum().backward()
    assert close(x.grad, g["gin"]["x"], RTOL), rel_err(x.grad, g["gin"]["x"])
    named = dict(layer.named_parameters())
    scale = max(float(v.abs().max()) for v in g["g"].values())
    for k, want in g["g"].items():
        assert close(named[k].grad, want, RTOL, atol=RTOL * scale), (k, rel_err(named[k].grad, want))


# (B, d, r, E): SIMT GEMMs (d 10, or a packed side under 16), the tensor-core GEMMs (d 20 with N1, K2 >= 16; d 624),
# one and several lanes' worth of rank columns, E*r at the kernels' bound (256), a single row (squeezed output),
# and C3's B 8192 (many CTAs adding into dC)
SHAPES = [(5, 10, 4, 3), (1, 10, 7, 1), (5, 20, 4, 4), (8192, 20, 7, 3), (5, 20, 1, 8), (1, 624, 32, 4),
          (8192, 624, 32, 4), (5, 624, 64, 4), (8192, 624, 32, 8), (8192, 624, 1, 1), (5, 624, 7, 8)]


@pytest.mark.parametrize("mode", ["fp32", "tf32x3", "tf32", "bf16"])
@pytest.mark.parametrize("B,d,r,E", SHAPES)
def test_layer_matches_float64_oracle(mode, B, d, r, E, mode_of):
    from fuxictr_b200 import layers
    nl = 2
    torch.manual_seed(B + d + 10 * r + E)
    layer = layers.CrossNetMix(d, layer_num=nl, low_rank=r, num_experts=E)
    with torch.no_grad():
        for b in layer.bias:
            b.normal_(0, 0.1)
        for gl in layer.gating:
            gl.weight.mul_(4.0)                   # gates far from uniform, so the softmax matters
    state = {k: v.detach().double().cuda().requires_grad_(True) for k, v in layer.state_dict().items()}
    gen = torch.Generator().manual_seed(d * 7 + B)
    x = torch.randn(B, d, generator=gen) * 0.5
    gout = torch.randn(B, d, generator=gen)
    xr = x.double().cuda().requires_grad_(True)
    yr = O.crossnet_mix(state, "", xr, nl, E)
    yr.backward(gout.double().cuda())
    layer = layer.cuda()
    mode_of(mode)
    xg = x.cuda().requires_grad_(True)
    yg = layer(xg)
    if B == 1:
        assert tuple(yg.shape) == (d,)                # the reference's x_l.squeeze()
    yg.backward(gout.cuda().view(yg.shape))
    named = dict(layer.named_parameters())
    if mode in ("fp32", "tf32x3"):
        assert close(yg, yr.view(yg.shape), RTOL), rel_err(yg, yr.view(yg.shape))
        assert close(xg.grad, xr.grad, RTOL, atol=RTOL * float(xr.grad.abs().max())), rel_err(xg.grad, xr.grad)
        for k, ref in state.items():
            assert close(named[k].grad, ref.grad, RTOL, atol=RTOL * float(ref.grad.abs().max())), \
                (k, rel_err(named[k].grad, ref.grad))
        return
    tol_y, tol = FRO[mode]
    assert fro(yg, yr.view(yg.shape)) <= tol_y
    assert fro(xg.grad, xr.grad) <= tol
    for k, ref in state.items():
        assert fro(named[k].grad, ref.grad) <= tol, k


# ------------------------------------------------------------------ DCNv2 with the mixture, along the golden trajectory
@pytest.mark.parametrize("mode", ["fp32", "tf32x3"])
def test_dcnv2_mix_matches_reference_trajectory(mode, mode_of):
    """zoo.DCNv2's embedding, parallel MLP and fc around a mirror CrossNetMix, with torch's clip + Adam
    (the reference's train_step), against model_DCNv2_mix.npz at test_gpu_parity.py's model bars."""
    from fuxictr_b200 import layers, zoo
    from fuxictr_b200.schema import FeatureMap
    g = Golden("model_DCNv2_mix")
    kw = dict(g.meta["kwargs"])
    mix = {k: kw.pop(k) for k in ("use_low_rank_mixture", "low_rank", "num_experts")}
    fm = FeatureMap.from_specs(g.meta["specs"], labels=g.meta["labels"], embedding_dim=kw["embedding_dim"])
    model = zoo.DCNv2(fm, gpu=-1, **kw)
    model.crossnet = layers.CrossNetMix(fm.sum_emb_out_dim(), kw["num_cross_layers"], mix["low_rank"], mix["num_experts"])
    assert list(model.state_dict().keys()) == list(g["w"].keys())
    model.load_state_dict(g["w"])
    model.device = torch.device("cuda:0")
    model.model_to_device()
    model.compile("adam", "binary_crossentropy", 1e-3)
    model.train()
    mode_of(mode)
    B = g.meta["batch"]
    mat = g["in"]["matrix"].cuda()
    batches = [fm.batch_dict(mat[i * B:(i + 1) * B]) for i in range(3)]
    ret = model.forward(batches[0])
    assert close(ret["y_pred"], g["out"]["y_pred"], RTOL)
    loss = model.compute_loss(ret, model.get_labels(batches[0]))
    assert close(loss, g["out"]["loss"], RTOL)
    loss.backward()
    named = dict(model.named_parameters())
    for k, ref in g["g"].items():
        assert close(named[k].grad, ref, RTOL), (k, rel_err(named[k].grad, ref))
    losses = []
    for i in range(3):
        losses.append(float(model.train_step(batches[i])))
        if i == 0:
            sd = model.state_dict()
            for k, ref in g["w1"].items():
                assert close(sd[k], ref, RTOL), (k, rel_err(sd[k], ref))
    assert close(torch.tensor(losses), g["out"]["step_losses"], RTOL)
    sd = model.state_dict()
    for k, ref in g["w3"].items():
        assert close(sd[k], ref, 2e-5), (k, rel_err(sd[k], ref))


# ------------------------------------------------------------------ the unmodified reference DCNv2 under patch.enable()
def build_ref(gpu, tmp):
    R = refenv.import_reference()
    params = refenv.load_params("DCNv2", "DCNv2_test", model_root=os.path.join(tmp, "ckpt_%d" % gpu))
    params.update(gpu=gpu, num_workers=0, verbose=0, shuffle=False, use_low_rank_mixture=True)
    R.torch_utils.seed_everything(seed=params["seed"])
    fm = refenv.load_feature_map(params)
    model = refenv.load_model_class("DCNv2")(fm, **params)
    return R, params, fm, model


@pytest.mark.skipif(not refenv.available(), reason=refenv.why_unavailable())
@pytest.mark.parametrize("mode", ["fp32", "tf32x3"])
def test_reference_dcnv2_mix_runs_on_the_kernels(mode, mode_of):
    """test_reference_boundary.py's recipe and bars for the reference DCNv2_test YAML with
    use_low_rank_mixture=True (d 14*40 = 560, low_rank 32, 4 experts)."""
    from fuxictr_b200 import patch
    logging.disable(logging.INFO)
    mode_of(mode)
    with tempfile.TemporaryDirectory() as tmp:
        R, params, fm, cpu_model = build_ref(-1, tmp)
        _, _, _, gpu_model = build_ref(0, tmp)
        assert type(cpu_model.crossnet).__name__ == "CrossNetMix"
        assert cpu_model.crossnet.U_list[0].shape == (4, 560, 32)
        with torch.no_grad():
            for mod in cpu_model.modules():
                if isinstance(mod, torch.nn.Embedding):
                    mod.weight[1:].normal_(0, 0.05)
        gpu_model.load_state_dict(cpu_model.state_dict())
        keys = list(cpu_model.state_dict().keys())
        gen, _ = R.dataloaders.RankDataLoader(fm, stage="train", **params).make_iterator()
        batches = []
        for b in gen:
            batches.append(b)
            if len(batches) == 3:
                break
        for m in (cpu_model, gpu_model):
            m._max_gradient_norm = 10.0
        patch.enable()
        try:
            before = patch.call_counts().get("CrossNetMix", 0)
            cpu_model.eval(), gpu_model.eval()
            with torch.no_grad():
                y_ref = cpu_model.forward(batches[0])["y_pred"]
                y_gpu = gpu_model.forward(batches[0])["y_pred"]
            assert y_gpu.is_cuda
            assert rel_err(y_gpu, y_ref) <= 1e-5, "forward differs from the reference"
            assert patch.call_counts().get("CrossNetMix", 0) > before, "CrossNetMix did not take the kernel path"
            cpu_model.train(), gpu_model.train()
            w0 = {k: v.detach().clone() for k, v in cpu_model.state_dict().items()}
            for step, b in enumerate(batches):
                l_ref = cpu_model.train_step(b)
                l_gpu = gpu_model.train_step(b)
                assert abs(float(l_gpu) - float(l_ref)) <= 1e-5 * abs(float(l_ref)) + 1e-7
                if step == 0:
                    g_ref = {k: p.grad for k, p in cpu_model.named_parameters() if p.grad is not None}
                    g_gpu = {k: p.grad for k, p in gpu_model.named_parameters() if p.grad is not None}
                    assert set(g_ref) == set(g_gpu)
                    scale = max(float(g.abs().max()) for g in g_ref.values())
                    for k in g_ref:
                        err = float((g_gpu[k].cpu() - g_ref[k]).abs().max())
                        assert err <= 1e-5 * max(float(g_ref[k].abs().max()), 1e-3 * scale), "grad %s: %g" % (k, err)
            sd_ref, sd_gpu = cpu_model.state_dict(), gpu_model.state_dict()
            moved = 3 * params["learning_rate"]
            for k in keys:
                err = float((sd_gpu[k].cpu() - sd_ref[k]).abs().max())
                assert err <= 1e-3 * moved + 1e-5 * float((sd_ref[k] - w0[k]).abs().max()), \
                    "%s after 3 train_steps: %g" % (k, err)
        finally:
            patch.disable()
            logging.disable(logging.NOTSET)

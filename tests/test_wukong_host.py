"""WuKong without a GPU: the float64 restatement against the reference's goldens, construction against the reference's
digests (names, children, registration order, initial draws), the refusals, the C-ABI range checks, the launch
sequence of a layer per matmul mode, and the new kernels' register use."""
import ctypes
import hashlib
import json
import os
import subprocess
import sys

import pytest
import torch

from conftest import Golden, GOLDEN, ROOT, close, rel_err

sys.path.insert(0, ROOT)
from oracle import fuxictr_oracle as O  # noqa: E402
import wukong_oracle as WO  # noqa: E402
from fuxictr_b200 import _lib, functional as F2, layers, zoo  # noqa: E402
from fuxictr_b200.schema import FeatureMap  # noqa: E402


def _fm(n=3, dim=4):
    specs = [("C%d" % i, {"type": "categorical", "source": "", "padding_idx": 0, "vocab_size": 9 + i})
             for i in range(n)]
    return FeatureMap.from_specs(specs, embedding_dim=dim)


# ------------------------------------------------------------------ oracle vs the reference's goldens
LAYER_CASES = ["proj", "identity", "noln"]


@pytest.mark.parametrize("c", LAYER_CASES)
def test_oracle_layer_matches_reference_golden(c):
    g = Golden("next_WuKongLayer")
    _, nf, lcb, fmb, D, k, units, ln = [q for q in g.meta["cases"] if q[0] == c][0]
    st = {key: v.clone().double().requires_grad_(True) for key, v in g["w_" + c].items()}
    x = g["in"]["x_" + c].clone().double().requires_grad_(True)
    out = WO.wukong_layer(x, st, "", len(units), ln)
    assert close(out, g["out"]["y_" + c], 2e-6), rel_err(out, g["out"]["y_" + c])
    (out * g["in"]["gout_" + c].double()).sum().backward()
    assert close(x.grad, g["gin"]["x_" + c], 2e-6), rel_err(x.grad, g["gin"]["x_" + c])
    want = g["g_" + c]
    assert set(want) == set(st)
    scale = max(float(v.abs().max()) for v in want.values())
    for key, ref in want.items():
        assert close(st[key].grad, ref, 5e-6, atol=5e-6 * scale), (key, rel_err(st[key].grad, ref))


MODEL_CASES = ["bn", "nobn", "noln"]


def oracle_pred_fn(g):
    kw, specs = g.meta["kwargs"], g.specs()
    return lambda s, X: torch.sigmoid(WO.wukong_logit(
        specs, s, X, kw["num_wukong_layers"], len(kw["fmb_mlp_units"]), len(kw["mlp_hidden_units"]),
        kw["mlp_batch_norm"], kw.get("layer_norm", True)))


def noise_only(g, key):
    """A parameter whose exact gradient is zero, so that what any implementation computes for it is rounding noise
    (which Adam then turns into steps of lr): residual_proj.bias before the output LayerNorm(D), which removes a constant
    per field, and the last LayerNorm's bias before fc's BatchNorm1d, which removes a constant per column.  Found from
    the reference's gradients: below 1e-6 of the largest.  The trajectories compare the other parameters (not BatchNorm's buffers)."""
    scale = max(float(v.abs().max()) for v in g["g"].values())
    return key not in g["g"] or float(g["g"][key].abs().max()) <= 1e-6 * scale


@pytest.mark.parametrize("name", MODEL_CASES)
def test_oracle_models_match_reference_trajectory(name):
    """test_oracle_golden.py's recipe: forward, loss and every gradient on batch 0, then three clip + Adam steps."""
    g = Golden("model_WuKong_" + name)
    fm = FeatureMap.from_specs(g.meta["specs"], labels=g.meta["labels"])
    B = g.meta["batch"]
    mat = g["in"]["matrix"]
    batches = [fm.batch_dict(mat[i * B:(i + 1) * B]) for i in range(3)]
    tr = O.OracleTrainer(dict(g["w"]), oracle_pred_fn(g), g.specs(), g.meta["labels"])
    y_pred, y = tr.forward(batches[0])
    assert rel_err(y_pred, g["out"]["y_pred"]) <= 1e-6
    loss = O.bce_mean(y_pred, y)
    assert rel_err(loss, g["out"]["loss"]) <= 1e-6
    loss.backward()
    for key, ref in g["g"].items():
        if noise_only(g, key):
            assert float(tr.state[key].grad.abs().max()) < 1e-6 and float(ref.abs().max()) < 1e-6
        else:
            assert rel_err(tr.state[key].grad, ref) <= 2e-5, key
    losses = []
    for i in range(3):
        losses.append(float(tr.train_step(batches[i])))
        if i == 0:
            for key, ref in g["w1"].items():
                assert noise_only(g, key) or rel_err(tr.state[key], ref) <= 2e-5, key
    assert rel_err(torch.tensor(losses), g["out"]["step_losses"]) <= 2e-6
    for key, ref in g["w3"].items():
        assert noise_only(g, key) or rel_err(tr.state[key], ref) <= 5e-5, key


def _digests(module):
    return [[k, str(v.dtype), list(v.shape), hashlib.sha256(v.detach().contiguous().numpy().tobytes()).hexdigest()]
            for k, v in module.state_dict().items()]


def _init_cases():
    with open(os.path.join(GOLDEN, "wukong_init.json")) as fd:
        return json.load(fd)


def test_mirror_state_dict_matches_reference_construction():
    """Keys, registration order, shapes and initial values (same RNG draws) of the reference's WuKongLayer: projection
    residual, identity residual, layer_norm=False, empty fmb_mlp_units, dropout."""
    cases = _init_cases()["layers"]
    assert len(cases) == 5
    for name, case in cases.items():
        nf, lcb, fmb, D, k, units, p, ln = case["args"]
        torch.manual_seed(case["seed"])
        m = layers.WuKongLayer(nf, lcb, fmb, D, k, units, "relu", p, ln)
        assert _digests(m) == case["state_dict"], name


@pytest.mark.parametrize("name", MODEL_CASES)
def test_zoo_state_dict_matches_reference_construction(name):
    """The whole model after construction (embedding, layer stack, fc, then reset_parameters)."""
    case = _init_cases()["models"][name]
    torch.manual_seed(case["seed"])
    fm = FeatureMap.from_specs(case["specs"], labels=case["labels"], embedding_dim=case["kwargs"]["embedding_dim"])
    model = zoo.WuKong(fm, gpu=-1, **case["kwargs"])
    assert _digests(model) == case["state_dict"]


def test_zoo_module_order_and_state_dict_keys():
    model = zoo.WuKong(_fm(), gpu=-1, embedding_dim=4, num_wukong_layers=2, lcb_features=2, fmb_features=3,
                       fmb_mlp_units=[8], fmp_rank_k=2, mlp_hidden_units=[8], unknown_keyword=3)
    assert [n for n, _ in model.named_children()][-3:] == ["embedding_layer", "wukong_stack", "fc"]
    keys = list(model.state_dict().keys())
    layer0 = [k for k in keys if k.startswith("wukong_stack.0.")]
    assert layer0 == ["wukong_stack.0." + k for k in (
        "fmb.proj_Y", "fmb.layer_norm.weight", "fmb.layer_norm.bias", "fmb.mlp.mlp.0.weight", "fmb.mlp.mlp.0.bias",
        "fmb.mlp.mlp.2.weight", "fmb.mlp.mlp.2.bias", "lcb.linear.weight", "layer_norm.weight", "layer_norm.bias",
        "residual_proj.weight", "residual_proj.bias")]
    assert "wukong_stack.1.residual_proj.weight" not in keys and keys[-1].startswith("fc.mlp.")


# ------------------------------------------------------------------ refusals
def test_refusals():
    assert F2.wukong_bound(39, 80, 64, 8) is None and F2.wukong_bound(80, 80, 64, 8) is None
    assert F2.wukong_bound(32, 128, 128, 32) is None
    assert "vanilla" in F2.wukong_bound(39, 80, 64, None)
    assert "input fields" in F2.wukong_bound(129, 80, 64, 1)
    assert "lcb_features + fmb_features" in F2.wukong_bound(39, 129, 64, 1)
    assert "embedding_dim" in F2.wukong_bound(39, 80, 129, 8)
    assert "fmp_rank_k" in F2.wukong_bound(16, 80, 64, 33)
    assert "at most 1024" in F2.wukong_bound(80, 80, 64, 13)
    with pytest.raises(NotImplementedError, match="vanilla"):
        zoo.WuKong(_fm(), gpu=-1, embedding_dim=4, fmp_rank_k=None)
    with pytest.raises(NotImplementedError, match="vanilla"):
        layers.FactorizationMachineBlock(4, 4, 4, None)
    with pytest.raises(NotImplementedError, match="num_wukong_layers"):
        zoo.WuKong(_fm(), gpu=-1, embedding_dim=4, num_wukong_layers=0)
    with pytest.raises(NotImplementedError, match="embedding_dim"):
        zoo.WuKong(_fm(), gpu=-1, embedding_dim=256)
    with pytest.raises(NotImplementedError, match="input fields"):
        zoo.WuKong(_fm(n=130), gpu=-1, embedding_dim=4)
    with pytest.raises(NotImplementedError, match="at least 1"):
        layers.WuKongLayer(4, 0, 4, 4, 2)
    model = zoo.WuKong(_fm(), gpu=-1, embedding_dim=4, lcb_features=2, fmb_features=2, fmp_rank_k=2)
    assert zoo.WuKong._routes_sharded_front is True
    with pytest.raises(NotImplementedError, match="lazy"):
        model.use_fused_optimizer(lazy_tables=True)
    with pytest.raises(ValueError, match="want_fm=False"):
        model.enable_sharding(None, 16, 4, want_fm=True)


# ------------------------------------------------------------------ C-ABI range checks (no CUDA call is reached)
def test_kernel_range_is_checked_before_any_cuda_call():
    import __graft_entry__
    __graft_entry__.build()
    L = _lib.load()
    p = ctypes.c_void_p(4096)
    z = ctypes.c_void_p(0)

    def fm_fwd(B=8, F=39, D=64, k=8, layout=0, x=p, aux=z, dt=0, ld=0, xp=z):
        return L.b2_wukong_fm_fwd(x, layout, B, F, D, k, p, p, p, 1e-5, p, aux, dt, ld, xp, z, 0, p, p, None)

    def fm_bwd(B=8, F=39, D=64, k=8, layout=1, gxp=z):
        return L.b2_wukong_fm_bwd(p, layout, B, F, D, k, p, p, p, p, p, gxp, p, 0, p, p, p, None)

    def out_fwd(B=8, F=39, D=64, lcb=40, fmb=40, res=2, aux=z, dt=0, ld=0, layout=1, xp=z):
        return L.b2_wukong_out_fwd(p, p, xp, B, F, D, lcb, fmb, res, z, z, 1e-5, layout, p, aux, dt, ld, z, z, None)

    def out_bwd(B=8, F=39, D=64, lcb=40, fmb=40, res=2, gxp=z, dbias=p, aux=z, dt=0, ld=0):
        return L.b2_wukong_out_bwd(p, p, p, B, F, D, lcb, fmb, res, z, z, z, 1, p, p, p, aux, dt, ld, gxp, 0, dbias,
                                   z, z, None)
    assert fm_fwd(F=129) == -1 and b"fields" in L.b2_last_error()
    assert fm_fwd(F=0) == -1 and b"fields" in L.b2_last_error()
    assert fm_fwd(D=129) == -1 and b"embedding_dim" in L.b2_last_error()
    assert fm_fwd(k=33) == -1 and b"rank" in L.b2_last_error()
    assert fm_fwd(F=80, k=13) == -1 and b"fields * rank" in L.b2_last_error()
    assert fm_fwd(B=-1) == -1 and b"negative" in L.b2_last_error()
    assert fm_fwd(B=1 << 20, D=128, F=128) == -1 and b"2^31" in L.b2_last_error()
    assert fm_fwd(B=1 << 50) == -1 and b"2^31" in L.b2_last_error()
    assert fm_fwd(layout=2) == -1 and b"layout" in L.b2_last_error()
    assert fm_fwd(layout=1, xp=p) == -1 and b"X'_0" in L.b2_last_error()
    assert fm_fwd(x=z) == -1 and b"NULL" in L.b2_last_error()
    assert fm_fwd(aux=p, dt=_lib.B2_BF16, ld=311) == -1 and b"ld_aux" in L.b2_last_error()
    assert fm_fwd(aux=p, dt=7, ld=312) == -1 and b"aux_dtype" in L.b2_last_error()
    assert fm_bwd(gxp=p) == -1 and b"gxp" in L.b2_last_error()
    assert out_fwd(lcb=0) == -1 and b"lcb" in L.b2_last_error()
    assert out_fwd(lcb=64, fmb=65) == -1 and b"lcb" in L.b2_last_error()
    assert out_fwd(res=1) == -1 and b"identity residual" in L.b2_last_error()
    assert out_fwd(res=1, F=80) == -1 and b"X'" in L.b2_last_error()
    assert out_fwd(res=3) == -1 and b"res_mode" in L.b2_last_error()
    assert out_fwd(layout=2) == -1 and b"out_layout" in L.b2_last_error()
    assert out_fwd(aux=p, dt=_lib.B2_F32, ld=79) == -1 and b"ld_aux" in L.b2_last_error()
    assert out_fwd(B=1 << 50) == -1 and b"2^31" in L.b2_last_error()
    assert out_bwd(res=1, F=80) == -1 and b"gxp" in L.b2_last_error()
    assert out_bwd(dbias=z) == -1 and b"dbias" in L.b2_last_error()
    assert out_bwd(aux=p, dt=_lib.B2_F32, ld=119) == -1 and b"ld_aux" in L.b2_last_error()   # dC is lcb + Fo wide
    assert L.b2_wukong_pack(p, p, z, 39, 40, 80, p, p, None) == -1 and b"b_res" in L.b2_last_error()
    assert L.b2_wukong_pack(p, z, z, 0, 40, 80, p, z, None) == -1
    assert L.b2_wukong_unpack(p, 39, 129, 80, p, z, None) == -1
    assert fm_fwd(B=0) == 0 and fm_bwd(B=0) == 0 and out_fwd(B=0) == 0 and out_bwd(B=0) == 0


# ------------------------------------------------------------------ launch sequence (no GPU: _lib.call recorded)
@pytest.fixture
def recorder(monkeypatch):
    calls = []

    def fake_call(name, *a):
        info = None
        if name == "b2_gemm_tc_ex":
            d = ctypes.cast(a[0], ctypes.POINTER(_lib.b2_gemm_desc)).contents
            info = dict(M=d.M, N=d.N, K=d.K, a_mn=d.a_mn_major, b_mn=d.b_mn_major, bias=bool(d.bias),
                        acc=bool(d.beta_accumulate), bf16=d.elem_dtype == _lib.B2_BF16,
                        inline=bool(d.flags & _lib.B2_GEMM_X3_INLINE))
        elif name == "b2_gemm_f32":
            info = dict(M=a[8], N=a[9], K=a[10], bias=bool(a[11].value), acc=bool(a[15]))
        elif name == "b2_wukong_fm_fwd":
            info = dict(layout=a[1], aux=bool(a[11].value), xp=bool(a[14].value), xp_aux=bool(a[15].value))
        elif name == "b2_wukong_fm_bwd":
            info = dict(layout=a[1], gxp=bool(a[11].value), acc=a[13])
        elif name == "b2_wukong_out_fwd":
            info = dict(res=a[8], layout=a[12], aux=bool(a[14].value))
        elif name == "b2_wukong_out_bwd":
            info = dict(res=a[8], layout=a[12], aux=bool(a[16].value), gxp=bool(a[19].value), acc=a[20])
        calls.append((name, info))
        return 0

    monkeypatch.setattr(_lib, "call", fake_call)
    monkeypatch.setattr(F2, "_stream", lambda: None)
    monkeypatch.setattr(F2, "_require_cuda", lambda *t: None)
    yield calls
    F2.set_matmul_precision("fp32")
    F2.set_x3_inline(True)


def run_stack(mode, B, F, D, lcb, fmb, k, units, nlayers=1, ln=True):
    F2.set_matmul_precision(mode)
    torch.manual_seed(3)
    net = [layers.WuKongLayer(F if i == 0 else lcb + fmb, lcb, fmb, D, k, units, "relu", 0.0, ln)
           for i in range(nlayers)]
    x = torch.randn(B, F, D, requires_grad=True)
    out = layers.wukong_stack(net, x)
    assert type(out.grad_fn).__name__ == "_WuKongMixBackward" and tuple(out.shape) == (B, (lcb + fmb) * D)
    out.backward(torch.randn_like(out))
    for m in net:
        for p in m.parameters():
            assert p.grad is not None and p.grad.shape == p.shape
    assert x.grad is not None and x.grad.shape == x.shape


def _wukong_calls(recorder, B, D):
    """(name, info) of the WuKong launches and the field-axis GEMMs (M or K = B D), in order."""
    out = []
    for n, i in recorder:
        if n.startswith("b2_wukong_"):
            out.append((n, i))
        elif n in ("b2_gemm_tc_ex", "b2_gemm_f32") and B * D in (i["M"], i["K"]):
            out.append(("gemm", i))
    return out


@pytest.mark.parametrize("mode", ["tf32x3", "tf32", "bf16"])
def test_default_layers_launch_sequence(recorder, mode):
    """WuKong_default's shape (F 39 -> 80, D 64, k 8): layer 0 is the FM kernel (which also writes X'_0 at pitch 40),
    the pack, one GEMM N 120 K 40 with b_res in the epilogue, the combine kernel; layer 1 (identity) has no pack.
    Backward per layer: the combine kernel, dgrad (accumulating into X''s one gradient buffer), wgrad, the unpack
    (layer 0 only), the FM kernel."""
    B, D = 512, 64
    run_stack(mode, B, 39, D, 40, 40, 8, [64, 32], nlayers=2)
    got = [n for n, _ in _wukong_calls(recorder, B, D)]
    assert got == ["b2_wukong_fm_fwd", "b2_wukong_pack", "gemm", "b2_wukong_out_fwd",
                   "b2_wukong_fm_fwd", "gemm", "b2_wukong_out_fwd",
                   "b2_wukong_out_bwd", "gemm", "gemm", "b2_wukong_fm_bwd",
                   "b2_wukong_out_bwd", "gemm", "gemm", "b2_wukong_unpack", "b2_wukong_fm_bwd"]
    calls = _wukong_calls(recorder, B, D)
    g = [i for n, i in calls if n == "gemm"]
    assert all(c.get("bf16", False) == (mode == "bf16") for c in g)
    assert (g[0]["M"], g[0]["N"], g[0]["K"], g[0]["bias"]) == (B * D, 120, 40, True)
    assert (g[1]["M"], g[1]["N"], g[1]["K"], g[1]["bias"]) == (B * D, 40, 80, False)
    # backward of layer 1 (identity: the combine kernel wrote X''s gradient first, the dgrad adds), then layer 0
    assert (g[2]["M"], g[2]["N"], g[2]["K"], g[2]["acc"], g[2]["b_mn"]) == (B * D, 80, 40, True, 1)
    assert (g[3]["M"], g[3]["N"], g[3]["K"]) == (40, 80, B * D)
    assert (g[4]["M"], g[4]["N"], g[4]["K"], g[4]["acc"]) == (B * D, 40, 120, False)
    assert (g[5]["M"], g[5]["N"], g[5]["K"]) == (120, 40, B * D)
    fm0, fm1 = [i for n, i in calls if n == "b2_wukong_fm_fwd"]
    assert fm0["layout"] == 0 and fm0["xp"] and fm1["layout"] == 1 and not fm1["xp"]
    assert fm0["xp_aux"] == (mode == "bf16") and fm0["aux"] == (mode == "bf16")
    o0, o1 = [i for n, i in calls if n == "b2_wukong_out_fwd"]
    assert (o0["res"], o0["layout"], o0["aux"]) == (2, 1, mode == "bf16")
    assert (o1["res"], o1["layout"]) == (1, 0)
    b1, b0 = [i for n, i in calls if n == "b2_wukong_out_bwd"]
    assert (b1["res"], b1["gxp"], b1["acc"]) == (1, True, 0) and (b0["res"], b0["gxp"]) == (2, False)
    f1, f0 = [i for n, i in calls if n == "b2_wukong_fm_bwd"]
    assert (f1["layout"], f1["acc"]) == (1, 1) and (f0["layout"], f0["gxp"], f0["acc"]) == (0, True, 0)


@pytest.mark.parametrize("mode", ["fp32", "tf32x3", "tf32", "bf16"])
def test_simt_gemm_at_small_fields(recorder, mode):
    """WuKong_test's lcb 8: the stacked weight (8 + 16, 40) and lcb-only (8, 16) are not tensor-core shapes; the SIMT
    GEMM runs in every mode, the same row kernels around it.  F 5 pads to 8: the pack runs without a projection too."""
    B, D = 33, 16
    run_stack(mode, B, 5, D, 8, 8, 8, [32, 32], nlayers=2)
    calls = _wukong_calls(recorder, B, D)
    assert all(n != "gemm" or "bias" in i and "a_mn" not in i for n, i in calls)
    names = [n for n, _ in calls]
    assert names.count("b2_wukong_pack") == 1 and names.count("b2_wukong_unpack") == 1
    g = [i for n, i in calls if n == "gemm"]
    assert (g[0]["M"], g[0]["N"], g[0]["K"]) == (B * D, 24, 8)


def test_identity_at_unaligned_fields_packs_the_padding(recorder):
    """F 6 == lcb + fmb (identity residual) pads X' to 8 fields: the pack zero-pads W_lcb, the unpack strips it."""
    B, D = 9, 4
    run_stack("fp32", B, 6, D, 3, 3, 2, [8])
    names = [n for n, _ in _wukong_calls(recorder, B, D)]
    assert names == ["b2_wukong_fm_fwd", "b2_wukong_pack", "gemm", "b2_wukong_out_fwd", "b2_wukong_out_bwd", "gemm",
                     "gemm", "b2_wukong_unpack", "b2_wukong_fm_bwd"]


# ------------------------------------------------------------------ register use
def test_new_kernels_do_not_spill(tmp_path):
    nvcc = "/usr/local/cuda/bin/nvcc"
    from fuxictr_b200 import build
    nvcc = os.environ.get("NVCC") or (nvcc if os.path.exists(nvcc) else "nvcc")
    r = subprocess.run([nvcc] + build.NVCC_FLAGS + ["-Xptxas", "-v", "-I", build.INCLUDE, "-c",
                        os.path.join(build.CSRC, "wukong.cu"), "-o", str(tmp_path / "wukong.o")],
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    log = r.stdout + r.stderr
    kernels = [line for line in log.splitlines() if "Compiling entry function" in line]
    assert len(kernels) == 8, log
    assert all("wk_" in k for k in kernels)
    spills = [line for line in log.splitlines() if "spill" in line]
    assert len(spills) == 8 and all("0 bytes spill stores, 0 bytes spill loads" in s for s in spills), log

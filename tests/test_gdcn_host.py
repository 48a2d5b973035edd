"""GDCN without a GPU: the float64 oracle against the reference's goldens (layer and both models), the mirror's and
the zoo models' construction against the reference's, the zoo models' refusals and routing flags, the C-ABI's range
checks, the launch sequence of a layer per matmul mode, and the new kernels' register use."""
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
import gdcn_oracle as GO  # noqa: E402
from fuxictr_b200 import _lib, functional as F2, layers, zoo  # noqa: E402
from fuxictr_b200.schema import FeatureMap  # noqa: E402


# ------------------------------------------------------------------ oracle vs the reference's goldens
@pytest.mark.parametrize("d", [20, 13])
def test_oracle_layer_matches_reference_golden(d):
    g = Golden("next_GateCorssLayer")
    nl = g.meta["cn_layers"]
    st = {k: v.clone().double().requires_grad_(True) for k, v in g["w_d%d" % d].items()}
    x = g["in"]["x_d%d" % d].clone().double().requires_grad_(True)
    out = GO.gate_cross_net(x, st, "", nl)
    assert close(out, g["out"]["y_d%d" % d], 2e-6), rel_err(out, g["out"]["y_d%d" % d])
    (out * g["in"]["gout_d%d" % d].double()).sum().backward()
    assert close(x.grad, g["gin"]["x_d%d" % d], 2e-6), rel_err(x.grad, g["gin"]["x_d%d" % d])
    want = g["g_d%d" % d]
    assert set(want) == set(st)
    scale = max(float(v.abs().max()) for v in want.values())
    for k, ref in want.items():
        assert close(st[k].grad, ref, 2e-6, atol=2e-6 * scale), (k, rel_err(st[k].grad, ref))


def oracle_pred_fn(name, g):
    kw, specs = g.meta["kwargs"], g.specs()
    fn = GO.gdcn_logit if name == "GDCN" else GO.gdcnp_logit
    nl = kw.get("num_cross_layers", 3)
    return lambda s, X: torch.sigmoid(fn(specs, s, X, nl, len(kw["dnn_hidden_units"])))


@pytest.mark.parametrize("name", ["GDCN", "GDCNP"])
def test_oracle_models_match_reference_trajectory(name):
    """test_oracle_golden.py's recipe: forward, loss and every gradient on batch 0, then three clip + Adam steps."""
    g = Golden("model_" + name)
    fm = FeatureMap.from_specs(g.meta["specs"], labels=g.meta["labels"])
    B = g.meta["batch"]
    mat = g["in"]["matrix"]
    batches = [fm.batch_dict(mat[i * B:(i + 1) * B]) for i in range(3)]
    tr = O.OracleTrainer(dict(g["w"]), oracle_pred_fn(name, g), g.specs(), g.meta["labels"])
    y_pred, y = tr.forward(batches[0])
    assert rel_err(y_pred, g["out"]["y_pred"]) <= 1e-6
    loss = O.bce_mean(y_pred, y)
    assert rel_err(loss, g["out"]["loss"]) <= 1e-6
    loss.backward()
    for k, ref in g["g"].items():
        assert rel_err(tr.state[k].grad, ref) <= 2e-6, k
    losses = []
    for i in range(3):
        losses.append(float(tr.train_step(batches[i])))
        if i == 0:
            for k, ref in g["w1"].items():
                assert rel_err(tr.state[k], ref) <= 2e-6, k
    assert rel_err(torch.tensor(losses), g["out"]["step_losses"]) <= 2e-6
    for k, ref in g["w3"].items():
        assert rel_err(tr.state[k], ref) <= 5e-6, k


# ------------------------------------------------------------------ construction
def _digests(module):
    return [[k, str(v.dtype), list(v.shape), hashlib.sha256(v.detach().contiguous().numpy().tobytes()).hexdigest()]
            for k, v in module.state_dict().items()]


def _init_cases():
    with open(os.path.join(GOLDEN, "gdcn_init.json")) as fd:
        return json.load(fd)


def test_mirror_state_dict_matches_reference_construction():
    """Keys, registration order, shapes and initial values (same RNG draws) of the reference's GateCorssLayer."""
    cases = _init_cases()["layers"]
    assert len(cases) >= 3
    for name, case in cases.items():
        torch.manual_seed(case["seed"])
        assert _digests(layers.GateCorssLayer(*case["args"])) == case["state_dict"], name


@pytest.mark.parametrize("name", ["GDCN", "GDCNP"])
def test_zoo_state_dict_matches_reference_construction(name):
    """The whole model after construction (embedding, dnn, cross_net[, fc], then reset_parameters)."""
    case = _init_cases()["models"][name]
    torch.manual_seed(case["seed"])
    fm = FeatureMap.from_specs(case["specs"], labels=case["labels"], embedding_dim=case["kwargs"]["embedding_dim"])
    model = getattr(zoo, name)(fm, gpu=-1, **case["kwargs"])
    assert _digests(model) == case["state_dict"]


def test_crossing_layers_is_ignored_as_in_the_reference():
    """The GDCN_test YAML's `crossing_layers` is no constructor argument: num_cross_layers (default 3) decides."""
    g = Golden("model_GDCN")
    assert "crossing_layers" in g.meta["kwargs"] and "num_cross_layers" not in g.meta["kwargs"]
    fm = FeatureMap.from_specs(g.meta["specs"], labels=g.meta["labels"], embedding_dim=g.meta["kwargs"]["embedding_dim"])
    model = zoo.GDCN(fm, gpu=-1, **g.meta["kwargs"])
    assert model.cross_net.cn_layers == 3
    assert list(model.state_dict().keys()) == list(g["w"].keys())
    gp = Golden("model_GDCNP")
    model = zoo.GDCNP(fm, gpu=-1, crossing_layers=7, **gp.meta["kwargs"])
    assert model.cross_net.cn_layers == gp.meta["kwargs"]["num_cross_layers"]
    assert list(model.state_dict().keys()) == list(gp["w"].keys())


@pytest.mark.parametrize("name", ["GDCN", "GDCNP"])
def test_empty_dnn_is_refused_at_construction(name):
    fm = FeatureMap.from_specs([("C0", {"type": "categorical", "source": "", "padding_idx": 0, "vocab_size": 9})],
                               embedding_dim=4)
    with pytest.raises(ValueError, match="dnn_hidden_units"):
        getattr(zoo, name)(fm, gpu=-1, embedding_dim=4)


@pytest.mark.parametrize("name", ["GDCN", "GDCNP"])
def test_sharded_front_routing_and_lazy_tables_refusal(name):
    cls = getattr(zoo, name)
    assert cls._routes_sharded_front is True
    assert not getattr(cls, "_replays_lazy_tables", False)
    fm = FeatureMap.from_specs([("C0", {"type": "categorical", "source": "", "padding_idx": 0, "vocab_size": 9})],
                               embedding_dim=4)
    model = cls(fm, gpu=-1, embedding_dim=4, dnn_hidden_units=[8])
    with pytest.raises(NotImplementedError, match="lazy"):
        model.use_fused_optimizer(lazy_tables=True)


# ------------------------------------------------------------------ C-ABI range checks (no CUDA call is reached)
def test_kernel_range_is_checked_before_any_cuda_call():
    import __graft_entry__
    __graft_entry__.build()
    L = _lib.load()
    p = ctypes.c_void_p(4096)
    assert L.b2_gdcn_fwd(p, p, p, p, 8, 0, p, None, 0, 0, None) == -1 and b"d = 0" in L.b2_last_error()
    assert L.b2_gdcn_fwd(None, p, p, p, 8, 16, p, None, 0, 0, None) == -1 and b"NULL" in L.b2_last_error()
    assert L.b2_gdcn_fwd(p, p, p, p, 1 << 26, 16, p, None, 0, 0, None) == -1 and b"2^31" in L.b2_last_error()
    assert L.b2_gdcn_fwd(p, p, p, p, 8, 16, p, p, _lib.B2_BF16, 8, None) == -1 and b"ld_aux" in L.b2_last_error()
    assert L.b2_gdcn_fwd(p, p, p, p, 8, 16, p, p, 7, 16, None) == -1 and b"aux_dtype" in L.b2_last_error()
    assert L.b2_gdcn_fwd(p, p, p, p, -1, 16, p, None, 0, 0, None) == -1 and b"negative" in L.b2_last_error()
    assert L.b2_gdcn_bwd(p, p, p, p, 8, 16, p, p, _lib.B2_F32, 31, p, p, None) == -1 \
        and b"ld_aux" in L.b2_last_error()                                  # dP's row is 2d wide
    assert L.b2_gdcn_bwd(p, p, p, p, 8, 16, p, None, 0, 0, p, None, None) == -1 and b"NULL" in L.b2_last_error()
    assert L.b2_gdcn_bwd(p, p, p, p, 1 << 30, 1, p, None, 0, 0, p, p, None) == -1
    assert L.b2_gdcn_pack(p, p, 0, p, None) == -1 and L.b2_gdcn_pack(p, None, 4, p, None) == -1
    assert L.b2_gdcn_unpack(p, -3, p, p, None) == -1 and L.b2_gdcn_unpack(p, 4, None, p, None) == -1
    assert L.b2_gdcn_fwd(p, p, p, p, 0, 16, p, None, 0, 0, None) == 0            # empty batch: nothing to launch
    assert L.b2_gdcn_bwd(p, p, p, p, 0, 7, p, None, 0, 0, p, p, None) == 0


# ------------------------------------------------------------------ launch sequence (no GPU: _lib.call recorded)
@pytest.fixture
def recorder(monkeypatch):
    calls = []

    def fake_call(name, *a):
        info = None
        if name == "b2_gemm_tc_ex":
            d = ctypes.cast(a[0], ctypes.POINTER(_lib.b2_gemm_desc)).contents
            info = dict(M=d.M, N=d.N, K=d.K, a_mn=d.a_mn_major, b_mn=d.b_mn_major, bias=bool(d.bias), mul=bool(d.mul),
                        add=bool(d.add), c_pre=bool(d.c_pre), bf16=d.elem_dtype == _lib.B2_BF16,
                        aux=bool(d.a_small) and bool(d.b_small), inline=bool(d.flags & _lib.B2_GEMM_X3_INLINE))
        elif name == "b2_gemm_f32":
            info = dict(M=a[8], N=a[9], K=a[10], bias=bool(a[11].value), add=bool(a[14].value))
        elif name in ("b2_gdcn_fwd", "b2_gdcn_bwd"):
            info = dict(aux=bool(a[7].value), dtype=a[8], ld=a[9])
        calls.append((name, info))
        return 0

    monkeypatch.setattr(_lib, "call", fake_call)
    monkeypatch.setattr(F2, "_stream", lambda: None)
    monkeypatch.setattr(F2, "_require_cuda", lambda *t: None)
    yield calls
    F2.set_matmul_precision("fp32")
    F2.set_x3_inline(True)


def run_net(mode, B, d, nl=1, inline=True):
    F2.set_x3_inline(inline)
    F2.set_matmul_precision(mode)
    torch.manual_seed(3)
    net = layers.GateCorssLayer(d, nl)
    x = torch.randn(B, d, requires_grad=True)
    out = net(x)
    assert type(out.grad_fn).__name__ == "_GatedCrossLayerBackward"
    out.backward(torch.randn_like(out))
    for p in net.parameters():
        assert p.grad is not None and p.grad.shape == p.shape
    assert x.grad is not None


FWD = ["b2_gdcn_pack", "b2_gemm_tc_ex", "b2_gdcn_fwd"]
BWD = ["b2_gdcn_bwd", "b2_gemm_tc_ex", "b2_gemm_tc_ex", "b2_gdcn_unpack"]


@pytest.mark.parametrize("mode", ["tf32x3", "tf32", "bf16"])
def test_layer_is_three_launches_forward_and_four_backward(recorder, mode):
    """B 8192, d 624: pack, P = x_i Wp^T, the row kernel; backward the row kernel, dx_i = g + dP Wp (K = 2d) and
    dWp = dP^T x_i, then the unpack into W and Wg.  bf16 adds only the bf16 copies of x_i and Wp (the row kernels
    write those of x_next and dP themselves)."""
    B, d = 8192, 624
    run_net(mode, B, d)
    names = [n for n, _ in recorder if n != "b2_to_bf16"]
    assert names == FWD + BWD
    assert [n for n, _ in recorder].count("b2_to_bf16") == (2 if mode == "bf16" else 0)
    p, dx, dw = [i for n, i in recorder if n == "b2_gemm_tc_ex"]
    assert all(g["bf16"] == (mode == "bf16") and g["inline"] == (mode == "tf32x3") for g in (p, dx, dw))
    assert (p["M"], p["N"], p["K"], p["a_mn"], p["b_mn"]) == (B, 2 * d, d, 0, 0)
    assert not (p["bias"] or p["mul"] or p["add"] or p["c_pre"])
    assert (dx["M"], dx["N"], dx["K"], dx["a_mn"], dx["b_mn"], dx["add"]) == (B, d, 2 * d, 0, 1, True)
    assert (dw["M"], dw["N"], dw["K"], dw["a_mn"], dw["b_mn"], dw["add"]) == (2 * d, d, B, 1, 1, False)
    fwd, bwd = [i for n, i in recorder if n in ("b2_gdcn_fwd", "b2_gdcn_bwd")]
    assert fwd["aux"] == bwd["aux"] == (mode == "bf16")
    if mode == "bf16":
        assert fwd["dtype"] == bwd["dtype"] == _lib.B2_BF16 and fwd["ld"] == d and bwd["ld"] == 2 * d


def test_next_layer_reads_the_operand_copy_the_row_kernel_wrote(recorder):
    """bf16, 3 layers: one bf16 copy of x_0 and one of each layer's Wp; x_1 and x_2 come from b2_gdcn_fwd."""
    run_net("bf16", 64, 32, nl=3)
    names = [n for n, _ in recorder]
    assert names.count("b2_to_bf16") == 1 + 3
    assert names[:4] == ["b2_gdcn_pack", "b2_to_bf16", "b2_to_bf16", "b2_gemm_tc_ex"]
    assert names[5:9] == ["b2_gdcn_pack", "b2_to_bf16", "b2_gemm_tc_ex", "b2_gdcn_fwd"]


def test_x3_aux_layout_adds_only_the_input_and_weight_splits(recorder):
    run_net("tf32x3", 512, 624, inline=False)
    names = [n for n, _ in recorder]
    assert names.count("b2_split_tf32") == 2            # x_i, Wp; x_next and dP come with their small parts
    g = [i for n, i in recorder if n == "b2_gemm_tc_ex"]
    assert len(g) == 3 and all(d["aux"] and not d["inline"] for d in g)


@pytest.mark.parametrize("mode,d", [("fp32", 624), ("tf32x3", 13), ("tf32", 30), ("bf16", 12), ("tf32x3", 1)])
def test_simt_gemm_where_the_tensor_cores_cannot_go(recorder, mode, d):
    """fp32 mode, d % 4 != 0 or d under 16: the SIMT GEMM, with the same row kernels."""
    B = 37
    run_net(mode, B, d)
    names = [n for n, _ in recorder]
    assert names == [n.replace("gemm_tc_ex", "gemm_f32") for n in FWD + BWD]
    p, dx, dw = [i for n, i in recorder if n == "b2_gemm_f32"]
    assert (p["M"], p["N"], p["K"], p["bias"], p["add"]) == (B, 2 * d, d, False, False)
    assert (dx["M"], dx["N"], dx["K"], dx["add"]) == (B, d, 2 * d, True)
    assert (dw["M"], dw["N"], dw["K"]) == (2 * d, d, B)
    assert all(not i["aux"] for n, i in recorder if n in ("b2_gdcn_fwd", "b2_gdcn_bwd"))


# ------------------------------------------------------------------ register use
def test_new_kernels_do_not_spill(tmp_path):
    nvcc = "/usr/local/cuda/bin/nvcc"
    from fuxictr_b200 import build
    nvcc = os.environ.get("NVCC") or (nvcc if os.path.exists(nvcc) else "nvcc")
    r = subprocess.run([nvcc] + build.NVCC_FLAGS + ["-Xptxas", "-v", "-I", build.INCLUDE, "-c",
                        os.path.join(build.CSRC, "gdcn.cu"), "-o", str(tmp_path / "gdcn.o")],
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    log = r.stdout + r.stderr
    kernels = [line for line in log.splitlines() if "Compiling entry function" in line]
    assert len(kernels) == 6, log
    assert all("gdcn_" in k for k in kernels)
    spills = [line for line in log.splitlines() if "spill" in line]
    assert len(spills) == 6 and all("0 bytes spill stores, 0 bytes spill loads" in s for s in spills), log

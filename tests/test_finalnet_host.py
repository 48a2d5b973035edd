"""FinalNet without a GPU: the float64 restatement against the reference's goldens, construction against the
reference's digests (names, children, registration order, initial draws, the dropout index quirk), the refusals, the
C-ABI range and NULL checks, the launch sequence of a block per matmul mode, and the new kernels' register use."""
import ctypes
import hashlib
import json
import os
import subprocess
import sys

import pytest
import torch

from conftest import Golden, GOLDEN, ROOT, rel_err

sys.path.insert(0, ROOT)
from oracle import fuxictr_oracle as O  # noqa: E402
import finalnet_oracle as FO  # noqa: E402
from fuxictr_b200 import _lib, functional as F2, layers, zoo  # noqa: E402
from fuxictr_b200.schema import FeatureMap  # noqa: E402


def _fm(n=3, dim=4):
    specs = [("C%d" % i, {"type": "categorical", "source": "", "padding_idx": 0, "vocab_size": 9 + i})
             for i in range(n)]
    return FeatureMap.from_specs(specs, embedding_dim=dim)


# ------------------------------------------------------------------ oracle vs the reference's goldens
BLOCK_CASES = ["concat_bn_train", "sum_bn_train", "concat_nobn", "sum_nobn", "concat_bn_eval"]
MODEL_CASES = ["2B", "1B_sum", "nobn"]


@pytest.mark.parametrize("c", BLOCK_CASES)
def test_oracle_block_matches_reference_golden(c):
    g = Golden("next_FinalBlock")
    _, din, units, acts, bn, res, training = [q for q in g.meta["cases"] if q[0] == c][0]
    state = {k: v.double().requires_grad_(v.is_floating_point() and "running" not in k)
             for k, v in g["w_" + c].items()}
    x = g["in"]["x_" + c].double().requires_grad_(True)
    y = FO.final_block(x, state, "", len(units), res, acts, bn, training)
    assert rel_err(y, g["out"]["y_" + c]) <= 1e-6
    y.backward(g["in"]["gout_" + c].double())
    assert rel_err(x.grad, g["gin"]["x_" + c]) <= 1e-5
    for key, ref in g["g_" + c].items():
        assert rel_err(state[key].grad, ref) <= 1e-5, key


@pytest.mark.parametrize("c", ["f5_d4", "f7_d3"])
def test_oracle_gating_matches_reference_golden(c):
    g = Golden("next_FeatureGating")
    state = {k: v.double().requires_grad_(True) for k, v in g["w_" + c].items()}
    x = g["in"]["x_" + c].double().requires_grad_(True)
    y = FO.feature_gating(x, state, "")
    assert rel_err(y, g["out"]["y_" + c]) <= 1e-6
    y.backward(g["in"]["gout_" + c].double())
    assert rel_err(x.grad, g["gin"]["x_" + c]) <= 1e-5
    for key, ref in g["g_" + c].items():
        assert rel_err(state[key].grad, ref) <= 1e-5, key


@pytest.mark.parametrize("name", MODEL_CASES)
def test_oracle_model_matches_reference_golden(name):
    """y_pred, the add_loss loss and every gradient on batch 0 of the reference's trajectories."""
    g = Golden("model_FinalNet_" + name)
    fm = FeatureMap.from_specs(g.meta["specs"], labels=g.meta["labels"])
    B = g.meta["batch"]
    batch = fm.batch_dict(g["in"]["matrix"][:B])
    tr = O.OracleTrainer(dict(g["w"]), None, g.specs(), g.meta["labels"])
    state = {k: (v.double().detach().requires_grad_(v.requires_grad) if v.is_floating_point() else v)
             for k, v in tr.state.items()}
    X, y = O.split_inputs(g.specs(), g.meta["labels"], batch)
    y1, y2 = FO.finalnet_logits(g.specs(), state, X, g.meta["kwargs"])
    loss, y_pred = FO.finalnet_loss(y1, y2, y.double())
    assert rel_err(y_pred, g["out"]["y_pred"]) <= 1e-6
    assert rel_err(loss, g["out"]["loss"]) <= 1e-6
    loss.backward()
    for key, ref in g["g"].items():
        assert rel_err(state[key].grad, ref) <= 2e-5, key


# ------------------------------------------------------------------ construction
def _digests(module):
    return [[k, str(v.dtype), list(v.shape), hashlib.sha256(v.detach().contiguous().numpy().tobytes()).hexdigest()]
            for k, v in module.state_dict().items()]


def _init_cases():
    with open(os.path.join(GOLDEN, "finalnet_init.json")) as fd:
        return json.load(fd)


def test_mirror_state_dict_matches_reference_construction():
    """Keys, registration order, shapes and initial draws of the reference's FinalBlock (both residuals, batch norm on
    and off, dropout, mixed per-layer rates) and FeatureGating; the dropout children sit where the reference puts
    them: [0, 0.5, 0] registers one Dropout(0.5) as dropout.0, which layer 0 then applies."""
    cases = _init_cases()
    assert len(cases["blocks"]) == 5 and len(cases["gates"]) == 2
    for name, case in cases["blocks"].items():
        torch.manual_seed(case["seed"])
        m = layers.FinalBlock(*case["args"])
        assert _digests(m) == case["state_dict"], name
        assert [[k, mod.p] for k, mod in m.dropout.named_children()] == case["dropout"], name
    assert cases["blocks"]["mixed_dropout"]["dropout"] == [["0", 0.5]]
    for name, case in cases["gates"].items():
        torch.manual_seed(case["seed"])
        assert _digests(layers.FeatureGating(*case["args"])) == case["state_dict"], name


@pytest.mark.parametrize("name", MODEL_CASES)
def test_zoo_state_dict_matches_reference_construction(name):
    """The whole model after construction (embedding, gating, blocks, heads, then reset_parameters)."""
    case = _init_cases()["models"][name]
    torch.manual_seed(case["seed"])
    fm = FeatureMap.from_specs(case["specs"], labels=case["labels"], embedding_dim=case["kwargs"]["embedding_dim"])
    model = zoo.FinalNet(fm, gpu=-1, **case["kwargs"])
    assert _digests(model) == case["state_dict"]
    if case["kwargs"]["use_feature_gating"]:
        assert float(model.feature_gating.linear.weight.detach().abs().max()) == 0.0
        assert bool((model.feature_gating.linear.bias == 1).all())


def test_zoo_accepts_unknown_keywords_and_keeps_module_order():
    model = zoo.FinalNet(_fm(), gpu=-1, embedding_dim=4, use_feature_gating=True, block1_hidden_units=[8],
                         block2_hidden_units=[6], unknown_keyword=3)
    assert [n for n, _ in model.named_children()] == ["output_activation", "embedding_layer", "feature_gating",
                                                      "block1", "fc1", "block2", "fc2"]


def test_refusals(monkeypatch):
    with pytest.raises(AssertionError, match="divisible by 2"):
        layers.FinalBlock(10, [7], None, 0, True, "concat")
    with pytest.raises(AssertionError, match="divisible by 2"):
        zoo.FinalNet(_fm(), gpu=-1, block1_hidden_units=[8, 5])
    for act in ("Tanh", "Softmax", "PReLU"):
        with pytest.raises((NotImplementedError, AssertionError)):
            layers.FinalBlock(10, [8], act, 0, True, "concat")
    with pytest.raises(NotImplementedError, match="hidden units"):
        layers.FinalBlock(10, [2048], None, 0, True, "concat")
    with pytest.raises(NotImplementedError, match="hidden units"):
        layers.FinalBlock(10, [1025], None, 0, True, "sum")
    fm = _fm(n=3, dim=129)
    with pytest.raises(NotImplementedError, match="embedding_dim"):
        zoo.FinalNet(fm, gpu=-1, embedding_dim=129, use_feature_gating=True)
    zoo.FinalNet(fm, gpu=-1, embedding_dim=129, use_feature_gating=False)      # no gating: no field bound
    with pytest.raises(NotImplementedError, match="gate_residual"):
        layers.FeatureGating(4, gate_residual="sum")
    with pytest.raises(AssertionError, match="block_type"):
        zoo.FinalNet(_fm(), gpu=-1, block_type="3B")
    model = zoo.FinalNet(_fm(), gpu=-1, embedding_dim=4, block1_hidden_units=[8], block2_hidden_units=[8])
    with pytest.raises(NotImplementedError, match="lazy tables"):
        model.use_fused_optimizer(lazy_tables=True)
    with pytest.raises(ValueError, match="FM term"):
        model.enable_sharding(None, 8, 4, want_fm=True)
    norm = torch.nn.BatchNorm1d(8)
    monkeypatch.setattr(F2, "_require_cuda", lambda *t: None)        # refused before any launch
    with pytest.raises(ValueError, match="more than 1 value"):
        F2.factorized_interaction(torch.zeros(1, 4), torch.zeros(8, 4), torch.zeros(8), "concat",
                                  batch_norm=(norm, True))
    assert F2.finalnet_bound(fields=39, embedding_dim=40) is None
    assert F2.finalnet_bound([64, 64, 64], fields=128, embedding_dim=64) is None
    assert "fields" in F2.finalnet_bound(fields=129, embedding_dim=4)
    assert "8192" in F2.finalnet_bound(fields=128, embedding_dim=128)


# ------------------------------------------------------------------ C-ABI range and NULL checks
def test_kernel_range_is_checked_before_any_cuda_call():
    import __graft_entry__
    __graft_entry__.build()
    L = _lib.load()
    p = ctypes.c_void_p(4096)
    z = ctypes.c_void_p(0)
    C, S = _lib.B2_FINALNET_CONCAT, _lib.B2_FINALNET_SUM

    def fwd(B=8, half=32, res=C, gamma=p, training=1, ws=p, nbt=p, act=0, h=p, aux=z, dt=0, ld=0, rm=p):
        return L.b2_finalnet_fi_fwd(h, B, half, res, gamma, gamma, 1e-5, 0.1, training, rm, rm, nbt, ws, act, z, 0,
                                    0, 0.0, p, aux, dt, ld, p, p, None)

    def bwd(B=8, half=32, res=C, gamma=p, ws=p, dg=p, g=p):
        return L.b2_finalnet_fi_bwd(p, B, half, res, gamma, gamma, p, p, 1, ws, 0, 0, z, 0, 0, 0.0, g, p, z, 0, 0,
                                    p, dg, dg, None)
    assert fwd(res=2) == -1 and b"residual" in L.b2_last_error()
    assert fwd(half=513) == -1 and b"layer width" in L.b2_last_error()
    assert fwd(half=0) == -1 and b"layer width" in L.b2_last_error()
    assert fwd(half=1025, res=S) == -1 and b"layer width" in L.b2_last_error()
    assert fwd(act=3) == -1 and b"act" in L.b2_last_error()
    assert fwd(B=-1) == -1 and b"negative" in L.b2_last_error()
    assert fwd(B=1) == -1 and b"more than 1 value" in L.b2_last_error()
    assert fwd(B=1 << 50) == -1 and b"2^31" in L.b2_last_error()
    assert fwd(h=z) == -1 and b"NULL" in L.b2_last_error()
    assert fwd(ws=z) == -1 and b"stats_ws" in L.b2_last_error()
    assert fwd(rm=z) == -1 and b"running" in L.b2_last_error()
    assert fwd(aux=p, dt=_lib.B2_BF16, ld=63) == -1 and b"ld_aux" in L.b2_last_error()
    assert fwd(aux=p, dt=7, ld=64) == -1 and b"aux_dtype" in L.b2_last_error()
    assert bwd(ws=z) == -1 and b"stats_ws" in L.b2_last_error()
    assert bwd(dg=z) == -1
    assert bwd(g=z) == -1 and b"NULL" in L.b2_last_error()
    assert bwd(half=600) == -1 and b"layer width" in L.b2_last_error()
    assert L.b2_finalnet_gate_fwd(p, 8, 129, 4, p, p, p, z, 0, 0, None) == -1 and b"fields" in L.b2_last_error()
    assert L.b2_finalnet_gate_fwd(p, 8, 4, 129, p, p, p, z, 0, 0, None) == -1 and b"dim" in L.b2_last_error()
    assert L.b2_finalnet_gate_fwd(p, 8, 128, 65, p, p, p, z, 0, 0, None) == -1 and b"fields * dim" in L.b2_last_error()
    assert L.b2_finalnet_gate_fwd(z, 8, 4, 4, p, p, p, z, 0, 0, None) == -1 and b"NULL" in L.b2_last_error()
    assert L.b2_finalnet_gate_bwd(p, 8, 4, 4, p, p, p, p, 0, p, z, None) == -1 and b"NULL" in L.b2_last_error()
    assert L.b2_finalnet_gate_bwd(p, 1 << 40, 4, 4, p, p, p, p, 0, p, p, None) == -1 and b"2^31" in L.b2_last_error()
    assert L.b2_finalnet_loss(p, z, p, 8, p, p, p, p, None) == -1 and b"NULL" in L.b2_last_error()
    assert L.b2_finalnet_loss(p, p, p, 0, p, p, p, p, None) == -1 and b"batch" in L.b2_last_error()
    assert fwd(B=0, training=0) == 0 and bwd(B=0) == 0
    assert L.b2_finalnet_gate_fwd(p, 0, 4, 4, p, p, p, z, 0, 0, None) == 0


# ------------------------------------------------------------------ launch sequence (no GPU: _lib.call recorded)
@pytest.fixture
def recorder(monkeypatch):
    calls = []

    def fake_call(name, *a):
        info = None
        if name == "b2_gemm_tc_ex":
            d = ctypes.cast(a[0], ctypes.POINTER(_lib.b2_gemm_desc)).contents
            info = dict(M=d.M, N=d.N, K=d.K, bias=bool(d.bias), acc=bool(d.beta_accumulate),
                        bf16=d.elem_dtype == _lib.B2_BF16)
        elif name == "b2_gemm_f32":
            info = dict(M=a[8], N=a[9], K=a[10], bias=bool(a[11].value), acc=bool(a[15]))
        elif name == "b2_finalnet_fi_fwd":
            info = dict(half=a[2], res=a[3], bn=bool(a[4].value), training=a[8], act=a[13], aux=bool(a[19].value))
        elif name == "b2_finalnet_fi_bwd":
            info = dict(half=a[2], training=a[8], zero_ws=a[10], aux=bool(a[18].value))
        elif name == "b2_finalnet_gate_fwd":
            info = dict(F=a[2], D=a[3], aux=bool(a[7].value))
        elif name == "b2_finalnet_gate_bwd":
            info = dict(acc=a[8])
        calls.append((name, info))
        return 0

    monkeypatch.setattr(_lib, "call", fake_call)
    monkeypatch.setattr(F2, "_stream", lambda: None)
    monkeypatch.setattr(F2, "_require_cuda", lambda *t: None)
    yield calls
    F2.set_matmul_precision("fp32")
    F2.set_x3_inline(True)


def _run_gated_block(mode, B=512, F=39, D=40, units=(64, 64, 64)):
    """FinalNet_default's block 1: gating over a shared_grad view of the embedding, then three concat layers with
    batch norm in training mode."""
    F2.set_matmul_precision(mode)
    torch.manual_seed(3)
    gate = layers.FeatureGating(F)
    block = layers.FinalBlock(2 * F * D, list(units), None, 0, True, "concat")
    e = torch.randn(B, F * D, requires_grad=True)
    flat, sink = F2.shared_grad(e)
    x = gate.run(flat, sink=sink, want_aux=F2._tc_layer_ok(block.layer[0].linear.weight))
    out = block.run(x)
    assert tuple(out.shape) == (B, units[-1])
    out.backward(torch.randn_like(out))
    for p in list(gate.parameters()) + list(block.parameters()):
        assert p.grad is not None and p.grad.shape == p.shape


@pytest.mark.parametrize("mode", ["tf32x3", "tf32", "bf16"])
def test_default_block_launch_sequence(recorder, mode):
    """Per layer forward: the GEMM (bias in the epilogue) and one row entry point (zero fill, statistics and apply);
    backward: one row entry point (statistics and apply, the forward having cleared its sums), the dgrad and the
    wgrad; the gating one row kernel each way, its backward adding into the embedding's shared gradient."""
    B, F, D = 512, 39, 40
    _run_gated_block(mode, B, F, D)
    names = [n for n, _ in recorder if n.startswith("b2_finalnet") or n in ("b2_gemm_tc_ex", "b2_gemm_f32")]
    fwd = ["b2_finalnet_gate_fwd"] + ["b2_gemm_tc_ex", "b2_finalnet_fi_fwd"] * 3
    bwd = ["b2_finalnet_fi_bwd", "b2_gemm_tc_ex", "b2_gemm_tc_ex"] * 3 + ["b2_finalnet_gate_bwd"]
    assert names == fwd + bwd
    g = [i for n, i in recorder if n == "b2_gemm_tc_ex"]
    assert all(c["bf16"] == (mode == "bf16") for c in g)
    assert (g[0]["M"], g[0]["N"], g[0]["K"], g[0]["bias"]) == (B, 64, 2 * F * D, True)
    assert (g[1]["M"], g[1]["N"], g[1]["K"], g[1]["bias"]) == (B, 64, 64, True)
    assert (g[-2]["M"], g[-2]["N"], g[-2]["K"], g[-2]["acc"]) == (B, 2 * F * D, 64, False)       # dgrad of layer 0
    assert (g[-1]["M"], g[-1]["N"], g[-1]["K"]) == (64, 2 * F * D, B)                          # its wgrad
    fi = [i for n, i in recorder if n == "b2_finalnet_fi_fwd"]
    assert all(i["half"] == 32 and i["bn"] and i["training"] == 1 for i in fi)
    assert [i["aux"] for i in fi] == [mode == "bf16", mode == "bf16", False]
    fb = [i for n, i in recorder if n == "b2_finalnet_fi_bwd"]
    assert all(i["training"] == 1 and i["zero_ws"] == 0 and i["aux"] == (mode == "bf16") for i in fb)
    gf = [i for n, i in recorder if n == "b2_finalnet_gate_fwd"][0]
    assert (gf["F"], gf["D"], gf["aux"]) == (F, D, mode == "bf16")
    assert [i for n, i in recorder if n == "b2_finalnet_gate_bwd"][0]["acc"] == 0


@pytest.mark.parametrize("mode", ["fp32", "tf32x3", "tf32", "bf16"])
def test_simt_gemm_at_small_widths(recorder, mode):
    """A 10-wide layer (not a tensor-core shape) runs on the SIMT GEMM in every mode, the same row kernels around it;
    in eval the backward clears its own sums."""
    F2.set_matmul_precision(mode)
    block = layers.FinalBlock(6, [10], "ReLU", 0, True, "sum").eval()
    x = torch.randn(33, 6, requires_grad=True)
    block.run(x).sum().backward()
    names = [n for n, _ in recorder if n.startswith("b2_finalnet") or n.startswith("b2_gemm")]
    assert names == ["b2_gemm_f32", "b2_finalnet_fi_fwd", "b2_finalnet_fi_bwd", "b2_gemm_f32", "b2_gemm_f32"]
    fb = [i for n, i in recorder if n == "b2_finalnet_fi_bwd"][0]
    assert fb["training"] == 0 and fb["zero_ws"] == 1
    g = [i for n, i in recorder if n == "b2_gemm_f32"]
    assert (g[0]["M"], g[0]["N"], g[0]["K"], g[0]["bias"]) == (33, 20, 6, True)


def test_fused_loss_is_one_launch(recorder):
    y1 = torch.randn(16, 1, requires_grad=True)
    y2 = torch.randn(16, 1, requires_grad=True)
    F2.finalnet_loss(torch.zeros(16, 1), y1, y2)
    assert [n for n, _ in recorder] == ["b2_finalnet_loss"]


# ------------------------------------------------------------------ register use
def test_new_kernels_do_not_spill(tmp_path):
    nvcc = "/usr/local/cuda/bin/nvcc"
    from fuxictr_b200 import build
    nvcc = os.environ.get("NVCC") or (nvcc if os.path.exists(nvcc) else "nvcc")
    r = subprocess.run([nvcc] + build.NVCC_FLAGS + ["-Xptxas", "-v", "-I", build.INCLUDE, "-c",
                        os.path.join(build.CSRC, "finalnet.cu"), "-o", str(tmp_path / "finalnet.o")],
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    log = r.stdout + r.stderr
    kernels = [line for line in log.splitlines() if "Compiling entry function" in line]
    assert len(kernels) == 11, log
    assert all("fn_" in k for k in kernels)
    spills = [line for line in log.splitlines() if "spill" in line]
    assert len(spills) == 11 and all("0 bytes spill stores, 0 bytes spill loads" in s for s in spills), log

"""AutoInt without a GPU: the float64 restatement against the reference's goldens, construction against the
reference's digests (names, children, registration order, initial draws), the refusals, the C-ABI range checks, the
launch sequence of a layer per matmul mode, and the new kernels' register use."""
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
import autoint_oracle as AO  # noqa: E402
from fuxictr_b200 import _lib, functional as F2, layers, zoo  # noqa: E402
from fuxictr_b200.schema import FeatureMap  # noqa: E402

_SPECS = [("C%d" % i, {"type": "categorical", "source": "", "padding_idx": 0, "vocab_size": 9 + i}) for i in range(3)]


def _fm(n=3, dim=4):
    specs = [("C%d" % i, {"type": "categorical", "source": "", "padding_idx": 0, "vocab_size": 9 + i})
             for i in range(n)]
    return FeatureMap.from_specs(specs, embedding_dim=dim)


# ------------------------------------------------------------------ oracle vs the reference's goldens
LAYER_CASES = ["wres", "h3_scale", "ln"]


@pytest.mark.parametrize("c", LAYER_CASES)
def test_oracle_layer_matches_reference_golden(c):
    g = Golden("next_MultiHeadSelfAttention")
    _, din, A, H, res, scale, ln = [k for k in g.meta["cases"] if k[0] == c][0]
    st = {k: v.clone().double().requires_grad_(True) for k, v in g["w_" + c].items()}
    x = g["in"]["x_" + c].clone().double().requires_grad_(True)
    out = AO.self_attention(x, st, "", H, res, scale, ln)
    assert close(out, g["out"]["y_" + c], 2e-6), rel_err(out, g["out"]["y_" + c])
    (out * g["in"]["gout_" + c].double()).sum().backward()
    assert close(x.grad, g["gin"]["x_" + c], 2e-6), rel_err(x.grad, g["gin"]["x_" + c])
    want = g["g_" + c]
    assert set(want) == set(st)
    scale_ = max(float(v.abs().max()) for v in want.values())
    for k, ref in want.items():
        assert close(st[k].grad, ref, 2e-6, atol=2e-6 * scale_), (k, rel_err(st[k].grad, ref))


MODEL_CASES = ["test", "wide", "nodnn"]


def oracle_pred_fn(g):
    kw, specs = g.meta["kwargs"], g.specs()
    nh = len(kw["dnn_hidden_units"]) if kw["dnn_hidden_units"] else None
    return lambda s, X: torch.sigmoid(AO.autoint_logit(
        specs, s, X, kw["attention_layers"], kw["num_heads"], nh, use_scale=kw.get("use_scale", False),
        layer_norm=kw.get("layer_norm", False), use_wide=kw.get("use_wide", False)))


@pytest.mark.parametrize("name", MODEL_CASES)
def test_oracle_models_match_reference_trajectory(name):
    """test_oracle_golden.py's recipe: forward, loss and every gradient on batch 0, then three clip + Adam steps."""
    g = Golden("model_AutoInt_" + name)
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


def _digests(module):
    return [[k, str(v.dtype), list(v.shape), hashlib.sha256(v.detach().contiguous().numpy().tobytes()).hexdigest()]
            for k, v in module.state_dict().items()]


def _init_cases():
    with open(os.path.join(GOLDEN, "autoint_init.json")) as fd:
        return json.load(fd)


def test_mirror_state_dict_matches_reference_construction():
    """Keys, registration order, shapes and initial values (same RNG draws) of the reference's MultiHeadSelfAttention:
    W_res, identity residual, use_residual=False, layer_norm, dropout."""
    cases = _init_cases()["layers"]
    assert len(cases) == 5
    for name, case in cases.items():
        din, A, H, p, res, scale, ln = case["args"]
        torch.manual_seed(case["seed"])
        m = layers.MultiHeadSelfAttention(din, attention_dim=A, num_heads=H, dropout_rate=p, use_residual=res,
                                          use_scale=scale, layer_norm=ln)
        assert _digests(m) == case["state_dict"], name


@pytest.mark.parametrize("name", MODEL_CASES)
def test_zoo_state_dict_matches_reference_construction(name):
    """The whole model after construction (embedding, LR, DNN, attention stack, fc, then reset_parameters)."""
    case = _init_cases()["models"][name]
    torch.manual_seed(case["seed"])
    fm = FeatureMap.from_specs(case["specs"], labels=case["labels"], embedding_dim=case["kwargs"]["embedding_dim"])
    model = zoo.AutoInt(fm, gpu=-1, **case["kwargs"])
    assert _digests(model) == case["state_dict"]


# ------------------------------------------------------------------ construction
def test_mirror_children_and_registration_order():
    m = layers.MultiHeadSelfAttention(4, attention_dim=8, num_heads=2, dropout_rate=0.1, layer_norm=True)
    assert [n for n, _ in m.named_children()] == ["W_q", "W_k", "W_v", "W_res", "dot_attention", "layer_norm"]
    assert list(m.state_dict().keys()) == ["W_q.weight", "W_k.weight", "W_v.weight", "W_res.weight",
                                           "layer_norm.weight", "layer_norm.bias"]
    assert m.dot_attention.dropout.p == 0.1 and m.head_dim == 4 and m.scale is None
    same = layers.MultiHeadSelfAttention(8, num_heads=2, use_scale=True)
    assert same.W_res is None and same.layer_norm is None and same.scale == 2.0
    assert layers.MultiHeadSelfAttention(4, attention_dim=8, use_residual=False).W_res is None


def test_mirror_draws_as_nn_linear_in_order():
    """The initial draws: W_q, W_k, W_v, W_res as four bias-free nn.Linear in that order."""
    torch.manual_seed(5)
    m = layers.MultiHeadSelfAttention(4, attention_dim=8, num_heads=2)
    torch.manual_seed(5)
    want = [torch.nn.Linear(4, 8, bias=False).weight for _ in range(4)]
    got = [m.W_q.weight, m.W_k.weight, m.W_v.weight, m.W_res.weight]
    assert all(torch.equal(a, b) for a, b in zip(got, want))


def test_zoo_module_order_and_state_dict_keys():
    fm = _fm()
    model = zoo.AutoInt(fm, gpu=-1, embedding_dim=4, attention_dim=8, num_heads=2, attention_layers=2,
                        dnn_hidden_units=[16], use_wide=True, layer_norm=True, unknown_keyword=3)
    assert [n for n, _ in model.named_children()][-5:] == ["embedding_layer", "lr_layer", "dnn", "self_attention",
                                                          "fc"]
    keys = list(model.state_dict().keys())
    assert "self_attention.0.W_res.weight" in keys and "self_attention.1.W_res.weight" not in keys
    assert keys[-2:] == ["fc.weight", "fc.bias"] and model.fc.in_features == 3 * 8
    assert "lr_layer.bias" not in keys
    none = zoo.AutoInt(fm, gpu=-1, embedding_dim=4, attention_dim=4, dnn_hidden_units=[])
    assert none.dnn is None and none.lr_layer is None
    bn = zoo.AutoInt(fm, gpu=-1, embedding_dim=4, dnn_hidden_units=[8], batch_norm=True)
    assert any(isinstance(m, torch.nn.BatchNorm1d) for m in bn.dnn.modules())


# ------------------------------------------------------------------ refusals
def test_heads_must_divide_attention_dim():
    with pytest.raises(AssertionError, match="not divisible"):
        layers.MultiHeadSelfAttention(4, attention_dim=10, num_heads=3)
    with pytest.raises(AssertionError, match="not divisible"):
        zoo.AutoInt(_fm(), gpu=-1, embedding_dim=4, attention_dim=10, num_heads=3)


def test_shapes_outside_the_kernel_range_are_refused():
    assert F2.autoint_bound(39, 40, 2) is None and F2.autoint_bound(64, 64, 64) is None
    assert "fields" in F2.autoint_bound(65, 40, 2)
    assert "attention_dim" in F2.autoint_bound(39, 65, 1)
    assert "divide" in F2.autoint_bound(39, 10, 4)
    with pytest.raises(NotImplementedError, match="attention_dim"):
        layers.MultiHeadSelfAttention(4, attention_dim=128, num_heads=2)
    with pytest.raises(NotImplementedError, match="fields"):
        zoo.AutoInt(_fm(n=65), gpu=-1, embedding_dim=4)


def test_lazy_tables_and_sharding_with_fm_are_refused():
    assert zoo.AutoInt._routes_sharded_front is True
    assert not getattr(zoo.AutoInt, "_replays_lazy_tables", False)
    model = zoo.AutoInt(_fm(), gpu=-1, embedding_dim=4, use_wide=True)
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

    def fwd(B=8, F=39, din=40, A=40, H=2, res=1, scale=0.0, P=p, aux=z, dt=0, ld=0):
        return L.b2_autoint_fwd(P, p, B, F, din, A, H, res, scale, z, z, 1e-5, z, 0, 0, 0.0, p, aux, dt, ld, p, p, z,
                                z, None)

    def bwd(B=8, F=39, din=40, A=40, H=2, res=2, aux=z, dt=0, ld=0, gres=z):
        return L.b2_autoint_bwd(p, p, p, p, p, p, z, z, B, F, din, A, H, res, 0.0, z, z, 0, 0, 0.0, p, aux, dt, ld,
                                gres, z, z, None)
    assert fwd(F=65) == -1 and b"fields" in L.b2_last_error()
    assert fwd(F=0) == -1 and b"fields" in L.b2_last_error()
    assert fwd(A=65, din=65) == -1 and b"attention_dim" in L.b2_last_error()
    assert fwd(H=3) == -1 and b"divide" in L.b2_last_error()
    assert fwd(din=0, res=2) == -1 and b"input_dim" in L.b2_last_error()
    assert fwd(din=8, res=1) == -1 and b"identity residual" in L.b2_last_error()
    assert fwd(B=-1) == -1 and b"negative" in L.b2_last_error()
    assert fwd(B=1 << 20, F=64, A=64, din=64) == -1 and b"2^31" in L.b2_last_error()
    assert fwd(B=1 << 50) == -1 and b"2^31" in L.b2_last_error()          # no wrap in the bound's product
    assert bwd(B=(1 << 62) // 3) == -1 and b"2^31" in L.b2_last_error()
    assert fwd(P=z) == -1 and b"NULL" in L.b2_last_error()
    assert fwd(scale=-1.0) == -1 and b"scale" in L.b2_last_error()
    assert fwd(aux=p, dt=_lib.B2_BF16, ld=39) == -1 and b"ld_aux" in L.b2_last_error()
    assert fwd(aux=p, dt=7, ld=40) == -1 and b"aux_dtype" in L.b2_last_error()
    assert bwd(aux=p, dt=_lib.B2_F32, ld=159) == -1 and b"ld_aux" in L.b2_last_error()    # dP's row is 4A wide
    assert bwd(res=1) == -1 and b"gres" in L.b2_last_error()
    assert bwd(res=3) == -1 and b"res_mode" in L.b2_last_error()
    assert L.b2_autoint_pack(p, p, p, z, 0, 8, p, None) == -1 and L.b2_autoint_pack(p, z, p, z, 4, 8, p, None) == -1
    assert L.b2_autoint_unpack(p, 4, 65, p, p, p, z, None) == -1 and L.b2_autoint_unpack(p, 4, 8, p, z, p, z, None) == -1
    assert fwd(B=0) == 0 and bwd(B=0) == 0                  # empty batch: nothing to launch


# ------------------------------------------------------------------ launch sequence (no GPU: _lib.call recorded)
@pytest.fixture
def recorder(monkeypatch):
    calls = []

    def fake_call(name, *a):
        info = None
        if name == "b2_gemm_tc_ex":
            d = ctypes.cast(a[0], ctypes.POINTER(_lib.b2_gemm_desc)).contents
            info = dict(M=d.M, N=d.N, K=d.K, a_mn=d.a_mn_major, b_mn=d.b_mn_major, add=bool(d.add),
                        bf16=d.elem_dtype == _lib.B2_BF16, inline=bool(d.flags & _lib.B2_GEMM_X3_INLINE))
        elif name == "b2_gemm_f32":
            info = dict(M=a[8], N=a[9], K=a[10], add=bool(a[14].value))
        elif name == "b2_autoint_fwd":
            info = dict(res=a[7], aux=bool(a[17].value), drop=bool(a[12].value))
        elif name == "b2_autoint_bwd":
            info = dict(res=a[13], aux=bool(a[21].value), gres=bool(a[24].value))
        calls.append((name, info))
        return 0

    monkeypatch.setattr(_lib, "call", fake_call)
    monkeypatch.setattr(F2, "_stream", lambda: None)
    monkeypatch.setattr(F2, "_require_cuda", lambda *t: None)
    yield calls
    F2.set_matmul_precision("fp32")
    F2.set_x3_inline(True)


def run_layer(mode, B, F, din, A, H, **kw):
    F2.set_matmul_precision(mode)
    torch.manual_seed(3)
    net = layers.MultiHeadSelfAttention(din, A, H, **kw)
    x = torch.randn(B, F, din, requires_grad=True)
    out = net(x)
    assert type(out.grad_fn).__name__ == "_SelfAttentionLayerBackward"
    out.backward(torch.randn_like(out))
    for p in net.parameters():
        assert p.grad is not None and p.grad.shape == p.shape
    assert x.grad is not None and x.grad.shape == x.shape


FWD = ["b2_autoint_pack", "b2_gemm_tc_ex", "b2_autoint_fwd"]
BWD = ["b2_autoint_bwd", "b2_gemm_tc_ex", "b2_gemm_tc_ex", "b2_autoint_unpack"]


@pytest.mark.parametrize("mode", ["tf32x3", "tf32", "bf16"])
@pytest.mark.parametrize("din", [40, 16])
def test_layer_is_three_launches_forward_and_four_backward(recorder, mode, din):
    """AutoInt_default's layer (B 10000, F 39, A 40, H 2): pack, P = X Wp^T, the row kernel; backward the row kernel,
    dX = dP Wp (+ dR in the epilogue for the identity residual) and dWp = dP^T X, then the unpack.  bf16 adds only the
    bf16 copies of X and Wp."""
    B, F, A = 10000, 39, 40
    run_layer(mode, B, F, din, A, 2)
    names = [n for n, _ in recorder if n != "b2_to_bf16"]
    assert names == FWD + BWD
    assert [n for n, _ in recorder].count("b2_to_bf16") == (2 if mode == "bf16" else 0)
    NP = 3 * A if din == A else 4 * A
    p, dx, dw = [i for n, i in recorder if n == "b2_gemm_tc_ex"]
    assert all(g["bf16"] == (mode == "bf16") and g["inline"] == (mode == "tf32x3") for g in (p, dx, dw))
    assert (p["M"], p["N"], p["K"], p["a_mn"], p["b_mn"], p["add"]) == (B * F, NP, din, 0, 0, False)
    assert (dx["M"], dx["N"], dx["K"], dx["a_mn"], dx["b_mn"], dx["add"]) == (B * F, din, NP, 0, 1, din == A)
    assert (dw["M"], dw["N"], dw["K"], dw["a_mn"], dw["b_mn"]) == (NP, din, B * F, 1, 1)
    fwd, bwd = [i for n, i in recorder if n in ("b2_autoint_fwd", "b2_autoint_bwd")]
    assert fwd["res"] == bwd["res"] == (1 if din == A else 2)
    assert bwd["gres"] == (din == A)
    assert bwd["aux"] == (mode == "bf16") and not fwd["aux"]


@pytest.mark.parametrize("mode", ["fp32", "tf32x3", "tf32", "bf16"])
def test_simt_gemm_where_the_tensor_cores_cannot_go(recorder, mode):
    """AutoInt_test's layer 0 (d_in 4, A 8): the SIMT GEMM in every mode, with the same row kernels."""
    B, F = 37, 39
    run_layer(mode, B, F, 4, 8, 2)
    names = [n for n, _ in recorder]
    assert names == [n.replace("gemm_tc_ex", "gemm_f32") for n in FWD + BWD]
    p, dx, dw = [i for n, i in recorder if n == "b2_gemm_f32"]
    assert (p["M"], p["N"], p["K"]) == (B * F, 32, 4)
    assert (dx["M"], dx["N"], dx["K"], dx["add"]) == (B * F, 4, 32, False)
    assert (dw["M"], dw["N"], dw["K"]) == (32, 4, B * F)


def test_stack_hands_the_operand_copy_to_the_next_layer(recorder):
    """bf16, AutoInt's 3-layer stack at the default shape: one bf16 copy of the embedding and one of each layer's Wp;
    layers 1 and 2 read the copy that the previous row kernel wrote, and one dropout snapshot serves all three."""
    F2.set_matmul_precision("bf16")
    fm = _fm(n=39, dim=40)
    model = zoo.AutoInt(fm, gpu=-1, embedding_dim=40, attention_dim=40, num_heads=2, attention_layers=3,
                        dnn_hidden_units=[], net_dropout=0.2)
    model.train()
    monkey_snap = []
    orig = F2.dropout_snapshot
    F2.dropout_snapshot = lambda dev, n: monkey_snap.append(n) or torch.zeros(2, dtype=torch.int64)
    try:
        model.attention(torch.randn(64, 39, 40))
    finally:
        F2.dropout_snapshot = orig
    assert monkey_snap == [3]
    names = [n for n, _ in recorder]
    assert names.count("b2_to_bf16") == 1 + 3
    fwd = [i for n, i in recorder if n == "b2_autoint_fwd"]
    assert [f["aux"] for f in fwd] == [True, True, False] and all(f["drop"] for f in fwd)


# ------------------------------------------------------------------ register use
def test_new_kernels_do_not_spill(tmp_path):
    nvcc = "/usr/local/cuda/bin/nvcc"
    from fuxictr_b200 import build
    nvcc = os.environ.get("NVCC") or (nvcc if os.path.exists(nvcc) else "nvcc")
    r = subprocess.run([nvcc] + build.NVCC_FLAGS + ["-Xptxas", "-v", "-I", build.INCLUDE, "-c",
                        os.path.join(build.CSRC, "autoint.cu"), "-o", str(tmp_path / "autoint.o")],
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    log = r.stdout + r.stderr
    kernels = [line for line in log.splitlines() if "Compiling entry function" in line]
    assert len(kernels) == 6, log
    assert all("ai_" in k for k in kernels)
    spills = [line for line in log.splitlines() if "spill" in line]
    assert len(spills) == 6 and all("0 bytes spill stores, 0 bytes spill loads" in s for s in spills), log

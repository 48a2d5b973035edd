"""CrossNetMix (DCN-Mix) without a GPU: the mirror's construction against the reference's, the factorised
layer that the kernels compute (packed W1 / W2, gate logits from the same GEMM, mixture folded into one
GEMM) against the oracle and the reference's golden, the row kernel's backward formulas against autograd,
the launch sequence per matmul mode, the C-ABI's range checks, and the patch's routing."""
import ctypes
import hashlib
import json
import os
import sys

import pytest
import torch

from conftest import Golden, GOLDEN, ROOT, close, rel_err

sys.path.insert(0, ROOT)
from oracle import fuxictr_oracle as O  # noqa: E402
from fuxictr_b200 import _lib, functional as F2, layers  # noqa: E402
from baseline import refenv  # noqa: E402


# ------------------------------------------------------------------ the factorised layer in torch
def pack(U, V, G):
    """W1 (N1, d), W2 (d, K2) by the layout of include/fuxictr_b200.h "CrossNetMix"."""
    E, d, r = U.shape
    R = E * r
    n1, k2 = (R + E + 3) // 4 * 4, (R + 3) // 4 * 4
    W1 = torch.cat([V.permute(0, 2, 1).reshape(R, d), G, G.new_zeros(n1 - R - E, d)], dim=0)
    W2 = torch.cat([U.permute(1, 0, 2).reshape(d, R), U.new_zeros(d, k2 - R)], dim=1)
    return W1, W2


def row_forward(P, C):
    """b2_crossmix_fwd: P (B, N1) -> A2 (B, K2)."""
    E, r, _ = C.shape
    B, R = P.shape[0], E * r
    h = torch.tanh(P[:, :R]).view(B, E, r)
    v = torch.tanh(torch.einsum("bek,ejk->bej", h, C))
    p = torch.softmax(P[:, R:R + E], dim=1)
    A2 = (p.unsqueeze(2) * v).reshape(B, R)
    k2 = (R + 3) // 4 * 4
    return torch.cat([A2, A2.new_zeros(B, k2 - R)], dim=1)


def row_backward(P, C, dA2):
    """b2_crossmix_bwd's formulas: dA1 = [dP | dlogit | 0] and dC."""
    E, r, _ = C.shape
    B, R, n1 = P.shape[0], E * r, P.shape[1]
    h = torch.tanh(P[:, :R]).view(B, E, r)
    v = torch.tanh(torch.einsum("bek,ejk->bej", h, C))
    p = torch.softmax(P[:, R:R + E], dim=1)
    g = dA2[:, :R].view(B, E, r)
    dv = p.unsqueeze(2) * g
    dp = (g * v).sum(2)
    dlogit = p * (dp - (p * dp).sum(1, keepdim=True))
    dz = dv * (1 - v * v)
    dh = torch.einsum("bej,ejk->bek", dz, C)
    dP = dh * (1 - h * h)
    dA1 = torch.cat([dP.reshape(B, R), dlogit, P.new_zeros(B, n1 - R - E)], dim=1)
    dC = torch.einsum("bej,bek->ejk", dz, h)
    return dA1, dC


def factorised(x0, U, V, C, G, bias, layer_num):
    xl = x0
    for i in range(layer_num):
        W1, W2 = pack(U[i], V[i], G)
        A2 = row_forward(xl @ W1.t(), C[i])
        xl = xl + x0 * (A2 @ W2.t() + bias[i].view(1, -1))
    return xl


def test_factorised_layer_matches_the_reference_golden():
    """The mixture folded into one GEMM (sum_e p_e = 1) and the gate logits taken from GEMM1 give the
    reference's output and every gradient within the oracle's own bar (2e-6): this pins the packed layouts
    and shows that the bias term's constant shift of dL/dp_e cancels in the softmax backward."""
    g = Golden("next_CrossNetMix")
    m = g.meta
    nl, E = m["layer_num"], m["num_experts"]
    st = {k: v.clone().double().requires_grad_(True) for k, v in g["w"].items()}
    x = g["in"]["x"].clone().double().requires_grad_(True)
    G = torch.cat([st["gating.%d.weight" % e] for e in range(E)], dim=0)
    out = factorised(x, [st["U_list.%d" % i] for i in range(nl)], [st["V_list.%d" % i] for i in range(nl)],
                     [st["C_list.%d" % i] for i in range(nl)], G, [st["bias.%d" % i] for i in range(nl)], nl)
    tol = 2e-6
    assert close(out, g["out"]["y"], tol), rel_err(out, g["out"]["y"])
    ref = O.crossnet_mix({k: v.detach() for k, v in st.items()}, "", x.detach(), nl, E)
    assert close(out, ref, 1e-12)
    (out * g["in"]["gout"].double()).sum().backward()
    assert close(x.grad, g["gin"]["x"], tol), rel_err(x.grad, g["gin"]["x"])
    scale = max(float(v.abs().max()) for v in g["g"].values())
    for k, want in g["g"].items():
        assert close(st[k].grad, want, tol, atol=tol * scale), (k, rel_err(st[k].grad, want))


@pytest.mark.parametrize("B,r,E", [(7, 4, 3), (5, 1, 8), (9, 7, 1), (3, 32, 4)])
def test_row_kernel_backward_formulas_match_autograd(B, r, E):
    gen = torch.Generator().manual_seed(B * 100 + r * 10 + E)
    R = E * r
    n1, k2 = (R + E + 3) // 4 * 4, (R + 3) // 4 * 4
    P = torch.randn(B, n1, generator=gen, dtype=torch.float64).requires_grad_(True)
    C = (torch.randn(E, r, r, generator=gen, dtype=torch.float64) / r ** 0.5).requires_grad_(True)
    dA2 = torch.randn(B, k2, generator=gen, dtype=torch.float64)
    A2 = row_forward(P, C)
    assert float(A2.detach()[:, R:].abs().sum()) == 0.0
    A2.backward(dA2)
    dA1, dC = row_backward(P.detach(), C.detach(), dA2)
    assert torch.allclose(dA1[:, :R + E], P.grad[:, :R + E], rtol=1e-12, atol=1e-13)
    assert float(dA1[:, R + E:].abs().sum()) == 0.0
    assert torch.allclose(dC, C.grad, rtol=1e-12, atol=1e-13)


# ------------------------------------------------------------------ construction
def test_mirror_state_dict_matches_reference_construction():
    """Keys, registration order, shapes and initial values (same RNG draws) of the reference's CrossNetMix
    built under the same seed (tests/golden/crossnet_mix_init.json, written by make_crossnet_mix_golden.py)."""
    with open(os.path.join(GOLDEN, "crossnet_mix_init.json")) as fd:
        cases = json.load(fd)
    assert len(cases) >= 3
    for name, case in cases.items():
        d, nl, r, E = case["args"]
        torch.manual_seed(case["seed"])
        layer = layers.CrossNetMix(d, layer_num=nl, low_rank=r, num_experts=E)
        got = [[k, str(v.dtype), list(v.shape), hashlib.sha256(v.detach().contiguous().numpy().tobytes()).hexdigest()]
               for k, v in layer.state_dict().items()]
        assert got == case["state_dict"], name


@pytest.mark.parametrize("r,E", [(65, 1), (0, 4), (64, 5), (32, 9), (4, 0)])
def test_mirror_refuses_ranks_outside_the_kernels(r, E):
    with pytest.raises(NotImplementedError, match="low_rank|num_experts"):
        layers.CrossNetMix(16, layer_num=1, low_rank=r, num_experts=E)


def test_kernel_range_is_checked_before_any_cuda_call():
    import __graft_entry__
    __graft_entry__.build()
    L = _lib.load()
    p = ctypes.c_void_p(4096)
    assert L.b2_crossmix_fwd(p, p, 8, 65, 1, p, None, 0, 0, None) == -1 and b"low_rank" in L.b2_last_error()
    assert L.b2_crossmix_bwd(p, p, p, 8, 32, 9, p, None, 0, 0, p, None) == -1 and b"num_experts" in L.b2_last_error()
    assert L.b2_crossmix_pack(p, p, p, 16, 0, 4, p, p, None) == -1
    assert L.b2_crossmix_unpack(p, p, 16, 64, 5, p, p, p, None) == -1
    assert L.b2_crossmix_fwd(None, p, 8, 4, 3, p, None, 0, 0, None) == -1 and b"NULL" in L.b2_last_error()
    assert L.b2_crossmix_fwd(p, p, 8, 4, 3, p, p, _lib.B2_BF16, 8, None) == -1 and b"ld_aux" in L.b2_last_error()
    assert L.b2_crossmix_fwd(p, p, 0, 4, 3, p, None, 0, 0, None) == 0            # empty batch: nothing to launch


# ------------------------------------------------------------------ launch sequence (no GPU: _lib.call recorded)
@pytest.fixture
def recorder(monkeypatch):
    calls = []

    def fake_call(name, *a):
        info = None
        if name == "b2_gemm_tc_ex":
            d = ctypes.cast(a[0], ctypes.POINTER(_lib.b2_gemm_desc)).contents
            info = dict(M=d.M, N=d.N, K=d.K, a_mn=d.a_mn_major, b_mn=d.b_mn_major, bias=bool(d.bias), mul=bool(d.mul),
                        add=bool(d.add), c_pre=bool(d.c_pre), colsum=bool(d.colsum), act=d.act,
                        bf16=d.elem_dtype == _lib.B2_BF16, aux=bool(d.a_small) and bool(d.b_small),
                        inline=bool(d.flags & _lib.B2_GEMM_X3_INLINE))
        elif name == "b2_gemm_f32":
            info = dict(M=a[8], N=a[9], K=a[10], bias=bool(a[11].value), add=bool(a[14].value))
        calls.append((name, info))
        return 0

    monkeypatch.setattr(_lib, "call", fake_call)
    monkeypatch.setattr(F2, "_stream", lambda: None)
    monkeypatch.setattr(F2, "_require_cuda", lambda *t: None)
    yield calls
    F2.set_matmul_precision("fp32")
    F2.set_x3_inline(True)


def run_layer(mode, B, d, r, E, inline=True):
    F2.set_x3_inline(inline)
    F2.set_matmul_precision(mode)
    torch.manual_seed(3)
    x0 = torch.randn(B, d, requires_grad=True)
    xl = torch.randn(B, d, requires_grad=True)
    U = torch.nn.Parameter(torch.randn(E, d, r))
    V = torch.nn.Parameter(torch.randn(E, d, r))
    C = torch.nn.Parameter(torch.randn(E, r, r))
    gates = [torch.nn.Parameter(torch.randn(1, d)) for _ in range(E)]
    bias = torch.nn.Parameter(torch.zeros(d, 1))
    out = F2.crossnet_mix_layer(x0, xl, U, V, C, gates, bias)
    assert type(out.grad_fn).__name__ == "_CrossMixLayerBackward"
    out.backward(torch.randn_like(out))
    for p in [U, V, C, bias] + gates:
        assert p.grad is not None and p.grad.shape == p.shape


@pytest.mark.parametrize("mode", ["tf32x3", "tf32", "bf16"])
def test_c3_layer_is_four_launches_forward_and_seven_backward(recorder, mode):
    """C3 (B 8192, d 624, r 32, E 4): pack, GEMM1, row kernel, GEMM2 with the CrossNetV2 epilogue; backward
    g*x_0 pass, dA2 dgrad, dW2 wgrad, row kernel, dx_l dgrad (+g), dW1 wgrad, unpack.  bf16 adds only the
    bf16 copies of x_l, W1, W2 and dlin (the row kernels write those of A2 and dA1 themselves)."""
    B, d, r, E = 8192, 624, 32, 4
    n1, k2 = 132, 128
    run_layer(mode, B, d, r, E)
    names = [n for n, _ in recorder if n != "b2_to_bf16"]
    assert names == ["b2_crossmix_pack", "b2_gemm_tc_ex", "b2_crossmix_fwd", "b2_gemm_tc_ex",
                     "b2_prep_operand", "b2_gemm_tc_ex", "b2_gemm_tc_ex", "b2_crossmix_bwd", "b2_gemm_tc_ex",
                     "b2_gemm_tc_ex", "b2_crossmix_unpack"]
    assert [n for n, _ in recorder].count("b2_to_bf16") == (4 if mode == "bf16" else 0)
    g1, g2, da2, dw2, dx, dw1 = [i for n, i in recorder if n == "b2_gemm_tc_ex"]
    assert all(g["bf16"] == (mode == "bf16") and g["inline"] == (mode == "tf32x3") for g in (g1, g2, da2, dw2, dx, dw1))
    assert (g1["M"], g1["N"], g1["K"], g1["a_mn"], g1["b_mn"]) == (B, n1, d, 0, 0)
    assert not (g1["bias"] or g1["mul"] or g1["add"] or g1["c_pre"])
    assert (g2["M"], g2["N"], g2["K"], g2["a_mn"], g2["b_mn"]) == (B, d, k2, 0, 0)
    assert g2["bias"] and g2["mul"] and g2["add"] and g2["c_pre"]
    assert (da2["M"], da2["N"], da2["K"], da2["a_mn"], da2["b_mn"], da2["add"]) == (B, k2, d, 0, 1, False)
    assert (dw2["M"], dw2["N"], dw2["K"], dw2["a_mn"], dw2["b_mn"]) == (d, k2, B, 1, 1)
    assert (dx["M"], dx["N"], dx["K"], dx["a_mn"], dx["b_mn"], dx["add"]) == (B, d, n1, 0, 1, True)
    assert (dw1["M"], dw1["N"], dw1["K"], dw1["a_mn"], dw1["b_mn"]) == (n1, d, B, 1, 1)


def test_x3_aux_layout_adds_only_the_weight_and_input_splits(recorder):
    run_layer("tf32x3", 512, 624, 32, 4, inline=False)
    names = [n for n, _ in recorder]
    assert names.count("b2_split_tf32") == 3            # x_l, W1, W2; A2, dA1 and dlin come with their small parts
    g = [i for n, i in recorder if n == "b2_gemm_tc_ex"]
    assert len(g) == 6 and all(d["aux"] and not d["inline"] for d in g)


@pytest.mark.parametrize("mode,d,r,E", [("fp32", 624, 32, 4), ("tf32x3", 30, 4, 3), ("tf32", 20, 4, 3),
                                        ("bf16", 64, 1, 8), ("tf32x3", 12, 8, 1)])
def test_simt_gemms_where_the_tensor_cores_cannot_go(recorder, mode, d, r, E):
    """fp32 mode, d % 4 != 0, or a packed dimension under 16 (E*r + E -> N1, E*r -> K2): the SIMT GEMM,
    with the same row kernels."""
    B = 37
    R = E * r
    n1, k2 = (R + R // r + 3) // 4 * 4, (R + 3) // 4 * 4
    run_layer(mode, B, d, r, E)
    names = [n for n, _ in recorder]
    assert names == ["b2_crossmix_pack", "b2_gemm_f32", "b2_crossmix_fwd", "b2_gemm_f32",
                     "b2_prep_operand", "b2_gemm_f32", "b2_gemm_f32", "b2_crossmix_bwd", "b2_gemm_f32",
                     "b2_gemm_f32", "b2_crossmix_unpack"]
    g1, g2, da2, dw2, dx, dw1 = [i for n, i in recorder if n == "b2_gemm_f32"]
    assert (g1["M"], g1["N"], g1["K"]) == (B, n1, d)
    assert (g2["M"], g2["N"], g2["K"], g2["bias"]) == (B, d, k2, True)
    assert (da2["M"], da2["N"], da2["K"]) == (B, k2, d)
    assert (dw2["M"], dw2["N"], dw2["K"]) == (d, k2, B)
    assert (dx["M"], dx["N"], dx["K"], dx["add"]) == (B, d, n1, True)
    assert (dw1["M"], dw1["N"], dw1["K"]) == (n1, d, B)


# ------------------------------------------------------------------ patch.enable() on the real reference
needs_ref = pytest.mark.skipif(not refenv.available(), reason=refenv.why_unavailable())


def build_ref_dcnv2_mix(g):
    from collections import OrderedDict
    R = refenv.import_reference()
    fm = R.FeatureMap("synthetic", "/tmp")
    fm.features = OrderedDict((k, dict(v)) for k, v in g.meta["specs"])
    fm.labels = g.meta["labels"]
    fm.default_emb_dim = g.meta["kwargs"]["embedding_dim"]
    fm.num_fields = fm.get_num_fields()
    fm.set_column_index()
    model = refenv.load_model_class("DCNv2")(fm, model_root="/tmp/b2_patch_mix/", metrics=["AUC"], verbose=0,
                                             optimizer="adam", loss="binary_crossentropy",
                                             task="binary_classification", gpu=-1, **g.meta["kwargs"])
    model.load_state_dict(g["w"])
    B = g.meta["batch"]
    mat = g["in"]["matrix"][:B]
    return model, {c: mat[:, fm.get_column_index(c)] for c in list(fm.features.keys()) + fm.labels}


@needs_ref
def test_enable_leaves_cpu_dcnv2_mix_bit_identical():
    from fuxictr_b200 import patch
    g = Golden("model_DCNv2_mix")
    model, batch = build_ref_dcnv2_mix(g)
    y0 = model.forward(batch)["y_pred"]
    assert rel_err(y0, g["out"]["y_pred"]) <= 1e-6
    patch.enable()
    try:
        assert type(model.crossnet).__name__ == "CrossNetMix"
        y1 = model.forward(batch)["y_pred"]
        assert torch.equal(y0, y1)
        assert "CrossNetMix" not in patch.call_counts()
    finally:
        patch.disable()


@needs_ref
def test_cuda_tensors_reach_the_crossnet_mix_kernels(monkeypatch):
    """No GPU here: with the tensors claimed to be CUDA, a supported CrossNetMix takes the kernel path (whose
    entry refuses CPU tensors loudly); one outside the kernels' range runs the reference's own forward."""
    from fuxictr_b200 import patch
    R = refenv.import_reference()
    torch.manual_seed(5)
    x = torch.randn(6, 20)
    ok = R.layers.CrossNetMix(20, layer_num=2, low_rank=4, num_experts=3)
    wide = R.layers.CrossNetMix(20, layer_num=1, low_rank=65, num_experts=1)
    want = wide(x)
    monkeypatch.setitem(patch._STATE, "calls", {})      # this test's counts stay out of the process-wide ones
    patch.enable()
    try:
        monkeypatch.setattr(patch, "_on_cuda", lambda a, k: True)
        with pytest.raises(RuntimeError, match="CUDA"):
            ok(x)
        assert patch.call_counts() == {"CrossNetMix": 1}
        assert torch.equal(wide(x), want)
        assert patch.call_counts() == {"CrossNetMix": 1}
    finally:
        patch.disable()

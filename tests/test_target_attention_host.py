"""MultiHeadTargetAttention without a GPU: the folded layer that the kernels compute (projections packed into
W_M, W_N, a masked softmax over the unprojected history) against the oracle and the reference's goldens, the
row kernels' backward formulas and the unpack against autograd, the mirror's construction against the
reference's, the C-ABI's range checks, the launch sequence per matmul mode, and the patch's routing."""
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


# ------------------------------------------------------------------ the folded layer in float64 torch
def pack(Wq, Wk, Wv, Wo, H, s):
    """W_M (H*d, d), W_N (d, H*d) by the layout of include/fuxictr_b200.h "MultiHeadTargetAttention"."""
    A, d = Wq.shape
    hd = A // H
    WM = torch.cat([(s * Wq[h * hd:(h + 1) * hd].t() @ Wk[h * hd:(h + 1) * hd]).t() for h in range(H)], dim=0)
    WN = torch.cat([(Wv[h * hd:(h + 1) * hd].t() @ Wo[:, h * hd:(h + 1) * hd].t()).t() for h in range(H)], dim=1)
    return WM, WN


def head_cols(H, w, xs):
    return [slice(h * xs, h * xs + w) for h in range(H)]


def row_forward(q, x, mask, H, w, xs, scale):
    """b2_mhta_fwd: p (B, H*w) and stats (B, H, 2) = {max score, sum of exp(score - max)}."""
    ps, stats = [], []
    for h, cols in enumerate(head_cols(H, w, xs)):
        sc = scale * torch.einsum("bk,blk->bl", q[:, h * w:(h + 1) * w], x[:, :, cols])
        if mask is not None:
            sc = sc.masked_fill(mask == 0, -1.e9)
        m = sc.max(dim=1, keepdim=True).values
        e = torch.exp(sc - m)
        a = e / e.sum(dim=1, keepdim=True)
        ps.append(torch.einsum("bl,blk->bk", a, x[:, :, cols]))
        stats.append(torch.stack([m[:, 0], e.sum(dim=1)], dim=1))
    return torch.cat(ps, dim=1), torch.stack(stats, dim=1)


def row_backward(q, x, mask, p, stats, dp, H, w, xs, scale):
    """b2_mhta_bwd's formulas: a recomputed from the stats, ds = a (dp.x - dp.p) (0 where masked)."""
    dq, dx = torch.zeros_like(q), torch.zeros_like(x)
    for h, cols in enumerate(head_cols(H, w, xs)):
        qh, dph, ph = q[:, h * w:(h + 1) * w], dp[:, h * w:(h + 1) * w], p[:, h * w:(h + 1) * w]
        xh = x[:, :, cols]
        sc = scale * torch.einsum("bk,blk->bl", qh, xh)
        if mask is not None:
            sc = sc.masked_fill(mask == 0, -1.e9)
        a = torch.exp(sc - stats[:, h, :1]) / stats[:, h, 1:]
        ds = a * (torch.einsum("bk,blk->bl", dph, xh) - (dph * ph).sum(1, keepdim=True))
        if mask is not None:
            ds = ds.masked_fill(mask == 0, 0.0)
        dx[:, :, cols] += a.unsqueeze(2) * dph.unsqueeze(1) + scale * ds.unsqueeze(2) * qh.unsqueeze(1)
        dq[:, h * w:(h + 1) * w] = scale * torch.einsum("bl,blk->bk", ds, xh)
    return dq, dx


def unpack(Wq, Wk, Wv, Wo, dWM, dWN, H, s):
    """b2_mhta_unpack: the four weight gradients from dW_M (H*d, d), dW_N (d, H*d)."""
    A, d = Wq.shape
    hd = A // H
    g = [torch.zeros_like(w) for w in (Wq, Wk, Wv, Wo)]
    for h in range(H):
        r = slice(h * hd, (h + 1) * hd)
        dM = dWM[h * d:(h + 1) * d].t()                  # dM_h (d x d)
        dN = dWN[:, h * d:(h + 1) * d].t()               # dN_h (d x d)
        g[0][r] = s * Wk[r] @ dM.t()
        g[1][r] = s * Wq[r] @ dM
        g[2][r] = Wo[:, r].t() @ dN.t()
        g[3][:, r] = dN.t() @ Wv[r].t()
    return g


def folded(t, x, mask, H, use_scale, W=None):
    """The layer as the kernels compute it (W: W_q, W_k, W_v, W_o or None)."""
    d = x.shape[2]
    if W is None:
        hd = d // H
        return row_forward(t, x, mask, H, hd, hd, hd ** -0.5 if use_scale else 1.0)[0]
    hd = W[0].shape[0] // H
    WM, WN = pack(*W, H, hd ** -0.5 if use_scale else 1.0)
    return row_forward(t @ WM.t(), x, mask, H, d, 0, 1.0)[0] @ WN.t()


@pytest.mark.parametrize("name", ["h1_qkvo1", "h3_qkvo1", "h2_qkvo0"])
def test_folded_layer_matches_the_reference_golden(name):
    """Projections folded into W_M, W_N (or the sliced heads) give the reference's output and every gradient
    within the oracle's own bar (2e-6), and the oracle to float64 rounding."""
    g = Golden("next_MHTA_" + name)
    m = g.meta
    st = {k: v.clone().double().requires_grad_(True) for k, v in g["w"].items()}
    t = g["in"]["target"].clone().double().requires_grad_(True)
    x = g["in"]["history"].clone().double().requires_grad_(True)
    mask = g["in"]["mask"].double()
    W = [st["W_%s.weight" % c] for c in "qkvo"] if m["use_qkvo"] else None
    out = folded(t, x, mask, m["heads"], m["use_scale"], W)
    tol = 2e-6
    assert close(out, g["out"]["y"], tol), rel_err(out, g["out"]["y"])
    ref = O.multi_head_target_attention({k: v.detach() for k, v in st.items()}, "", t.detach(), x.detach(), mask,
                                        m["heads"], m["use_scale"], m["use_qkvo"])
    assert close(out, ref, 1e-12)
    (out * g["in"]["gout"].double()).sum().backward()
    assert close(t.grad, g["gin"]["target"], tol), rel_err(t.grad, g["gin"]["target"])
    assert close(x.grad, g["gin"]["history"], tol), rel_err(x.grad, g["gin"]["history"])
    scale = max([float(v.abs().max()) for v in g["g"].values()] + [1e-30])
    for k, want in g["g"].items():
        assert close(st[k].grad, want, tol, atol=tol * scale), (k, rel_err(st[k].grad, want))


# (B, L, d, A, H, qkvo, use_scale, mask kind)
CASES = [(6, 7, 12, 12, 2, True, True, "ragged"), (5, 9, 12, 12, 2, True, True, "all_masked"),
         (4, 5, 8, 24, 3, True, False, None), (6, 40, 12, 12, 3, False, True, "ragged"),
         (5, 33, 12, 12, 2, False, False, "all_masked"), (3, 4, 6, 6, 1, False, True, None)]


def make_case(B, L, d, A, H, qkvo, use_scale, mask_kind, seed=0):
    gen = torch.Generator().manual_seed(seed + B * 100 + L)
    t = torch.randn(B, d, generator=gen, dtype=torch.float64)
    x = torch.randn(B, L, d, generator=gen, dtype=torch.float64)
    mask = None
    if mask_kind is not None:
        lens = torch.randint(1, L + 1, (B,), generator=gen)
        mask = (torch.arange(L)[None, :] < lens[:, None]).double()
        if mask_kind == "all_masked":
            mask[::2] = 0.0                                # every other row: a history of padding only
    W = [torch.randn(*s, generator=gen, dtype=torch.float64) / d ** 0.5
         for s in ((A, d), (A, d), (A, d), (d, A))] if qkvo else None
    return t, x, mask, W


@pytest.mark.parametrize("B,L,d,A,H,qkvo,use_scale,mask_kind", CASES)
def test_folded_layer_matches_the_oracle(B, L, d, A, H, qkvo, use_scale, mask_kind):
    t, x, mask, W = make_case(B, L, d, A, H, qkvo, use_scale, mask_kind)
    state = {"W_%s.weight" % c: w for c, w in zip("qkvo", W)} if qkvo else {}
    ref = O.multi_head_target_attention(state, "", t, x, mask, H, use_scale, qkvo)
    assert close(folded(t, x, mask, H, use_scale, W), ref, 1e-12)


@pytest.mark.parametrize("B,L,d,A,H,qkvo,use_scale,mask_kind", CASES)
def test_backward_formulas_and_unpack_match_autograd(B, L, d, A, H, qkvo, use_scale, mask_kind):
    """The row kernel's backward (no second sweep over L: sum_l a da = dp . p) and the unpack, chained as
    _TargetAttention.backward chains them, against autograd through the oracle."""
    t, x, mask, W = make_case(B, L, d, A, H, qkvo, use_scale, mask_kind, seed=1)
    leaves = [t, x] + (W if qkvo else [])
    leaves = [v.clone().requires_grad_(True) for v in leaves]
    state = {"W_%s.weight" % c: w for c, w in zip("qkvo", leaves[2:])} if qkvo else {}
    out = O.multi_head_target_attention(state, "", leaves[0], leaves[1], mask, H, use_scale, qkvo)
    gout = torch.randn(out.shape, generator=torch.Generator().manual_seed(7), dtype=torch.float64)
    out.backward(gout)
    hd = A // H
    s = hd ** -0.5 if use_scale else 1.0
    if qkvo:
        WM, WN = pack(*W, H, s)
        q = t @ WM.t()
        p, stats = row_forward(q, x, mask, H, d, 0, 1.0)
        dp, dWN = gout @ WN, gout.t() @ p
        dq, dx = row_backward(q, x, mask, p, stats, dp, H, d, 0, 1.0)
        dt, dWM = dq @ WM, dq.t() @ t
        grads = [dt, dx] + unpack(*W, dWM, dWN, H, s)
    else:
        p, stats = row_forward(t, x, mask, H, hd, hd, s)
        dq, dx = row_backward(t, x, mask, p, stats, gout, H, hd, hd, s)
        grads = [dq, dx]
    for got, leaf in zip(grads, leaves):
        assert torch.allclose(got, leaf.grad, rtol=1e-10, atol=1e-12), rel_err(got, leaf.grad)
    if mask_kind == "all_masked":
        # a history of padding only: uniform attention, so every position gets dp / L (sliced: its head's columns)
        assert float(stats[0, :, 0].max()) == -1.e9
        assert torch.all(stats[0, :, 1] == L)


# ------------------------------------------------------------------ construction
def test_mirror_state_dict_matches_reference_construction():
    """Keys, registration order, shapes, initial values (same RNG draws) and child names of the reference's
    MultiHeadTargetAttention built under the same seed (tests/golden/target_attention_init.json, written by
    make_target_attention_golden.py)."""
    with open(os.path.join(GOLDEN, "target_attention_init.json")) as fd:
        cases = json.load(fd)
    assert len(cases) >= 4
    for name, case in cases.items():
        d, A, H, qkvo = case["args"]
        torch.manual_seed(case["seed"])
        layer = layers.MultiHeadTargetAttention(input_dim=d, attention_dim=A, num_heads=H, use_qkvo=qkvo)
        got = [[k, str(v.dtype), list(v.shape), hashlib.sha256(v.detach().contiguous().numpy().tobytes()).hexdigest()]
               for k, v in layer.state_dict().items()]
        assert got == case["state_dict"], name
        assert [n for n, _ in layer.named_children()] == case["children"], name


@pytest.mark.parametrize("d,A,H,qkvo", [(512, 512, 4, True), (12, 66, 33, True), (1040, 1040, 2, False)])
def test_mirror_refuses_widths_outside_the_kernels(d, A, H, qkvo):
    with pytest.raises(NotImplementedError, match="num_heads|row width"):
        layers.MultiHeadTargetAttention(input_dim=d, attention_dim=A, num_heads=H, use_qkvo=qkvo)


def test_mirror_refuses_training_mode_attention_dropout():
    layer = layers.MultiHeadTargetAttention(input_dim=12, attention_dim=12, num_heads=2, dropout_rate=0.1)
    with pytest.raises(NotImplementedError, match="dropout"):
        layer(torch.zeros(2, 12), torch.zeros(2, 3, 12))
    with pytest.raises(NotImplementedError, match="inside"):
        layer.dot_attention(torch.zeros(1), torch.zeros(1), torch.zeros(1))


def test_kernel_range_is_checked_before_any_cuda_call():
    import __graft_entry__
    __graft_entry__.build()
    L = _lib.load()
    p = ctypes.c_void_p(4096)
    n = None
    # fwd: (q, x, mask, batch, L, d, heads, width, x_step, scale, p, stats, p_aux, aux_dtype, ld_aux, stream)
    assert L.b2_mhta_fwd(p, p, n, 8, 5, 512, 4, 512, 0, 1.0, p, p, n, 0, 0, n) == -1 \
        and b"width" in L.b2_last_error()
    assert L.b2_mhta_fwd(p, p, n, 8, 5, 66, 33, 2, 2, 1.0, p, p, n, 0, 0, n) == -1 and b"heads" in L.b2_last_error()
    assert L.b2_mhta_fwd(p, p, n, 8, 0, 12, 2, 6, 6, 1.0, p, p, n, 0, 0, n) == -1 and b"length" in L.b2_last_error()
    assert L.b2_mhta_fwd(p, p, n, 1 << 26, 64, 12, 2, 6, 6, 1.0, p, p, n, 0, 0, n) == -1 \
        and b"int32" in L.b2_last_error()
    assert L.b2_mhta_fwd(p, p, n, 8, 5, 12, 2, 6, 3, 1.0, p, p, n, 0, 0, n) == -1 and b"x_step" in L.b2_last_error()
    assert L.b2_mhta_fwd(p, p, n, 8, 5, 1040, 1, 1040, 0, 1.0, p, p, n, 0, 0, n) == -1
    assert L.b2_mhta_fwd(n, p, n, 8, 5, 12, 2, 12, 0, 1.0, p, p, n, 0, 0, n) == -1 and b"NULL" in L.b2_last_error()
    assert L.b2_mhta_fwd(p, p, n, 8, 5, 12, 2, 12, 0, 1.0, p, p, p, _lib.B2_BF16, 8, n) == -1 \
        and b"ld_aux" in L.b2_last_error()
    assert L.b2_mhta_fwd(p, p, n, 0, 5, 12, 2, 12, 0, 1.0, p, p, n, 0, 0, n) == 0     # empty batch: no launch
    # bwd: (q, x, mask, p, stats, dp, batch, L, d, heads, width, x_step, scale, dq, dx, dq_aux, aux_dtype, ld_aux, s)
    assert L.b2_mhta_bwd(p, p, n, p, p, p, 8, 5, 512, 4, 512, 0, 1.0, p, p, n, 0, 0, n) == -1 \
        and b"width" in L.b2_last_error()
    assert L.b2_mhta_bwd(p, p, n, p, p, p, 8, 5, 66, 33, 2, 2, 1.0, p, p, n, 0, 0, n) == -1
    assert L.b2_mhta_bwd(p, p, n, p, p, n, 8, 5, 12, 2, 12, 0, 1.0, p, p, n, 0, 0, n) == -1 \
        and b"NULL" in L.b2_last_error()
    # pack / unpack: heads * d within the width bound
    assert L.b2_mhta_pack(p, p, p, p, 512, 4, 128, 1.0, p, p, n) == -1 and b"input_dim" in L.b2_last_error()
    assert L.b2_mhta_pack(p, p, p, p, 12, 33, 2, 1.0, p, p, n) == -1 and b"heads" in L.b2_last_error()
    assert L.b2_mhta_unpack(p, p, p, p, p, p, 512, 4, 128, 1.0, p, p, p, p, n) == -1
    assert L.b2_mhta_unpack(p, p, p, p, p, p, 12, 2, 0, 1.0, p, p, p, p, n) == -1 and b"head_dim" in L.b2_last_error()


# ------------------------------------------------------------------ launch sequence (no GPU: _lib.call recorded)
@pytest.fixture
def recorder(monkeypatch):
    calls = []

    def fake_call(name, *a):
        info = None
        if name == "b2_gemm_tc_ex":
            d = ctypes.cast(a[0], ctypes.POINTER(_lib.b2_gemm_desc)).contents
            info = dict(M=d.M, N=d.N, K=d.K, a_mn=d.a_mn_major, b_mn=d.b_mn_major, bf16=d.elem_dtype == _lib.B2_BF16,
                        aux=bool(d.a_small) and bool(d.b_small), inline=bool(d.flags & _lib.B2_GEMM_X3_INLINE))
        elif name == "b2_gemm_f32":
            info = dict(M=a[8], N=a[9], K=a[10])
        elif name in ("b2_mhta_fwd", "b2_mhta_bwd"):
            k = 3 if name == "b2_mhta_fwd" else 6
            info = dict(mask=bool(a[2].value), geom=tuple(a[k:k + 7]), aux=bool(a[-4].value))
        calls.append((name, info))
        return 0

    monkeypatch.setattr(_lib, "call", fake_call)
    monkeypatch.setattr(F2, "_stream", lambda: None)
    monkeypatch.setattr(F2, "_require_cuda", lambda *t: None)
    yield calls
    F2.set_matmul_precision("fp32")
    F2.set_x3_inline(True)


def run_layer(mode, B, L, d, A, H, qkvo=True, inline=True, mask=True):
    F2.set_x3_inline(inline)
    F2.set_matmul_precision(mode)
    torch.manual_seed(3)
    layer = layers.MultiHeadTargetAttention(input_dim=d, attention_dim=A, num_heads=H, use_qkvo=qkvo)
    t = torch.randn(B, d, requires_grad=True)
    x = torch.randn(B, L, d, requires_grad=True)
    m = (torch.rand(B, L) < 0.7) if mask else None
    out = layer(t, x, m)
    assert type(out.grad_fn).__name__ == "_TargetAttentionBackward" and tuple(out.shape) == (B, d)
    out.backward(torch.randn_like(out))
    assert t.grad is not None and x.grad is not None
    for prm in layer.parameters():
        assert prm.grad is not None and prm.grad.shape == prm.shape


FOLD = ["b2_mhta_pack", "b2_gemm_tc_ex", "b2_mhta_fwd", "b2_gemm_tc_ex",
        "b2_gemm_tc_ex", "b2_gemm_tc_ex", "b2_mhta_bwd", "b2_gemm_tc_ex", "b2_gemm_tc_ex", "b2_mhta_unpack"]


@pytest.mark.parametrize("mode", ["tf32x3", "tf32", "bf16"])
def test_wide_layer_is_four_launches_forward_and_six_backward(recorder, mode):
    """B 4096, L 200, d 64, 4 heads: pack, GEMM1 q' = t W_M^T, row kernel, GEMM2 out = p W_N^T; backward dp
    dgrad, dW_N wgrad, row kernel, dt dgrad, dW_M wgrad, unpack.  bf16 adds only the bf16 copies of t, W_M,
    W_N and the incoming gradient (the row kernels write those of p and dq' themselves)."""
    B, L, d, H = 4096, 200, 64, 4
    run_layer(mode, B, L, d, 64, H)
    assert [n for n, _ in recorder if n != "b2_to_bf16"] == FOLD
    assert [n for n, _ in recorder].count("b2_to_bf16") == (4 if mode == "bf16" else 0)
    g1, g2, dp, dwn, dt, dwm = [i for n, i in recorder if n == "b2_gemm_tc_ex"]
    assert all(g["bf16"] == (mode == "bf16") and g["inline"] == (mode == "tf32x3") for g in (g1, g2, dp, dwn, dt, dwm))
    assert (g1["M"], g1["N"], g1["K"], g1["a_mn"], g1["b_mn"]) == (B, H * d, d, 0, 0)
    assert (g2["M"], g2["N"], g2["K"], g2["a_mn"], g2["b_mn"]) == (B, d, H * d, 0, 0)
    assert (dp["M"], dp["N"], dp["K"], dp["a_mn"], dp["b_mn"]) == (B, H * d, d, 0, 1)
    assert (dwn["M"], dwn["N"], dwn["K"], dwn["a_mn"], dwn["b_mn"]) == (d, H * d, B, 1, 1)
    assert (dt["M"], dt["N"], dt["K"], dt["a_mn"], dt["b_mn"]) == (B, d, H * d, 0, 1)
    assert (dwm["M"], dwm["N"], dwm["K"], dwm["a_mn"], dwm["b_mn"]) == (H * d, d, B, 1, 1)
    fwd, bwd = [i for n, i in recorder if n in ("b2_mhta_fwd", "b2_mhta_bwd")]
    assert fwd["geom"][:6] == bwd["geom"][:6] == (B, L, d, H, d, 0) and fwd["geom"][6] == 1.0 and fwd["mask"]
    assert fwd["aux"] == bwd["aux"] == (mode == "bf16")


def test_x3_aux_layout_adds_only_the_input_and_weight_splits(recorder):
    run_layer("tf32x3", 512, 50, 64, 64, 4, inline=False)
    names = [n for n, _ in recorder]
    assert names.count("b2_split_tf32") == 4            # t, W_M, W_N, the incoming gradient; p, dq' by the kernels
    g = [i for n, i in recorder if n == "b2_gemm_tc_ex"]
    assert len(g) == 6 and all(d["aux"] and not d["inline"] for d in g)


@pytest.mark.parametrize("mode,d,A,H", [("fp32", 64, 64, 4), ("tf32x3", 12, 64, 2), ("tf32", 12, 12, 1),
                                        ("bf16", 18, 36, 2), ("tf32x3", 8, 8, 1)])
def test_simt_gemms_where_the_tensor_cores_cannot_go(recorder, mode, d, A, H):
    """fp32 mode, d under 16 (the SIM / ETA item width 12), d % 4 != 0, or H*d under 16: the SIMT GEMM,
    with the same row kernels."""
    B, L = 37, 50
    run_layer(mode, B, L, d, A, H)
    assert [n for n, _ in recorder] == [n.replace("tc_ex", "f32") for n in FOLD]
    g1, g2, dp, dwn, dt, dwm = [i for n, i in recorder if n == "b2_gemm_f32"]
    assert (g1["M"], g1["N"], g1["K"]) == (B, H * d, d)
    assert (g2["M"], g2["N"], g2["K"]) == (B, d, H * d)
    assert (dp["M"], dp["N"], dp["K"]) == (B, H * d, d)
    assert (dwn["M"], dwn["N"], dwn["K"]) == (d, H * d, B)
    assert (dt["M"], dt["N"], dt["K"]) == (B, d, H * d)
    assert (dwm["M"], dwm["N"], dwm["K"]) == (H * d, d, B)


@pytest.mark.parametrize("mode", ["fp32", "bf16"])
@pytest.mark.parametrize("mask", [True, False])
def test_sliced_layer_is_the_row_kernels_alone(recorder, mode, mask):
    """use_qkvo=False: one launch each way whatever the precision; head h reads its hd columns, the kernel scales."""
    run_layer(mode, 9, 33, 12, 12, 3, qkvo=False, mask=mask)
    assert [n for n, _ in recorder] == ["b2_mhta_fwd", "b2_mhta_bwd"]
    fwd, bwd = [i for _, i in recorder]
    assert fwd["geom"][:6] == bwd["geom"][:6] == (9, 33, 12, 3, 4, 4) and fwd["mask"] == mask
    assert abs(fwd["geom"][6] - 0.5) < 1e-7 and not fwd["aux"]


# ------------------------------------------------------------------ patch.enable() on the real reference
needs_ref = pytest.mark.skipif(not refenv.available(), reason=refenv.why_unavailable())


@needs_ref
def test_cuda_tensors_reach_the_target_attention_kernels(monkeypatch):
    """No GPU here: with the tensors claimed to be CUDA, a supported MultiHeadTargetAttention takes the kernel path
    (whose entry refuses CPU tensors loudly); training-mode attention dropout and a width over the bound run the
    reference's own forward and launch nothing."""
    from fuxictr_b200 import patch
    R = refenv.import_reference()
    torch.manual_seed(5)
    t, x = torch.randn(6, 12), torch.randn(6, 7, 12)
    mask = torch.ones(6, 7)
    ok = R.layers.MultiHeadTargetAttention(12, 12, num_heads=2)
    drop = R.layers.MultiHeadTargetAttention(12, 12, num_heads=2, dropout_rate=0.2)
    wide = R.layers.MultiHeadTargetAttention(512, 64, num_heads=4)
    tw, xw = torch.randn(2, 512), torch.randn(2, 3, 512)
    want_wide = wide(tw, xw)
    monkeypatch.setitem(patch._STATE, "calls", {})
    launched = []
    monkeypatch.setattr(_lib, "call", lambda name, *a: launched.append(name))
    patch.enable()
    try:
        monkeypatch.setattr(patch, "_on_cuda", lambda a, k: True)
        with pytest.raises(RuntimeError, match="CUDA"):
            ok(t, x, mask)
        assert patch.call_counts() == {"MultiHeadTargetAttention": 1}
        drop.train()
        torch.manual_seed(9)
        y_drop = drop(t, x, mask)
        assert y_drop.shape == (6, 12)
        drop.eval()
        with pytest.raises(RuntimeError, match="CUDA"):
            drop(t, x, mask)                              # eval mode: dropout is a no-op, the kernels apply
        assert patch.call_counts() == {"MultiHeadTargetAttention": 2}
        assert torch.equal(wide(tw, xw), want_wide)
        assert patch.call_counts() == {"MultiHeadTargetAttention": 2}
        assert launched == []
    finally:
        patch.disable()

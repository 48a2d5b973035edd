"""Host logic of the dense path without a GPU: `_lib.call` is replaced by a recorder, so the autograd
wrappers run on CPU tensors and the test sees exactly which C-ABI entry points a step would launch,
in which order and with which descriptors (operand majors, fused-epilogue fields, arithmetic mode).
Numerics are NOT checked here (nothing is computed) — that is the `-m gpu` suite's job."""
import ctypes

import pytest
import torch

from fuxictr_b200 import _lib, functional as F2
from fuxictr_b200._lib import B2_ACT_NONE, B2_ACT_RELU


@pytest.fixture
def recorder(monkeypatch):
    calls = []

    def fake_call(name, *a):
        info = None
        if name == "b2_gemm_tc_ex":
            d = ctypes.cast(a[0], ctypes.POINTER(_lib.b2_gemm_desc)).contents
            info = dict(M=d.M, N=d.N, K=d.K, a_mn=d.a_mn_major, b_mn=d.b_mn_major, inline=bool(d.flags & _lib.B2_GEMM_X3_INLINE),
                        aux=bool(d.a_small) and bool(d.b_small), bf16=d.elem_dtype == _lib.B2_BF16, act=d.act,
                        ybwd=bool(d.ybwd), act_bwd=d.act_bwd, colsum=bool(d.colsum), bias=bool(d.bias),
                        c_small=bool(d.c_small), mul=bool(d.mul), add=bool(d.add), c_pre=bool(d.c_pre))
        calls.append((name, info))
        return 0

    monkeypatch.setattr(_lib, "call", fake_call)
    monkeypatch.setattr(F2, "_stream", lambda: None)
    monkeypatch.setattr(F2, "_require_cuda", lambda *t: None)
    yield calls
    F2.set_matmul_precision("fp32")
    F2.set_x3_inline(True)


def c2_mlp():
    torch.manual_seed(0)
    dims = [624, 300, 300, 300, 1]
    layers = []
    for i in range(4):
        w = torch.nn.Parameter(torch.randn(dims[i + 1], dims[i]) * 0.05)
        b = torch.nn.Parameter(torch.zeros(dims[i + 1]))
        layers.append((w, b, B2_ACT_RELU if i < 3 else B2_ACT_NONE))
    return layers


def run_chain(mode, inline=True):
    F2.set_x3_inline(inline)
    F2.set_matmul_precision(mode)
    x = torch.randn(4096, 624, requires_grad=True)
    y = F2.mlp_chain(x, c2_mlp())
    assert type(y.grad_fn).__name__.startswith("_MLPChain")
    y.backward(torch.randn_like(y))


def test_c2_mlp_step_is_eleven_launches_in_3xtf32(recorder):
    """DeepFM C2's MLP (624-300-300-300-1): 3 forward GEMMs + head, then head backward + 3 x (dgrad, wgrad) —
    no operand-preparation, split or transpose launch anywhere (DESIGN.md section 4: 16 launches per step with
    the fused front forward/backward, logit+BCE, sumsq and Adam)."""
    run_chain("tf32x3")
    names = [n for n, _ in recorder]
    assert names == ["b2_gemm_tc_ex"] * 3 + ["b2_head_fwd", "b2_head_bwd_ex"] + ["b2_gemm_tc_ex"] * 6
    g = [i for _, i in recorder if i is not None]
    fwd, bwd = g[:3], g[3:]
    assert [(d["M"], d["N"], d["K"]) for d in fwd] == [(4096, 300, 624), (4096, 300, 300), (4096, 300, 300)]
    for d in fwd:       # Y = act(X W^T + b): K-major operands, bias + ReLU in the epilogue, small parts made in-kernel
        assert d["inline"] and not d["aux"] and not d["bf16"] and d["bias"] and d["act"] == B2_ACT_RELU
        assert not d["a_mn"] and not d["b_mn"] and not d["c_small"]
    # backward, last hidden layer first: dX = dZ W (W consumed MN-major) then dW = dZ^T X (both MN-major)
    assert [(d["M"], d["N"], d["K"], d["a_mn"], d["b_mn"]) for d in bwd] == [
        (4096, 300, 300, 0, 1), (300, 300, 4096, 1, 1),
        (4096, 300, 300, 0, 1), (300, 300, 4096, 1, 1),
        (4096, 624, 300, 0, 1), (300, 624, 4096, 1, 1)]
    for k, d in enumerate(bwd):
        assert d["inline"] and not d["aux"]
        if k in (0, 2):     # a dgrad that feeds another layer applies THAT layer's ReLU backward and emits its bias gradient
            assert d["ybwd"] and d["act_bwd"] == B2_ACT_RELU and d["colsum"]
        else:
            assert not d["ybwd"] and not d["colsum"]


def test_aux_layout_adds_only_the_split_launches(recorder):
    run_chain("tf32x3", inline=False)
    names = [n for n, _ in recorder]
    assert names.count("b2_gemm_tc_ex") == 9 and "b2_prep_operand" not in names
    assert names.count("b2_split_tf32") == 4          # the input and the three tensor-core weights, once each
    g = [i for _, i in recorder if i is not None]
    assert all(d["aux"] and not d["inline"] for d in g)
    assert [d["c_small"] for d in g[:3]] == [True, True, False]       # a forward epilogue emits the next layer's small part


@pytest.mark.parametrize("mode", ["tf32", "bf16"])
def test_single_pass_modes(recorder, mode):
    run_chain(mode)
    g = [i for _, i in recorder if i is not None]
    assert len(g) == 9
    assert all(not d["inline"] and d["bf16"] == (mode == "bf16") for d in g)
    assert all(not d["aux"] for d in g)               # bf16 copies ARE the operands; 1xTF32 has none
    names = [n for n, _ in recorder]
    assert ("b2_to_bf16" in names) == (mode == "bf16") and "b2_split_tf32" not in names


def test_crossnet_v2_layer_is_one_gemm_forward_and_three_launches_backward(recorder):
    """x_next = x_i + x_0 * (x_i W^T + b) (cross_net.py:126-129): the cross itself is the GEMM's epilogue
    (mul = x_0, add = x_i, lin kept for the backward); backward = one g*x_0 pass + dgrad (+g in its epilogue) + wgrad."""
    F2.set_matmul_precision("tf32x3")
    torch.manual_seed(1)
    d = 624
    x0 = torch.randn(512, d, requires_grad=True)
    xi = torch.randn(512, d, requires_grad=True)
    w = torch.nn.Parameter(torch.randn(d, d) * 0.02)
    b = torch.nn.Parameter(torch.zeros(d))
    out = F2.cross_v2_layer(x0, xi, w, b)
    out.backward(torch.randn_like(out))
    names = [n for n, _ in recorder]
    assert names == ["b2_gemm_tc_ex", "b2_prep_operand", "b2_gemm_tc_ex", "b2_gemm_tc_ex"]
    fwd, dgrad, wgrad = [i for _, i in recorder if i is not None]
    assert fwd["mul"] and fwd["add"] and fwd["c_pre"] and fwd["bias"] and fwd["inline"] and not fwd["b_mn"]
    assert (dgrad["M"], dgrad["N"], dgrad["K"], dgrad["b_mn"], dgrad["add"]) == (512, d, d, 1, True)
    assert (wgrad["M"], wgrad["N"], wgrad["K"], wgrad["a_mn"], wgrad["b_mn"]) == (d, d, 512, 1, 1)

"""Where the dense layers send a Linear(K, 1), and the argument checks of the fp32 GEMM, the head backward and
the operand pass, without a GPU: `_lib.call` is replaced by a recorder (as in test_launch_sequence_dryrun.py), so
the autograd wrappers run on CPU tensors and the test sees which C-ABI entry points a step launches.  Numerics are
the `-m gpu` suite's (test_gpu_dense_sweep.py)."""
import ctypes
import os
import re

import pytest
import torch

from conftest import ROOT
from fuxictr_b200 import _lib, functional as F2
from fuxictr_b200._lib import B2_ACT_NONE, B2_ACT_RELU, B2_HEAD_MAX_K


@pytest.fixture
def recorder(monkeypatch):
    calls = []

    def fake_call(name, *a):
        info = None
        if name == "b2_gemm_f32":
            info = dict(M=a[8], N=a[9], K=a[10])
        elif name.startswith("b2_head_"):
            info = dict(M=a[4] if name != "b2_head_fwd" else a[3], K=a[5] if name != "b2_head_fwd" else a[4])
        calls.append((name, info))
        return 0

    monkeypatch.setattr(_lib, "call", fake_call)
    monkeypatch.setattr(F2, "_stream", lambda: None)
    monkeypatch.setattr(F2, "_require_cuda", lambda *t: None)
    yield calls
    F2.set_matmul_precision("fp32")


def names(calls):
    return [c[0] for c in calls]


def test_header_and_python_agree_on_the_head_bound():
    text = open(os.path.join(ROOT, "include", "fuxictr_b200.h")).read()
    assert int(re.search(r"#define B2_HEAD_MAX_K (\d+)", text).group(1)) == B2_HEAD_MAX_K
    # the backward stages 2 * K floats; with the kernel's static part that must fit sm_90's 227 KB per block
    assert 2 * 4 * B2_HEAD_MAX_K + 1024 <= 227 * 1024


@pytest.mark.parametrize("K", [B2_HEAD_MAX_K - 1, B2_HEAD_MAX_K, B2_HEAD_MAX_K + 1, 40000])
def test_linear_act_sends_a_width_one_layer_to_the_head_within_the_bound(recorder, K):
    x = torch.randn(3, K, requires_grad=True)
    w = torch.nn.Parameter(torch.randn(1, K))
    b = torch.nn.Parameter(torch.zeros(1))
    y = F2.linear_act(x, w, b, B2_ACT_NONE)
    y.backward(torch.ones_like(y))
    got = names(recorder)
    if K <= B2_HEAD_MAX_K:
        assert got == ["b2_head_fwd", "b2_head_bwd"], got
        assert recorder[0][1] == dict(M=3, K=K) and recorder[1][1] == dict(M=3, K=K)
    else:
        assert not any(n.startswith("b2_head") for n in got), got
        # forward, dgrad, wgrad on the SIMT GEMM; the bias gradient in the operand pass over dY
        gemms = [c[1] for c in recorder if c[0] == "b2_gemm_f32"]
        assert gemms == [dict(M=3, N=1, K=K), dict(M=3, N=K, K=1), dict(M=1, N=K, K=3)], gemms
        assert "b2_prep_operand" in got


@pytest.mark.parametrize("mode", ["tf32x3", "bf16"])
@pytest.mark.parametrize("K", [B2_HEAD_MAX_K, B2_HEAD_MAX_K + 4])
def test_mlp_chain_sends_a_width_one_layer_to_the_head_within_the_bound(recorder, mode, K):
    F2.set_matmul_precision(mode)
    x = torch.randn(4, 16, requires_grad=True)
    w0 = torch.nn.Parameter(torch.randn(K, 16) * 0.1)
    b0 = torch.nn.Parameter(torch.zeros(K))
    w1 = torch.nn.Parameter(torch.randn(1, K) * 0.01)
    b1 = torch.nn.Parameter(torch.zeros(1))
    y = F2.mlp_chain(x, [(w0, b0, B2_ACT_RELU), (w1, b1, B2_ACT_NONE)])
    assert type(y.grad_fn).__name__.startswith("_MLPChain")
    y.backward(torch.ones_like(y))
    got = names(recorder)
    if K <= B2_HEAD_MAX_K:
        assert y.grad_fn.kinds == ["tc", "head"]
        assert "b2_head_fwd" in got and "b2_head_bwd_ex" in got and "b2_gemm_f32" not in got, got
        assert [c[1]["K"] for c in recorder if c[0].startswith("b2_head")] == [K, K]
    else:
        assert y.grad_fn.kinds == ["tc", "simt"]
        assert not any(n.startswith("b2_head") for n in got), got
        gemms = [c[1] for c in recorder if c[0] == "b2_gemm_f32"]
        assert gemms == [dict(M=4, N=1, K=K), dict(M=4, N=K, K=1), dict(M=1, N=K, K=4)], gemms


def test_head_backward_refuses_k_above_the_bound():
    import __graft_entry__
    __graft_entry__.build()
    L = _lib.load()
    p = ctypes.c_void_p(4096)
    null = ctypes.c_void_p(0)
    args = lambda K: (p, p, null, p, 64, K, B2_ACT_NONE, p, p, p, B2_ACT_NONE, null, null, 0, null, 0, 0,
                      ctypes.c_float(0.0), null)
    for K in (B2_HEAD_MAX_K + 1, 1 << 20, 0):
        assert L.b2_head_bwd_ex(*args(K)) == -1
        assert b"B2_HEAD_MAX_K" in L.b2_last_error()
    with pytest.raises(_lib.B2Error, match="B2_HEAD_MAX_K"):
        _lib.call("b2_head_bwd", p, p, null, p, 64, B2_HEAD_MAX_K + 1, B2_ACT_NONE, p, p, p, null)


def test_prep_operand_refuses_a_transposed_small_part_without_the_transpose():
    """The kernel writes outT_small in its transpose pass, which runs only for outT."""
    import __graft_entry__
    __graft_entry__.build()
    p, null = ctypes.c_void_p(4096), ctypes.c_void_p(0)
    with pytest.raises(_lib.B2Error, match="outT_small needs outT"):
        _lib.call("b2_prep_operand", p, null, B2_ACT_NONE, 4, 4, p, null, null, p, null, null, 0, 0, 0.0, null)


def test_gemm_f32_refuses_epilogue_tensors_laid_out_unlike_out(recorder):
    M, N, K = 5, 6, 7
    a, b = torch.randn(M, K), torch.randn(K, N)
    out = torch.empty(M, N + 3)[:, :N]          # a column slice: leading dimension N + 3
    for bad in (torch.randn(M, N), torch.randn(M, N + 2)[:, :N], torch.randn(M, N + 3)[:, :N - 1]):
        with pytest.raises(ValueError, match="leading dimension"):
            F2.gemm_f32(a, b, out, mul=bad)
        with pytest.raises(ValueError, match="leading dimension"):
            F2.gemm_f32(a, b, out, add=bad)
    assert recorder == []
    ok = torch.randn(M, N + 3)[:, :N]
    F2.gemm_f32(a, b, out, mul=ok, add=ok)
    assert names(recorder) == ["b2_gemm_f32"]

"""The whole launch trace of the four dense autograd nodes (linear_act, mlp_chain, cross_v2_layer,
crossnet_mix_layer) without a GPU, against tests/golden/dense_launch_trace.json.  `_lib.call` is replaced by a
recorder (as in test_launch_sequence_dryrun.py), and every launch of a forward + backward is recorded in order:
the entry point, every scalar argument (for b2_gemm_tc_ex every scalar field of its descriptor) and, for every
pointer, the ordinal of that address's first appearance in the trace (0 for NULL), so that which operand is
which tensor (`add` is x_i, a wgrad's `b` is the forward's `a`, a saved auxiliary operand is the one the forward
made) is pinned too.  The golden file is written by tests/golden/make_dense_launch_trace.py; regenerate it only
with a change that means to launch something else.  Nothing is computed here: numerics are the `-m gpu` suite's."""
import contextlib
import ctypes
import json
import os

import pytest
import torch
from torch.utils._python_dispatch import TorchDispatchMode

from conftest import GOLDEN
from fuxictr_b200 import _lib, functional as F2
from fuxictr_b200._lib import B2_ACT_NONE, B2_ACT_RELU, B2_ACT_SIGMOID

GOLDEN_FILE = os.path.join(GOLDEN, "dense_launch_trace.json")
DESC_POINTERS = ("a", "b", "a_small", "b_small", "c", "c_small", "c_pre", "bias", "mul", "add", "ybwd", "colsum",
                 "drop_rng")
DESC_SCALARS = ("M", "N", "K", "lda", "ldb", "ldc", "ld_aux", "a_mn_major", "b_mn_major", "act", "act_bwd",
                "beta_accumulate", "elem_dtype", "flags", "drop_layer", "drop_thresh", "drop_scale")
assert set(DESC_POINTERS + DESC_SCALARS) == set(name for name, _ in _lib.b2_gemm_desc._fields_)

# precision name -> (set_matmul_precision, set_x3_inline)
PRECISIONS = {"fp32": ("fp32", True), "tf32": ("tf32", True), "tf32x3": ("tf32x3", True),
              "tf32x3_hbm_small": ("tf32x3", False), "bf16": ("bf16", True)}


class _KeepAlive(TorchDispatchMode):
    """Holds every tensor an operator returns, so that no address is handed out twice during one trace and an
    ordinal names one tensor whatever the allocator does with freed memory."""

    def __init__(self):
        super().__init__()
        self.kept = []

    def __torch_dispatch__(self, func, types, args=(), kwargs=None):
        out = func(*args, **(kwargs or {}))
        self.kept.append(out)
        return out


@contextlib.contextmanager
def recording():
    """Yields the list that `_lib.call` appends to: [entry point, argument, ...], pointers as ordinals."""
    trace, ordinals = [], {}

    def ordinal(address):
        if not address:
            return 0
        return ordinals.setdefault(address, len(ordinals) + 1)

    def fake_call(name, *args):
        rec = [name]
        if name == "b2_gemm_tc_ex":
            d = ctypes.cast(args[0], ctypes.POINTER(_lib.b2_gemm_desc)).contents
            rec += [ordinal(getattr(d, f)) for f in DESC_POINTERS] + [getattr(d, f) for f in DESC_SCALARS]
            args = args[1:]
        for a in args:
            rec.append(["p", ordinal(a.value)] if isinstance(a, ctypes.c_void_p) else a)
        trace.append(rec)
        return 0

    saved = _lib.call, F2._stream, F2._require_cuda, F2.get_matmul_precision(), F2._MATMUL["x3_inline"]
    _lib.call, F2._stream, F2._require_cuda = fake_call, (lambda: None), (lambda *t: None)
    F2._SMALL_CACHE.clear()
    try:
        with _KeepAlive():
            yield trace
    finally:
        _lib.call, F2._stream, F2._require_cuda = saved[:3]
        F2.set_matmul_precision(saved[3])
        F2.set_x3_inline(saved[4])
        F2._SMALL_CACHE.clear()


@pytest.fixture
def recorder():
    with recording() as trace:
        yield trace


# ------------------------------------------------------------------ the cases (shapes only: nothing is computed)
def tensor(*shape, grad=True):
    return torch.zeros(*shape, requires_grad=grad)


def param(*shape, grad=True):
    return torch.nn.Parameter(torch.zeros(*shape), requires_grad=grad)


def strided_param(n, k):
    """A weight whose rows are not contiguous: no tensor-core layer takes it, the SIMT GEMM does."""
    return torch.nn.Parameter(torch.zeros(n, k + 4)[:, :k])


def backward(y):
    assert y.grad_fn is not None
    y.backward(torch.zeros_like(y))


def linear(M, K, N, act=B2_ACT_RELU, bias=True, x_grad=True, w_grad=True, b_grad=True, lead=None, strided=False):
    def run():
        x = tensor(*((lead or ()) + (M, K)), grad=x_grad)
        w = strided_param(N, K) if strided else param(N, K, grad=w_grad)
        b = param(N, grad=b_grad) if bias else None
        backward(F2.linear_act(x, w, b, act))
    return run


def chain(dims, acts=None, drops=None, x_grad=True, frozen=(), frozen_bias=(), no_bias=(), strided=(), lead=None):
    L = len(dims) - 1
    acts = acts or [B2_ACT_RELU] * (L - 1) + [B2_ACT_NONE]
    drops = drops or [0.0] * L

    def run():
        x = tensor(*((lead or ()) + (64, dims[0])), grad=x_grad)
        layers = []
        for i in range(L):
            n, k = dims[i + 1], dims[i]
            w = strided_param(n, k) if i in strided else param(n, k, grad=i not in frozen)
            b = None if i in no_bias else param(n, grad=i not in frozen_bias)
            layers.append((w, b, acts[i], drops[i]) if drops[i] else (w, b, acts[i]))
        y = F2.mlp_chain(x, layers)
        assert type(y.grad_fn).__name__.startswith(("_MLPChain", "View"))
        backward(y)
    return run


def cross_v2(B, d, bias=True, x0_grad=True, xi_grad=True, w_grad=True, b_grad=True, strided=False):
    def run():
        x0, xi = tensor(B, d, grad=x0_grad), tensor(B, d, grad=xi_grad)
        w = strided_param(d, d) if strided else param(d, d, grad=w_grad)
        b = param(d, grad=b_grad) if bias else None
        backward(F2.cross_v2_layer(x0, xi, w, b))
    return run


def cross_mix(B, d, r, E, x0_grad=True, xl_grad=True, b_grad=True, gate_list=False):
    def run():
        x0, xl = tensor(B, d, grad=x0_grad), tensor(B, d, grad=xl_grad)
        U, V, C = param(E, d, r), param(E, d, r), param(E, r, r)
        gates = [param(1, d) for _ in range(E)] if gate_list else param(E, d)
        out = F2.crossnet_mix_layer(x0, xl, U, V, C, gates, param(d, 1, grad=b_grad))
        assert type(out.grad_fn).__name__ == "_CrossMixLayerBackward"
        backward(out)
    return run


R, S, NO = B2_ACT_RELU, B2_ACT_SIGMOID, B2_ACT_NONE
CASES = {
    # ---- linear_act: tensor-core shapes (in every mode but fp32)
    "linear/tc_relu_bias": linear(64, 48, 32),
    "linear/tc_sigmoid_bias": linear(64, 48, 32, act=S),
    "linear/tc_plain": linear(64, 48, 32, act=NO, bias=False),
    "linear/tc_bias_only": linear(64, 48, 32, act=NO),
    "linear/tc_act_only": linear(64, 48, 32, bias=False),
    "linear/tc_input_without_grad": linear(64, 48, 32, x_grad=False),
    "linear/tc_frozen_weight": linear(64, 48, 32, w_grad=False),
    "linear/tc_frozen_bias": linear(64, 48, 32, b_grad=False),
    "linear/tc_leading_dims": linear(16, 48, 32, lead=(4,)),
    # ---- linear_act: the SIMT GEMM (K % 4, N % 4, a dimension under 16, a strided weight)
    "linear/simt_k30_relu_bias": linear(64, 30, 32),
    "linear/simt_k30_plain": linear(64, 30, 32, act=NO, bias=False),
    "linear/simt_k30_bias_only": linear(64, 30, 32, act=NO),
    "linear/simt_k30_act_only": linear(64, 30, 32, bias=False),
    "linear/simt_n18": linear(64, 48, 18),
    "linear/simt_n8": linear(64, 48, 8),
    "linear/simt_k12": linear(64, 12, 32),
    "linear/simt_strided_weight": linear(64, 48, 32, strided=True),
    "linear/simt_input_without_grad": linear(64, 30, 32, x_grad=False),
    "linear/simt_frozen_weight": linear(64, 30, 32, w_grad=False),
    "linear/simt_frozen_bias_no_act": linear(64, 30, 32, act=NO, b_grad=False),
    # ---- linear_act: the N == 1 head
    "linear/head_plain": linear(64, 48, 1, act=NO, bias=False),
    "linear/head_bias": linear(64, 48, 1, act=NO),
    "linear/head_act": linear(64, 48, 1, act=S, bias=False),
    "linear/head_act_bias": linear(64, 48, 1, act=S),
    "linear/head_input_without_grad": linear(64, 48, 1, act=NO, x_grad=False),
    "linear/head_frozen_weight": linear(64, 48, 1, act=NO, w_grad=False),
    "linear/head_frozen_bias": linear(64, 48, 1, act=S, b_grad=False),
    # ---- mlp_chain
    "chain/tc3_head": chain([48, 32, 32, 32, 1]),
    "chain/tc3": chain([48, 32, 64, 32], acts=[R, S, R]),
    "chain/tc3_linear_top": chain([48, 32, 64, 32]),
    "chain/tc1": chain([48, 32], acts=[R]),
    "chain/head_only": chain([48, 1], acts=[S]),
    "chain/head_sigmoid": chain([48, 32, 1], acts=[R, S]),
    "chain/leading_dims": chain([48, 32, 1], lead=(2,)),
    "chain/no_bias_layers": chain([48, 32, 32, 1], no_bias=(0, 2)),
    "chain/linear_hidden_layer": chain([48, 32, 32, 1], acts=[R, NO, NO]),
    "chain/input_without_grad": chain([48, 32, 32, 1], x_grad=False),
    "chain/frozen_weight_middle": chain([48, 32, 32, 1], frozen=(1,)),
    "chain/frozen_weight_first_and_head": chain([48, 32, 32, 1], frozen=(0, 2)),
    "chain/frozen_biases": chain([48, 32, 32, 1], frozen_bias=(0, 1, 2)),
    "chain/simt_between_tc_strided": chain([48, 32, 32, 32], acts=[R, R, R], strided=(1,)),
    "chain/simt_between_tc_odd_width": chain([48, 32, 30, 32, 16], acts=[R, R, R, R]),
    "chain/simt_then_head": chain([30, 32, 1]),
    "chain/simt_narrow_then_head": chain([48, 8, 1]),
    "chain/all_simt": chain([30, 18, 10], acts=[R, S]),
    "chain/dropout_tc_layers": chain([48, 32, 32, 1], drops=[0.2, 0.3, 0.0]),
    "chain/dropout_tc_top": chain([48, 32, 32], acts=[R, R], drops=[0.0, 0.5]),
    "chain/dropout_tc_top_linear": chain([48, 32, 32], acts=[R, NO], drops=[0.1, 0.5]),
    "chain/dropout_head": chain([48, 32, 1], drops=[0.0, 0.25]),
    "chain/dropout_head_and_below": chain([48, 32, 1], acts=[R, S], drops=[0.2, 0.25]),
    "chain/dropout_head_only": chain([48, 1], acts=[NO], drops=[0.4]),
    "chain/dropout_simt_layer": chain([48, 32, 32, 32], acts=[R, R, R], drops=[0.1, 0.2, 0.3], strided=(1,)),
    "chain/dropout_simt_odd_width": chain([48, 30, 32, 1], drops=[0.2, 0.2, 0.0]),
    "chain/dropout_input_without_grad": chain([48, 32, 32, 1], drops=[0.2, 0.2, 0.0], x_grad=False),
    "chain/dropout_frozen_weight": chain([48, 32, 32, 1], drops=[0.2, 0.2, 0.0], frozen=(1,)),
    # ---- cross_v2_layer
    "cross_v2/tc": cross_v2(64, 48),
    "cross_v2/tc_no_bias": cross_v2(64, 48, bias=False),
    "cross_v2/tc_x0_without_grad": cross_v2(64, 48, x0_grad=False),
    "cross_v2/tc_xi_without_grad": cross_v2(64, 48, xi_grad=False),
    "cross_v2/tc_frozen_weight": cross_v2(64, 48, w_grad=False),
    "cross_v2/tc_frozen_bias": cross_v2(64, 48, b_grad=False),
    "cross_v2/simt_d30": cross_v2(64, 30),
    "cross_v2/simt_d12": cross_v2(64, 12),
    "cross_v2/simt_strided_weight": cross_v2(64, 48, strided=True),
    "cross_v2/simt_frozen_weight": cross_v2(64, 30, w_grad=False),
    "cross_v2/simt_x0_without_grad": cross_v2(64, 30, x0_grad=False, b_grad=False),
    # ---- crossnet_mix_layer
    "cross_mix/tc": cross_mix(64, 48, 8, 3),
    "cross_mix/tc_gate_list": cross_mix(64, 48, 8, 3, gate_list=True),
    "cross_mix/tc_x0_without_grad": cross_mix(64, 48, 8, 3, x0_grad=False),
    "cross_mix/tc_xl_without_grad": cross_mix(64, 48, 8, 3, xl_grad=False),
    "cross_mix/tc_frozen_bias": cross_mix(64, 48, 8, 3, b_grad=False),
    "cross_mix/simt_d30": cross_mix(37, 30, 4, 3),
    "cross_mix/simt_packed_under_16": cross_mix(37, 48, 4, 2),
    "cross_mix/simt_x0_without_grad": cross_mix(37, 30, 4, 3, x0_grad=False, b_grad=False),
}


def trace_case(case, precision):
    mode, inline = PRECISIONS[precision]
    with recording() as trace:
        F2.set_x3_inline(inline)
        F2.set_matmul_precision(mode)
        CASES[case]()
    return trace


def trace_all():
    """What the golden file holds.  Launches repeat across cases and precisions, so they are stored once:
    {"launches": [record, ...], "traces": {case: {precision: [index into launches, ...]}}}."""
    launches, index, traces = [], {}, {}
    for case in CASES:
        traces[case] = {}
        for precision in PRECISIONS:
            ids = []
            for rec in trace_case(case, precision):
                key = json.dumps(rec)
                if key not in index:
                    index[key] = len(launches)
                    launches.append(rec)
                ids.append(index[key])
            traces[case][precision] = ids
    return {"launches": launches, "traces": traces}


@pytest.fixture(scope="module")
def golden_traces():
    with open(GOLDEN_FILE) as fd:
        blob = json.load(fd)
    return {case: {p: [blob["launches"][i] for i in ids] for p, ids in per.items()}
            for case, per in blob["traces"].items()}


def test_golden_file_covers_exactly_these_cases(golden_traces):
    assert sorted(golden_traces) == sorted(CASES)
    assert all(sorted(per) == sorted(PRECISIONS) for per in golden_traces.values())


@pytest.mark.parametrize("precision", list(PRECISIONS))
@pytest.mark.parametrize("case", list(CASES))
def test_launch_trace_is_the_golden_one(golden_traces, case, precision):
    got = json.loads(json.dumps(trace_case(case, precision)))       # tuples and floats as the file holds them
    want = golden_traces[case][precision]
    assert [rec[0] for rec in got] == [rec[0] for rec in want]
    for k, (g, w) in enumerate(zip(got, want)):
        assert g == w, "launch %d (%s)" % (k, g[0])


def test_recorder_pins_aliasing_and_every_descriptor_field(recorder):
    """The recorder itself: in a CrossNetV2 layer `add` is x_i (the forward GEMM's `a`), `mul` is x_0, and the
    wgrad's `b` is that same x_i; a scalar argument is recorded as it is."""
    F2.set_matmul_precision("tf32")
    CASES["cross_v2/tc"]()
    names = [rec[0] for rec in recorder]
    assert names == ["b2_gemm_tc_ex", "b2_prep_operand", "b2_gemm_tc_ex", "b2_gemm_tc_ex"]
    fwd, prep, dgrad, wgrad = [dict(zip(DESC_POINTERS + DESC_SCALARS, rec[1:])) if rec[0] == "b2_gemm_tc_ex" else rec
                               for rec in recorder]
    assert fwd["a"] == fwd["add"] == wgrad["b"] and fwd["a"] != 0 and fwd["mul"] not in (0, fwd["a"])
    assert prep[2] == ["p", fwd["mul"]] and prep[3] == _lib.B2_PREP_MUL and prep[1] == ["p", dgrad["add"]]
    assert (wgrad["M"], wgrad["N"], wgrad["K"], wgrad["a_mn_major"], wgrad["b_mn_major"]) == (48, 48, 64, 1, 1)
    assert wgrad["a"] == dgrad["a"] == prep[6][1] and recorder[0][-1] is None

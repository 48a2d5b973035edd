"""The fp32 dense kernels against float64 at every branch of their launch plans: the SIMT GEMM (b2_gemm_f32),
the N = 1 head (b2_head_fwd, b2_head_bwd_ex), the operand pass over dY (b2_prep_operand), and the fp32-mode
MLP_Block that runs on them layer by layer.

The bar is test_gpu_kernel_sweep.py's: run a plain restatement in float32 (torch, on the CPU) and in float64, and
require for every output and gradient
    err(ours, fp64) <= max(1e-5, 3 * err(torch fp32, fp64))          (max-norm, relative)
Elementwise results and copies (activation backward, dropout mask, transposes, 3xTF32 small parts, an epilogue
applied to the plain product) are held bit-exact to a torch fp32 restatement in the kernel's operation order.
Every output buffer starts NaN and reaches past the (M, N) view; nothing outside the view may be written."""
import sys

import pytest
import torch
import torch.nn.functional as F

from conftest import rel_err, ROOT

sys.path.insert(0, ROOT)
pytestmark = pytest.mark.gpu

RTOL = 1e-5
NAN = float("nan")
DEV = torch.device("cuda:0")


@pytest.fixture(scope="module", autouse=True)
def _built():
    import __graft_entry__
    __graft_entry__.build()
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"


@pytest.fixture(autouse=True)
def _restore():
    yield
    from fuxictr_b200 import functional as F2
    F2.set_matmul_precision("fp32")


def bar(ours, ref32, ref64, what):
    e_ours, e_ref = rel_err(ours, ref64), rel_err(ref32, ref64)
    assert e_ours <= max(RTOL, 3 * e_ref), (what, e_ours, e_ref)


def tf32_small(x):
    """b2_tf32_small restated: x - big(x) rounded to tf32, to nearest with ties away from zero."""
    big = (x.view(torch.int32) & -8192).view(torch.float32)
    d = x - big
    return ((d.view(torch.int32) + 0x1000) & -8192).view(torch.float32)


def ulps(a, b):
    return int((a.view(torch.int32).long() - b.view(torch.int32).long()).abs().max())


def ceil_div(a, b):
    return -(-a // b)


def nan_mat(M, N, ld):
    """An (M, N) view of an NaN-filled (M, ld) buffer: (buffer, view)."""
    buf = torch.full((M, ld), NAN, device=DEV)
    return buf, buf[:, :N]


def nan_vec(n, pad=5):
    buf = torch.full((n + pad,), NAN, device=DEV)
    return buf, buf[:n]


# ================================================================== SIMT GEMM (b2_gemm_f32)
def gemm_plan(M, N, K, linear):
    """b2_gemm_f32's split-K plan restated: (number of K splits, k per split)."""
    tiles = ceil_div(M, 64) * ceil_div(N, 64)
    splits = 1
    if linear and tiles < 2 * 132 and K >= 128:
        splits = max(min(ceil_div(3 * 132, tiles), K // 64), 1)
    k_per = max(ceil_div(ceil_div(K, splits), 16) * 16, 16)
    return ceil_div(max(K, 1), k_per), k_per


def _pad8(n):
    return (n + 7) // 8 * 8


def operand(rows, cols, layout, gen):
    """A (rows, cols) CUDA view, NaN around it.  vec: 16-byte base, pitch % 4 == 0 (float4 loads); offset: the
    base one element past a 16-byte boundary; odd_ld: pitch % 4 != 0 (both scalar loads)."""
    if layout == "vec":
        buf = torch.full((rows, _pad8(cols)), NAN)
        view = buf[:, :cols]
    elif layout == "offset":
        buf = torch.full((rows, _pad8(cols + 1)), NAN)
        view = buf[:, 1:1 + cols]
    else:
        buf = torch.full((rows, _pad8(cols) + 1), NAN)
        view = buf[:, :cols]
    view.copy_(torch.randn(rows, cols, generator=gen))
    buf = buf.to(DEV)
    return buf[:, 1:1 + cols] if layout == "offset" else buf[:, :cols]


def gemm_operands(M, N, K, a_t, b_t, layout, gen):
    a = operand(*((K, M) if a_t else (M, K)), layout, gen)
    b = operand(*((N, K) if b_t else (K, N)), layout, gen)
    A = (a.t() if a_t else a).cpu()
    B = (b.t() if b_t else b).cpu()
    return a, b, A, B


def host_mat(M, N, gen, ld):
    """A random (M, N) matrix on the host and its copy in an NaN-padded device buffer of pitch ld."""
    h = torch.randn(M, N, generator=gen)
    buf, view = nan_mat(M, N, ld)
    view.copy_(h)
    return h, view


TEMPLATES = [(False, False), (False, True), (True, False), (True, True)]      # (a_t, b_t): the 4 load templates
# K < 128: no split, so every fused launch has the plain launch's accumulator.  M and N tails of the 64-wide tile,
# K tails of 16, K < 16, K = 1, M = 1, N = 1
EPI_SHAPES = [(1, 1, 1), (1, 70, 33), (70, 1, 17), (65, 129, 16), (130, 63, 15), (64, 64, 47), (129, 65, 127),
              (200, 77, 5)]
LAYOUTS = ["vec", "offset", "odd_ld"]


@pytest.mark.parametrize("layout", LAYOUTS)
@pytest.mark.parametrize("M,N,K", EPI_SHAPES)
@pytest.mark.parametrize("a_t,b_t", TEMPLATES)
def test_gemm_f32_epilogues(a_t, b_t, M, N, K, layout):
    from fuxictr_b200 import functional as F2
    from fuxictr_b200._lib import B2_ACT_RELU, B2_ACT_SIGMOID
    gen = torch.Generator().manual_seed(M * 1000 + N * 10 + K + 7 * a_t + 3 * b_t)
    a, b, A, B = gemm_operands(M, N, K, a_t, b_t, layout, gen)
    assert gemm_plan(M, N, K, True)[0] == 1
    ld = N + 3
    bias = torch.randn(N, generator=gen)
    mul, d_mul = host_mat(M, N, gen, ld)
    add, d_add = host_mat(M, N, gen, ld)
    c0, d_c0 = host_mat(M, N, gen, ld)
    bufs = {}

    def launch(name, out=None, **kw):
        if out is None:
            bufs[name] = nan_mat(M, N, ld)
            out = bufs[name][1]
        else:
            bufs[name] = (out._base, out)
        F2.gemm_f32(a, b, out, a_t=a_t, b_t=b_t, **kw)

    db = bias.to(DEV)
    launch("plain")
    launch("bias", bias=db)
    launch("relu", bias=db, act=B2_ACT_RELU)
    launch("sigmoid", bias=db, act=B2_ACT_SIGMOID)
    launch("mul_add", bias=db, mul=d_mul, add=d_add)
    launch("accumulate", out=d_c0, bias=db, accumulate=True)
    torch.cuda.synchronize()
    for name, (buf, view) in bufs.items():
        assert bool(torch.isnan(buf[:, N:]).all()), name
    got = {k: v[1].cpu() for k, v in bufs.items()}

    def epi(P, bias, mul, add, c0):
        t = P + bias
        return {"plain": P, "bias": t, "relu": torch.relu(t), "sigmoid": torch.sigmoid(t), "mul_add": t * mul + add,
                "accumulate": t + c0}
    r64 = epi(A.double() @ B.double(), bias.double(), mul.double(), add.double(), c0.double())
    r32 = epi(A @ B, bias, mul, add, c0)
    for k in got:
        bar(got[k], r32[k], r64[k], k)
    # the epilogue applied to the plain launch's accumulator, element for element
    lin = got["plain"]
    t = lin + bias
    assert torch.equal(got["bias"], t)
    assert torch.equal(got["relu"], torch.relu(t))
    assert torch.equal(got["accumulate"], t + c0)
    assert ulps(got["sigmoid"], 1.0 / (1.0 + torch.exp(-t.double()).float())) <= 4


# (M, N, K) with a linear epilogue: split over K when there are fewer than 264 tiles and K >= 128, into
# ceil(396 / tiles) splits capped at K / 64
SPLIT_CASES = {
    "k127_unsplit": (64, 64, 127, 1),
    "k128_cap_two": (64, 64, 128, 2),
    "cap_last_partial": (64, 64, 1000, 13),         # cap 15: 80 per split, the 13th holds 40
    "cap_equals_target": (40, 50, 25344, 396),      # one tile: 396 splits of 64
    "target_last_partial": (128, 128, 12700, 89),   # 4 tiles: 99 splits wanted, 144 per split, the 89th holds 28
    "tiles_263": (64, 263 * 64, 256, 2),
    "tiles_264_unsplit": (64, 264 * 64, 256, 1),
    "n_tail": (130, 67, 3001, 38),                  # 6 tiles: 66 wanted, cap 46, 80 per split, the 38th holds 41
}


@pytest.mark.parametrize("a_t,b_t", TEMPLATES)
@pytest.mark.parametrize("case", list(SPLIT_CASES))
def test_gemm_f32_split_k(case, a_t, b_t):
    """Split-K partial sums meet in C by float atomics: C is zeroed first (strided, ldc > N), the bias is added by
    the first split only, and with `accumulate` the partial sums land on the existing C."""
    from fuxictr_b200 import functional as F2
    M, N, K, splits = SPLIT_CASES[case]
    assert gemm_plan(M, N, K, True)[0] == splits
    layout = LAYOUTS[(2 * a_t + b_t) % 3]
    gen = torch.Generator().manual_seed(K + 2 * a_t + b_t)
    a, b, A, B = gemm_operands(M, N, K, a_t, b_t, layout, gen)
    ld = N + 5
    bias = torch.randn(N, generator=gen) * 4
    c0, d_c0 = host_mat(M, N, gen, ld)
    plain_buf, plain = nan_mat(M, N, ld)
    bias_buf, with_bias = nan_mat(M, N, ld)
    F2.gemm_f32(a, b, plain, a_t=a_t, b_t=b_t)
    F2.gemm_f32(a, b, with_bias, a_t=a_t, b_t=b_t, bias=bias.to(DEV))
    F2.gemm_f32(a, b, d_c0, a_t=a_t, b_t=b_t, bias=bias.to(DEV), accumulate=True)
    torch.cuda.synchronize()
    for buf in (plain_buf, with_bias._base, d_c0._base):
        assert bool(torch.isnan(buf[:, N:]).all())
    P64, P32 = A.double() @ B.double(), A @ B
    bar(plain, P32, P64, "plain")
    bar(with_bias, P32 + bias, P64 + bias.double(), "bias")
    bar(d_c0, P32 + bias + c0, P64 + bias.double() + c0.double(), "accumulate")


@pytest.mark.parametrize("act", ["relu", "sigmoid", "mul_add"])
def test_gemm_f32_nonlinear_epilogue_is_not_split(act):
    """Few tiles and a long K: a linear epilogue would be split; a non-linear one must run the whole K in one
    accumulator (a split one would apply the epilogue to partial sums, or meet them after it)."""
    from fuxictr_b200 import functional as F2
    M, N, K = 64, 70, 4000
    gen = torch.Generator().manual_seed(4000)
    a, b, A, B = gemm_operands(M, N, K, False, True, "vec", gen)
    ld = N + 2
    bias = torch.randn(N, generator=gen)
    mul, d_mul = host_mat(M, N, gen, ld)
    add, d_add = host_mat(M, N, gen, ld)
    buf, out = nan_mat(M, N, ld)
    kw = dict(mul=d_mul, add=d_add) if act == "mul_add" else dict(act=F2.ACT_CODE[act])
    F2.gemm_f32(a, b, out, b_t=True, bias=bias.to(DEV), **kw)
    torch.cuda.synchronize()
    assert bool(torch.isnan(buf[:, N:]).all())

    def ref(A, B, bias, mul, add):
        t = A @ B + bias
        return t * mul + add if act == "mul_add" else (torch.relu(t) if act == "relu" else torch.sigmoid(t))
    bar(out, ref(A, B, bias, mul, add), ref(A.double(), B.double(), bias.double(), mul.double(), add.double()), act)


def test_gemm_f32_cin_fallback_weight_gradient():
    """The CIN conv fallback's dW = dZ^T X: M = units, N = F * H (% 4 != 0), K = B * D."""
    from fuxictr_b200 import functional as F2
    units, FH, K = 16, 39 * 13, 4096 * 16
    assert gemm_plan(units, FH, K, True)[0] > 1
    gen = torch.Generator().manual_seed(65536)
    gz = torch.randn(K, units, generator=gen)
    x = torch.randn(K, FH, generator=gen)
    buf, gw = nan_mat(units, FH, FH + 1)
    F2.gemm_f32(gz.to(DEV), x.to(DEV), gw, a_t=True)
    torch.cuda.synchronize()
    assert bool(torch.isnan(buf[:, FH:]).all())
    bar(gw, gz.t() @ x, gz.t().double() @ x.double(), "gw")


# ================================================================== the N = 1 head (b2_head_fwd, b2_head_bwd_ex)
def kernel_mask(snap, layer, M, N, p):
    """keep * scale as b2_dropout_apply draws it (on ones); test_gpu_mlp_dropout.py holds that kernel to its
    restatement."""
    from fuxictr_b200 import functional as F2
    return F2.dropout_apply(torch.ones(M, N, device=DEV), snap, layer, p)


def _act(code, z):
    return torch.relu(z) if code == 1 else (torch.sigmoid(z) if code == 2 else z)


def head_case(M, K, act, bias=True, need_x=True, prev_act=0, small=False, gb_prev=False, p=None, zeroed=False,
              seed=0):
    """One forward and one backward of the head through the C-ABI, checked against float64."""
    from fuxictr_b200 import _lib, functional as F2
    from fuxictr_b200._lib import B2_ACT_RELU, B2_ACT_SIGMOID
    ptr = F2._ptr
    gen = torch.Generator().manual_seed(seed + 31 * K + M)
    # offsets keep gw, gb and gb_prev away from cancellation, where the order of the float atomics that form them
    # would decide the last digits
    x = torch.randn(M, K, generator=gen) + 0.5
    if prev_act == B2_ACT_RELU:         # x is the previous layer's activation output (and dropped output)
        x = torch.relu(x)
    elif prev_act == B2_ACT_SIGMOID:
        x = torch.sigmoid(x)
    drop = None
    if p is not None:
        snap = torch.tensor([0x5EED + K, 3 * M], dtype=torch.int64, device=DEV)
        mask = kernel_mask(snap, 1, M, K, p).cpu()
        thresh, scale = F2.dropout_consts(p)
        drop = (snap, 1, thresh, scale)
        x = x * mask
    w = torch.randn(K, generator=gen) / K ** 0.5
    b = torch.randn(1, generator=gen) * 0.1 if bias else None
    gy = torch.randn(M, generator=gen) + 0.5
    dx, dw, dgy = x.to(DEV), w.to(DEV), gy.to(DEV)
    db = b.to(DEV) if bias else None

    y_buf, y = nan_vec(M)
    _lib.call("b2_head_fwd", ptr(dx), ptr(dw), ptr(db), M, K, act, ptr(y), F2._stream())

    def grad_buf(n, want=True):
        if not want:
            return None, None
        buf, v = nan_vec(n)
        if zeroed:
            v.zero_()
        return buf, v
    gx_buf, gx = nan_vec(M * K) if need_x else (None, None)
    gs_buf, gs = nan_vec(M * K) if small else (None, None)
    gw_buf, gw = grad_buf(K)
    gb_buf, gb = grad_buf(1, bias)
    gp_buf, gp = grad_buf(K, gb_prev)
    d = drop if drop is not None else (None, 0, 0, 0.0)
    _lib.call("b2_head_bwd_ex", ptr(dx), ptr(dw), ptr(y), ptr(dgy), M, K, act, ptr(gx), ptr(gw), ptr(gb), prev_act,
              ptr(gs), ptr(gp), 1 if zeroed else 0, ptr(d[0]), d[1], d[2], d[3], F2._stream())
    torch.cuda.synchronize()
    for buf, v in ((y_buf, y), (gx_buf, gx), (gs_buf, gs), (gw_buf, gw), (gb_buf, gb), (gp_buf, gp)):
        if buf is not None:
            assert bool(torch.isnan(buf[v.numel():]).all())
    y = y.cpu()

    # ReLU: the restatement takes the kernel's branch (y > 0); any branch that differs from float64's must sit at
    # a pre-activation within rounding of 0
    z64 = x.double() @ w.double() + (b.double() if bias else 0.0)
    if act == B2_ACT_RELU:
        flip = (y > 0) != (z64 > 0)
        assert not bool(flip.any()) or float(z64[flip].abs().max()) <= RTOL * float(z64.abs().max())

    def ref(dt):
        X, W, GY = x.to(dt), w.to(dt), gy.to(dt)
        z = X @ W + (b.to(dt) if bias else 0.0)
        Y = _act(act, z)
        gz = GY
        if act == B2_ACT_RELU:
            gz = GY * (y > 0).to(dt)
        elif act == B2_ACT_SIGMOID:
            gz = GY * ((1 - Y) * Y)
        g = gz[:, None] * W[None, :]
        if drop is not None:
            g = g * mask.to(dt)
        if prev_act == B2_ACT_RELU:
            g = g * (X > 0).to(dt)
        elif prev_act == B2_ACT_SIGMOID:
            s = X / drop[3] if drop is not None else X
            g = g * ((1 - s) * s)
        return dict(y=Y, gw=gz @ X, gb=gz.sum().reshape(1), gx=g, gp=g.sum(0))
    r32, r64 = ref(torch.float32), ref(torch.float64)
    got = dict(y=y, gw=gw, gb=gb, gx=gx.view(M, K) if need_x else None, gp=gp)
    for k, v in got.items():
        if v is not None:
            bar(v, r32[k], r64[k], k)
    if need_x:
        # gx element for element in the kernel's order: gz * w, the mask, then prev_act'(x)
        gz = gy
        if act == B2_ACT_RELU:
            gz = torch.where(y > 0, gy, torch.zeros_like(gy))
        elif act == B2_ACT_SIGMOID:
            gz = gy * ((1.0 - y) * y)
        want = gz[:, None] * w[None, :]
        if drop is not None:
            want = torch.where(mask != 0, want * drop[3], torch.zeros_like(want))
        if prev_act == B2_ACT_RELU:
            want = torch.where(x > 0, want, torch.zeros_like(want))
        elif prev_act == B2_ACT_SIGMOID:
            s = x / drop[3] if drop is not None else x
            want = want * ((1.0 - s) * s)
        gx = gx.view(M, K).cpu()
        assert torch.equal(gx, want)
        if small:
            assert torch.equal(gs.view(M, K).cpu(), tf32_small(gx))


# The backward stages 2 * K floats in shared memory: past K = 6128 that and the kernel's 128 static bytes pass the
# default 48 KB per block (the launch needs the opt-in); B2_HEAD_MAX_K is the largest K it takes
def _head_ks():
    from fuxictr_b200._lib import B2_HEAD_MAX_K
    return [1, 31, 32, 255, 256, 257, 4096, 6128, 6129, 6144, 6145, B2_HEAD_MAX_K]


HEAD_MS = [5, 1001, 5000]     # below one CTA's 8 rows; 126 CTAs of 8 rows, the last holding 1; 264 CTAs of 19 rows


@pytest.mark.parametrize("act", [0, 1, 2])
@pytest.mark.parametrize("ki", range(12))
def test_head_sweep(ki, act):
    K = _head_ks()[ki]
    M = HEAD_MS[(ki + act) % 3]
    while M * K > 4_000_000:
        M //= 3
    head_case(M, K, act, bias=(ki + act) % 4 != 3, seed=ki)


@pytest.mark.parametrize("p", [None, 0.3])
@pytest.mark.parametrize("prev_act", [0, 1, 2])
@pytest.mark.parametrize("K", [257, 6144, "max"])
def test_head_fused_previous_layer(K, prev_act, p):
    """gx = prev_act'(x) * mask * gz * w (the previous layer's dZ), its 3xTF32 small part and its column sums
    (the previous layer's bias gradient)."""
    from fuxictr_b200._lib import B2_HEAD_MAX_K
    K = B2_HEAD_MAX_K if K == "max" else K
    M = {257: 5000, 6144: 300, B2_HEAD_MAX_K: 100}[K]
    head_case(M, K, 2, prev_act=prev_act, small=True, gb_prev=True, p=p, seed=prev_act)


def test_head_without_input_gradient():
    head_case(2500, 300, 1, need_x=False)


@pytest.mark.parametrize("prev_act", [0, 1])
def test_head_accumulates_into_zeroed_gradients(prev_act):
    head_case(5000, 257, 2, prev_act=prev_act, small=True, gb_prev=True, p=0.2, zeroed=True)


def test_head_weight_gradient_over_many_rows():
    # gw sums M rows: in a warp sequentially, over the CTA's 8 warps in shared memory, over 264 CTAs in global
    head_case(200_000, 32, 0)


# ================================================================== the operand pass (b2_prep_operand)
PREP_ACTS = ["none", "relu", "sigmoid", "mul", "drop_relu", "drop_sigmoid"]
OUTPUTS = ["out", "out_small", "outT", "outT_small", "colsum"]


def prep_case(R, C, act, want, seed=0):
    from fuxictr_b200 import _lib, functional as F2
    from fuxictr_b200._lib import B2_ACT_NONE, B2_ACT_RELU, B2_ACT_SIGMOID, B2_PREP_MUL
    ptr = F2._ptr
    gen = torch.Generator().manual_seed(seed + R * 1009 + C)
    x = torch.randn(R, C, generator=gen) + 0.5      # column sums away from cancellation (see head_case)
    pre = torch.randn(R, C, generator=gen)
    code = {"none": B2_ACT_NONE, "relu": B2_ACT_RELU, "sigmoid": B2_ACT_SIGMOID, "mul": B2_PREP_MUL,
            "drop_relu": B2_ACT_RELU, "drop_sigmoid": B2_ACT_SIGMOID}[act]
    y = None if act == "none" else (torch.relu(pre) if code == B2_ACT_RELU else
                                    (torch.sigmoid(pre) if code == B2_ACT_SIGMOID else pre))
    drop = None
    if act.startswith("drop"):
        snap = torch.tensor([0xD20 + R, C], dtype=torch.int64, device=DEV)
        mask = kernel_mask(snap, 2, R, C, 0.25).cpu()
        thresh, scale = F2.dropout_consts(0.25)
        drop = (snap, 2, thresh, scale)
        y = y * mask                    # y is the layer's dropped output
    bufs = {}
    for name in OUTPUTS:
        if name in want:
            bufs[name] = nan_vec(C if name == "colsum" else R * C)
    d = drop if drop is not None else (None, 0, 0, 0.0)
    view = lambda name: bufs[name][1] if name in bufs else None
    dx, dy = x.to(DEV), (y.to(DEV) if y is not None else None)

    def launch():
        _lib.call("b2_prep_operand", ptr(dx), ptr(dy), code, R, C, ptr(view("out")), ptr(view("out_small")),
                  ptr(view("outT")), ptr(view("outT_small")), ptr(view("colsum")), ptr(d[0]), d[1], d[2], d[3],
                  F2._stream())
    if "outT_small" in want and "outT" not in want:     # refused before anything is written
        with pytest.raises(_lib.B2Error, match="outT_small needs outT"):
            launch()
        torch.cuda.synchronize()
        assert all(bool(torch.isnan(buf).all()) for buf, _ in bufs.values())
        return
    launch()
    torch.cuda.synchronize()
    for name, (buf, v) in bufs.items():
        assert bool(torch.isnan(buf[v.numel():]).all()), name
    # the kernel's order: the mask, then the activation backward with y (sigmoid: s = y / scale under dropout)
    v = x
    if drop is not None:
        v = torch.where(mask != 0, x * drop[3], torch.zeros_like(x))
    if code == B2_ACT_RELU:
        v = torch.where(y > 0, v, torch.zeros_like(v))
    elif code == B2_ACT_SIGMOID:
        s = y / drop[3] if drop is not None else y
        v = v * ((1.0 - s) * s)
    elif code == B2_PREP_MUL:
        v = v * y
    want_of = {"out": v, "out_small": tf32_small(v), "outT": v.t().contiguous(),
               "outT_small": tf32_small(v).t().contiguous()}
    for name in OUTPUTS[:4]:
        if name in bufs:
            assert torch.equal(view(name).cpu().view(want_of[name].shape), want_of[name]), name
    if "colsum" in bufs:
        bar(view("colsum"), v.sum(0), v.double().sum(0), "colsum")


@pytest.mark.parametrize("act", PREP_ACTS)
@pytest.mark.parametrize("C", [1, 31, 32, 33, 1000])
@pytest.mark.parametrize("R", [1, 31, 32, 33, 1000])
def test_prep_operand_sweep(R, C, act):
    prep_case(R, C, act, OUTPUTS)


@pytest.mark.parametrize("act", PREP_ACTS)
def test_prep_operand_every_subset_of_outputs(act):
    for bits in range(32):
        prep_case(70, 45, act, [o for i, o in enumerate(OUTPUTS) if bits >> i & 1], seed=bits)


# ================================================================== fp32-mode MLP_Block, layer by layer
def _restated(mods, gates, zs):
    """The reference's Sequential of Linear / ReLU / Sigmoid; ReLU takes the kernel's branch (gates)."""
    def fn(x, *params):
        h, ps, gs = x, iter(params), iter(gates)
        for m in mods:
            if isinstance(m, torch.nn.Linear):
                w = next(ps)
                h = F.linear(h, w, next(ps) if m.bias is not None else None)
            elif isinstance(m, torch.nn.ReLU):
                zs.append(h.detach())
                h = h * next(gs).to(h.dtype)
            elif isinstance(m, torch.nn.Sigmoid):
                h = torch.sigmoid(h)
        return h
    return fn


def _check_relu_flips(gates, zs):
    for g, z in zip(gates, zs):
        flip = g != (z > 0)
        if bool(flip.any()):
            assert float(z[flip].abs().max()) <= RTOL * float(z.abs().max()), int(flip.sum())


def _grads(fn, inputs, gout, dtype):
    xs = [t.detach().to(dtype).requires_grad_(True) for t in inputs]
    y = fn(*xs)
    y.backward(gout.to(dtype))
    return y.detach(), [t.grad for t in xs]


MLP_CASES = {   # input shape, hidden units, output activation, use_bias
    "c2": ((4096, 624), [300, 300, 300], None, True),
    "sigmoid_head": ((1000, 100), [64], "Sigmoid", True),
    "narrow": ((513, 37), [13, 5, 2], None, True),
    "no_bias": ((700, 96), [50, 20], None, False),
    "input_3d": ((64, 7, 40), [24, 8], "Sigmoid", True),
    "head_k6140": ((2000, 6140), [], None, True),           # an xDeepFM / DCNv2 fc over F * D + hidden inputs
    "head_above_bound": ((200, "max+1"), [], "Sigmoid", True),
}


@pytest.mark.parametrize("case", list(MLP_CASES))
def test_fp32_mlp_block_matches_float64(case, monkeypatch):
    from fuxictr_b200 import layers, functional as F2
    from fuxictr_b200._lib import B2_ACT_RELU, B2_HEAD_MAX_K
    shape, hidden, out_act, use_bias = MLP_CASES[case]
    shape = tuple(B2_HEAD_MAX_K + 1 if s == "max+1" else s for s in shape)
    F2.set_matmul_precision("fp32")
    torch.manual_seed(len(case))
    block = layers.MLP_Block(shape[-1], hidden, "ReLU", output_dim=1, output_activation=out_act,
                             use_bias=use_bias)
    with torch.no_grad():
        for prm in block.parameters():
            if prm.dim() == 1:
                prm.normal_(0, 0.1)
    params = [prm.detach().clone() for prm in block.parameters()]
    gen = torch.Generator().manual_seed(len(case) + 1)
    x = torch.randn(*shape, generator=gen)
    relu_outs = []
    linear_act = F2.linear_act

    def recording(x, w, b=None, act=0):
        y = linear_act(x, w, b, act)
        if act == B2_ACT_RELU:
            relu_outs.append(y.detach().cpu())
        return y
    monkeypatch.setattr(F2, "linear_act", recording)
    block = block.to(DEV)
    xg = x.to(DEV).requires_grad_(True)
    y = block(xg)
    gout = torch.randn(y.shape, generator=gen) + 0.5       # the head's bias gradient away from cancellation
    y.backward(gout.to(DEV))
    gates = [h > 0 for h in relu_outs]
    assert len(gates) == len(hidden)
    zs = []
    fn = _restated(list(block.mlp), gates, zs)
    y64, g64 = _grads(fn, [x] + params, gout, torch.float64)
    _check_relu_flips(gates, zs)
    y32, g32 = _grads(fn, [x] + params, gout, torch.float32)
    names = ["x"] + [k for k, _ in block.named_parameters()]
    ours = [xg.grad] + [prm.grad for prm in block.parameters()]
    bar(y, y32, y64, "y")
    for name, o, a, b in zip(names, ours, g32, g64):
        bar(o, a, b, name)


def test_tf32x3_chain_with_a_simt_layer_and_dropout_before_the_head():
    """A tensor-core layer, then a SIMT layer (N = 18: not TMA-aligned) with dropout, then the head over K = 18:
    the head's backward regenerates the SIMT layer's mask and folds its ReLU backward and bias gradient."""
    from fuxictr_b200 import functional as F2
    from fuxictr_b200._lib import B2_ACT_NONE, B2_ACT_RELU
    F2.set_matmul_precision("tf32x3")
    dims, M, p = (64, 32, 18, 1), 777, 0.25
    gen = torch.Generator().manual_seed(18)
    x = torch.randn(M, dims[0], generator=gen)
    params = []
    for i in range(3):
        params += [torch.randn(dims[i + 1], dims[i], generator=gen) / dims[i] ** 0.5,
                   torch.randn(dims[i + 1], generator=gen) * 0.1]
    gout = torch.randn(M, 1, generator=gen) + 0.5
    xg = x.to(DEV).requires_grad_(True)
    pg = [torch.nn.Parameter(t.to(DEV)) for t in params]
    layers = [(pg[0], pg[1], B2_ACT_RELU), (pg[2], pg[3], B2_ACT_RELU, p), (pg[4], pg[5], B2_ACT_NONE)]
    state = F2.dropout_state(DEV)
    state.copy_(torch.tensor([0x5EED18, 0], dtype=torch.int64, device=DEV))
    snap = state.clone()                    # the forward snapshots exactly this
    y = F2.mlp_chain(xg, layers)
    assert y.grad_fn.kinds == ["tc", "simt", "head"]
    hs = y.grad_fn.saved_tensors
    y.backward(gout.to(DEV))
    keep = (kernel_mask(snap, 0, M, dims[2], p) != 0).cpu()
    gates = [(hs[1] > 0).cpu(), (hs[2] > 0).cpu() | ~keep]

    def fn(x, w0, b0, w1, b1, w2, b2, zs=None):
        z0 = F.linear(x, w0, b0)
        z1 = F.linear(z0 * gates[0].to(x.dtype), w1, b1)
        if zs is not None:
            zs += [z0.detach(), z1.detach()]
        h1 = z1 * gates[1].to(x.dtype) * (keep.to(x.dtype) * (1.0 / (1.0 - p)))
        return F.linear(h1, w2, b2)
    zs = []
    y64, g64 = _grads(lambda *t: fn(*t, zs=zs), [x] + params, gout, torch.float64)
    _check_relu_flips([gates[0], gates[1] & keep], [zs[0], torch.where(keep, zs[1], torch.full_like(zs[1], -1.0))])
    y32, g32 = _grads(fn, [x] + params, gout, torch.float32)
    bar(y, y32, y64, "y")
    for name, o, a, b in zip(["x", "W0", "b0", "W1", "b1", "W2", "b2"], [xg.grad] + [t.grad for t in pg], g32, g64):
        bar(o, a, b, name)

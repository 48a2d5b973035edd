"""The fused epilogue of the wgmma GEMM, element for element.

K stays below 16 k-blocks, so a plain linear GEMM is not split over K and has the same accumulator as the fused
launches of the same operands.  Each fused output must then equal, bit for bit, a torch fp32 restatement of the
epilogue applied to that plain output (sigmoid within 2 ulp: expf).  Column sums and split-K partials are float
atomics and match to reassociation tolerance.  The shapes make the planner pick each tile width and have M tails;
the layouts give 16-byte segments throughout, an N tail (N % 4 != 0) that ends in a partial segment, and an odd
leading dimension of C that sends every segment element by element."""
import pytest
import torch

from conftest import close

pytestmark = pytest.mark.gpu

MODES = ["tf32", "tf32x3", "tf32x3_aux", "bf16"]
MAJORS = [(False, False), (False, True), (True, True), (True, False)]
SHAPES = [(300, 72, 200), (3000, 200, 200), (2000, 520, 200)]     # bn = 32, 64, 128 (3xTF32: 64)
LAYOUTS = ["aligned", "n_tail", "odd_ldc"]


@pytest.fixture(scope="module", autouse=True)
def _built():
    import __graft_entry__
    __graft_entry__.build()
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"


@pytest.fixture
def precision():
    from fuxictr_b200 import functional as F2

    def set_mode(mode):
        F2.set_x3_inline(mode != "tf32x3_aux")
        F2.set_matmul_precision("tf32x3" if mode == "tf32x3_aux" else mode)
    yield set_mode
    F2.set_matmul_precision("fp32")
    F2.set_x3_inline(True)


def _pad8(n):
    return (n + 7) // 8 * 8


def operand(rows, K, mn, mode, gen):
    """A (rows, K) operand as the GEMM reads it (MN-major: stored (K, rows)), inside a buffer whose row pitch is a
    multiple of 8 elements, and its auxiliary operand for the mode."""
    from fuxictr_b200 import functional as F2
    shape = (K, rows) if mn else (rows, K)
    buf = torch.randn(shape[0], _pad8(shape[1]), generator=gen).cuda()
    view = buf[:, :shape[1]]
    if mode == "tf32x3_aux":        # the small part shares the operand's layout
        return view, F2.make_aux(buf)[:, :shape[1]]
    return view, F2.make_aux(view)


def tf32_small(x):
    """b2_tf32_small restated: x - big(x) rounded to tf32, to nearest with ties away from zero."""
    big = (x.view(torch.int32) & -8192).view(torch.float32)
    d = x - big
    return ((d.view(torch.int32) + 0x1000) & -8192).view(torch.float32)


def ulps(a, b):
    return int((a.view(torch.int32).long() - b.view(torch.int32).long()).abs().max())


@pytest.mark.parametrize("layout", LAYOUTS)
@pytest.mark.parametrize("M,N,K", SHAPES)
@pytest.mark.parametrize("a_mn,b_mn", MAJORS)
@pytest.mark.parametrize("mode", MODES)
def test_fused_epilogue_equals_its_fp32_restatement(M, N, K, a_mn, b_mn, layout, mode, precision):
    from fuxictr_b200 import functional as F2
    from fuxictr_b200._lib import B2_ACT_RELU, B2_ACT_SIGMOID
    precision(mode)
    if layout == "n_tail":
        N -= 2
    ld = N + 1 if layout == "odd_ldc" else _pad8(N)
    gen = torch.Generator().manual_seed(M + N + 2 * a_mn + b_mn)
    a, a_aux = operand(M, K, a_mn, mode, gen)
    b, b_aux = operand(N, K, b_mn, mode, gen)
    kw = dict(a_mn=a_mn, b_mn=b_mn, a_small=a_aux, b_small=b_aux)
    f32 = mode != "bf16"

    def mat(src=None):
        """(M, N) in a buffer of row pitch ld, NaN outside the view."""
        buf = torch.full((M, ld), float("nan"), device="cuda")
        if src is not None:
            buf[:, :N] = src.cuda()
        return buf, buf[:, :N]

    def small_out():
        if f32:
            return mat()
        buf = torch.full((M, _pad8(N)), float("nan"), device="cuda", dtype=torch.bfloat16)
        return buf, buf[:, :N]

    def launch(**extra):
        buf, out = mat(extra.pop("init", None))
        F2.gemm_ex(a, b, out, **kw, **extra)
        return buf, out

    def want_small(t):
        return tf32_small(t) if f32 else t.bfloat16()

    lin = torch.empty(M, N, device="cuda")
    F2.gemm_ex(a, b, lin, **kw)
    bias = torch.randn(N, generator=gen)
    mul, add = torch.randn(M, N, generator=gen), torch.randn(M, N, generator=gen)
    y_relu, y_sig = torch.rand(M, N, generator=gen) - 0.5, torch.rand(M, N, generator=gen)
    c0 = torch.randn(M, N, generator=gen)
    _, m_mul = mat(mul)
    _, m_add = mat(add)
    _, m_yr = mat(y_relu)
    _, m_ys = mat(y_sig)
    pre_buf, pre = mat()
    sr_buf, sr = small_out()
    ss_buf, ss = small_out()
    cs_r = torch.full((N,), float("nan"), device="cuda")
    cs_s = torch.full((N,), float("nan"), device="cuda")
    outs = {
        "bias_relu": launch(bias=bias.cuda(), act=B2_ACT_RELU, out_small=sr),
        "bias_sigmoid": launch(bias=bias.cuda(), act=B2_ACT_SIGMOID, out_small=ss),
        "mul_add_pre": launch(bias=bias.cuda(), mul=m_mul, add=m_add, out_pre=pre),
        "ybwd_relu": launch(ybwd=m_yr, act_bwd=B2_ACT_RELU, colsum=cs_r),
        "ybwd_sigmoid": launch(ybwd=m_ys, act_bwd=B2_ACT_SIGMOID, colsum=cs_s),
        "beta": launch(bias=bias.cuda(), accumulate=True, init=c0),
    }
    torch.cuda.synchronize()
    lin = lin.cpu()
    t = lin + bias
    got = {k: v[1].cpu() for k, v in outs.items()}
    for k, (buf, _) in outs.items():        # nothing written outside (M, N)
        assert torch.isnan(buf[:, N:]).all(), k
    for buf in (pre_buf, sr_buf, ss_buf):
        assert torch.isnan(buf[:, N:].float()).all()

    assert torch.equal(got["bias_relu"], torch.relu(t))
    assert torch.equal(sr.cpu(), want_small(got["bias_relu"]))
    assert torch.equal(pre.cpu(), t)
    assert torch.equal(got["mul_add_pre"], t * mul + add)
    want = torch.where(y_relu > 0, lin, torch.zeros_like(lin))
    assert torch.equal(got["ybwd_relu"], want)
    want = lin * ((1.0 - y_sig) * y_sig)
    assert torch.equal(got["ybwd_sigmoid"], want)
    for out, cs in ((got["ybwd_relu"], cs_r), (got["ybwd_sigmoid"], cs_s)):
        o = out.double()
        assert close(cs, o.sum(0), 1e-5, atol=1e-5 * float(o.abs().sum(0).max()))
    assert torch.equal(got["beta"], t + c0)
    # expf is within 2 ulp of exp; against a correctly rounded exp, the sum and the quotient may each round the
    # other way as well
    e = torch.exp(-t.double()).float()
    assert ulps(got["bias_sigmoid"], 1.0 / (1.0 + e)) <= 4
    assert torch.equal(ss.cpu(), want_small(got["bias_sigmoid"]))


@pytest.mark.parametrize("layout", LAYOUTS)
@pytest.mark.parametrize("a_mn,b_mn", MAJORS)
@pytest.mark.parametrize("mode", MODES)
def test_split_k_equals_its_partial_gemms(a_mn, b_mn, layout, mode, precision):
    """Few tiles and a long K: the planner splits a plain linear GEMM over K and adds the partial tiles (bias in the
    first) with vector or scalar reductions.  Each partial equals an unsplit GEMM over the same k-blocks (out_pre
    makes it non-linear, so it is not split); the split output is their sum up to fp32 reassociation.  (A whole
    unsplit GEMM is no reference in the single-pass modes: the tensor cores add its k-blocks in their accumulator.)"""
    from fuxictr_b200 import functional as F2
    from test_abi import _plan
    precision(mode)
    M, N, K = 136, 72, 3000
    if layout == "n_tail":
        N -= 2
    ld = N + 1 if layout == "odd_ldc" else _pad8(N)
    plan = _plan(M, N, K, a_mn, b_mn, mode=mode)
    assert plan.splits > 1
    chunk = plan.kb_per_split * (64 if mode == "bf16" else 32)
    gen = torch.Generator().manual_seed(11 + 2 * a_mn + b_mn)
    a, a_aux = operand(M, K, a_mn, mode, gen)
    b, b_aux = operand(N, K, b_mn, mode, gen)
    bias = torch.randn(N, generator=gen).cuda()
    buf = torch.full((M, ld), float("nan"), device="cuda")
    out = buf[:, :N]
    out.zero_()
    F2.gemm_ex(a, b, out, a_mn=a_mn, b_mn=b_mn, a_small=a_aux, b_small=b_aux, bias=bias, out_is_zero=True)
    ref = torch.zeros(M, N, dtype=torch.float64)
    for k0 in range(0, K, chunk):
        ks = (lambda t: None if t is None else t[k0:k0 + chunk]) if a_mn else \
             (lambda t: None if t is None else t[:, k0:k0 + chunk])
        kt = (lambda t: None if t is None else t[k0:k0 + chunk]) if b_mn else \
             (lambda t: None if t is None else t[:, k0:k0 + chunk])
        part, pre = torch.empty(M, N, device="cuda"), torch.empty(M, N, device="cuda")
        F2.gemm_ex(ks(a), kt(b), part, a_mn=a_mn, b_mn=b_mn, a_small=ks(a_aux), b_small=kt(b_aux),
                   bias=bias if k0 == 0 else None, out_pre=pre)
        ref += part.cpu().double()
    torch.cuda.synchronize()
    assert torch.isnan(buf[:, N:]).all()
    assert close(out, ref, 1e-6)

"""The wgmma GEMM with its ring sized per operand majors and, in 3xTF32, a K-major A split in registers.

Every output element must not depend on how the output is tiled: one GEMM equals, bit for bit, the same GEMM
computed as separate column slices of B (each slice starts a new tile grid, and its bn may differ).  The fused
epilogues stay within the per-mode bars against float64.  Shapes have tails in M, N and K."""
import pytest
import torch

from conftest import close

pytestmark = pytest.mark.gpu

MODES = ["tf32", "tf32x3", "bf16"]
MAJORS = [(False, False), (False, True), (True, True), (True, False)]
# relative bar against float64 per mode (bf16: against the bf16-rounded operands)
TOL = {"tf32": 3e-3, "tf32x3": 1e-5, "bf16": 3e-5}


@pytest.fixture(scope="module", autouse=True)
def _built():
    import __graft_entry__
    __graft_entry__.build()
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"


@pytest.fixture
def precision():
    from fuxictr_b200 import functional as F2

    def set_mode(mode):
        F2.set_x3_inline(True)
        F2.set_matmul_precision(mode)
    yield set_mode
    F2.set_matmul_precision("fp32")
    F2.set_x3_inline(True)


def operands(M, N, K, a_mn, b_mn, seed):
    """A (M, K) and B (N, K) on the host, and their device copies as they lie in memory (MN-major: transposed)."""
    gen = torch.Generator().manual_seed(seed)
    a, b = torch.randn(M, K, generator=gen), torch.randn(N, K, generator=gen)
    a_dev = (a.t().contiguous() if a_mn else a).cuda()
    b_dev = (b.t().contiguous() if b_mn else b).cuda()
    return a, b, a_dev, b_dev


def reference(a, b, mode):
    if mode == "bf16":
        a, b = a.bfloat16(), b.bfloat16()
    return a.double() @ b.double().t()


@pytest.mark.parametrize("M,N,K", [(328, 200, 100), (4096, 300, 300)])
@pytest.mark.parametrize("a_mn,b_mn", MAJORS)
@pytest.mark.parametrize("mode", MODES)
def test_gemm_equals_its_column_slices_bitwise(M, N, K, a_mn, b_mn, mode, precision):
    from fuxictr_b200 import functional as F2
    precision(mode)
    a, b, a_dev, b_dev = operands(M, N, K, a_mn, b_mn, M + 3 * N + 7 * K + a_mn + 2 * b_mn)
    a_aux, b_aux = F2.make_aux(a_dev), F2.make_aux(b_dev)
    bias = torch.randn(N, generator=torch.Generator().manual_seed(N)).cuda()
    # out_pre (acc + bias) makes the epilogue non-linear, so no launch is split over K
    out, pre = torch.full((M, N), float("nan"), device="cuda"), torch.full((M, N), float("nan"), device="cuda")
    F2.gemm_ex(a_dev, b_dev, out, a_mn=a_mn, b_mn=b_mn, a_small=a_aux, b_small=b_aux, bias=bias, out_pre=pre)
    sl_out, sl_pre = torch.full_like(out, float("nan")), torch.full_like(pre, float("nan"))
    edges = [0, 72, 136, N]                       # multiples of 8: 16-byte aligned slices in every mode
    for n0, n1 in zip(edges[:-1], edges[1:]):
        cols = (lambda t: t[:, n0:n1]) if b_mn else (lambda t: t[n0:n1])
        F2.gemm_ex(a_dev, cols(b_dev), sl_out[:, n0:n1], a_mn=a_mn, b_mn=b_mn, a_small=a_aux,
                   b_small=None if b_aux is None else cols(b_aux), bias=bias[n0:n1], out_pre=sl_pre[:, n0:n1])
    torch.cuda.synchronize()
    assert torch.equal(out, sl_out) and torch.equal(pre, sl_pre)
    want = reference(a, b, mode) + bias.cpu().double()
    assert close(pre, want, TOL[mode])


@pytest.mark.parametrize("epilogue", ["bias_relu", "ybwd_colsum", "pre_mul_add", "split_k"])
@pytest.mark.parametrize("a_mn", [False, True])
@pytest.mark.parametrize("mode", MODES)
def test_fused_epilogues_vs_fp64(epilogue, a_mn, mode, precision):
    from fuxictr_b200 import functional as F2
    from fuxictr_b200._lib import B2_ACT_RELU
    precision(mode)
    M, N, K = (136, 72, 4000) if epilogue == "split_k" else (712, 200, 164)
    b_mn = epilogue == "ybwd_colsum"              # the dgrad layout: W consumed MN-major
    a, b, a_dev, b_dev = operands(M, N, K, a_mn, b_mn, 17 + M + a_mn)
    gen = torch.Generator().manual_seed(5)
    z = reference(a, b, mode)
    kw = dict(a_mn=a_mn, b_mn=b_mn, a_small=F2.make_aux(a_dev), b_small=F2.make_aux(b_dev))
    out = torch.full((M, N), float("nan"), device="cuda")
    if epilogue == "bias_relu":
        bias = torch.randn(N, generator=gen)
        F2.gemm_ex(a_dev, b_dev, out, bias=bias.cuda(), act=B2_ACT_RELU, **kw)
        assert close(out, torch.relu(z + bias.double()), TOL[mode])
    elif epilogue == "ybwd_colsum":
        y = torch.rand(M, N, generator=gen) - 0.5
        colsum = torch.full((N,), float("nan"), device="cuda")
        F2.gemm_ex(a_dev, b_dev, out, ybwd=y.cuda(), act_bwd=B2_ACT_RELU, colsum=colsum, **kw)
        want = torch.where(y.double() > 0, z, torch.zeros_like(z))
        assert close(out, want, TOL[mode])
        assert close(colsum, want.sum(0), TOL[mode], atol=TOL[mode] * float(want.abs().sum(0).max()))
    elif epilogue == "pre_mul_add":
        bias, mul, add = torch.randn(N, generator=gen), torch.randn(M, N, generator=gen), torch.randn(M, N, generator=gen)
        pre = torch.full((M, N), float("nan"), device="cuda")
        F2.gemm_ex(a_dev, b_dev, out, bias=bias.cuda(), mul=mul.cuda(), add=add.cuda(), out_pre=pre, **kw)
        lin = z + bias.double()
        assert close(pre, lin, TOL[mode])
        assert close(out, add.double() + mul.double() * lin, TOL[mode])
    else:                                         # few tiles and a long K: the planner splits over K
        out.zero_()
        F2.gemm_ex(a_dev, b_dev, out, out_is_zero=True, **kw)
        assert close(out, z, TOL[mode])

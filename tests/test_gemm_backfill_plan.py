"""Host-only: the launch plan of a B2_GEMM_BACKFILL GEMM (a wgrad launched beside the dgrad chain) keeps the
tile width of the plain plan and splits a linear epilogue over K into CTAs of at least 16 k-blocks (up to 32
splits, and never fewer splits than the plain plan); a launch with a non-linear epilogue plans exactly as without the flag."""
import ctypes
import itertools

from fuxictr_b200 import _lib


def _plan(M, N, K, a_mn, b_mn, mode, epilogue, backfill):
    d = _lib.b2_gemm_desc()
    d.a, d.b, d.c = 0x10000000, 0x20000000, 0x30000000
    esz = 2 if mode == "bf16" else 4
    pad = 16 // esz
    d.lda = ((M if a_mn else K) + pad - 1) // pad * pad
    d.ldb = ((N if b_mn else K) + pad - 1) // pad * pad
    d.ldc = N
    d.M, d.N, d.K = M, N, K
    d.a_mn_major, d.b_mn_major = int(a_mn), int(b_mn)
    d.elem_dtype = _lib.B2_BF16 if mode == "bf16" else _lib.B2_F32
    d.flags = (_lib.B2_GEMM_X3_INLINE if mode == "tf32x3" else 0) | (_lib.B2_GEMM_BACKFILL if backfill else 0)
    if epilogue:
        d.bias, d.act = 0x60000000, 1
    plan = _lib.b2_gemm_plan()
    _lib.call("b2_gemm_tc_plan", ctypes.byref(d), ctypes.byref(plan))
    return plan


def _fields(p):
    return {k: getattr(p, k) for k, _ in _lib.b2_gemm_plan._fields_}


def test_backfill_plans():
    import __graft_entry__
    __graft_entry__.build()
    shapes = [(300, 300, 4096), (300, 624, 4096), (624, 624, 8192), (64, 415, 65536), (300, 300, 512),
              (128, 32, 32), (33, 257, 1000), (400, 624, 100000), (4096, 300, 300)]
    checked = 0
    for (M, N, K), a_mn, b_mn, mode, epi in itertools.product(shapes, (False, True), (False, True),
                                                               ("tf32", "tf32x3", "bf16"), (False, True)):
        esz = 2 if mode == "bf16" else 4
        if (a_mn and M % (16 // esz)) or (b_mn and N % (16 // esz)):
            continue
        tag = (M, N, K, a_mn, b_mn, mode, epi)
        plain = _plan(M, N, K, a_mn, b_mn, mode, epi, False)
        p = _plan(M, N, K, a_mn, b_mn, mode, epi, True)
        if epi:
            assert _fields(p) == _fields(plain), tag
            continue
        kb = -(-K // (128 // esz))
        assert (p.bn, p.tiles_m, p.tiles_n, p.stages, p.smem_bytes) == \
            (plain.bn, plain.tiles_m, plain.tiles_n, plain.stages, plain.smem_bytes), tag
        assert p.splits * p.kb_per_split >= kb and (p.splits - 1) * p.kb_per_split < kb, tag
        assert p.grid == p.tiles_m * p.tiles_n * p.splits, tag
        assert plain.splits <= p.splits <= 32, tag          # never fewer splits than the plain plan
        if p.splits > plain.splits:
            assert kb // p.splits >= 16, tag               # the added splits leave no CTA below the floor
        assert p.splits == 32 or kb // (2 * p.splits) < 16, tag   # and no more of them left to split off
        checked += 1
    assert checked > 50
    # DeepFM C2 (3xTF32): the wgrads of the 300-wide layers keep 8 splits, the first layer's goes from 4 to 8
    assert _plan(300, 300, 4096, True, True, "tf32x3", False, True).splits == 8
    assert _plan(300, 624, 4096, True, True, "tf32x3", False, False).splits == 4
    assert _plan(300, 624, 4096, True, True, "tf32x3", False, True).splits == 8
    # short K: the cost model's split stays (fewer than 32 k-blocks would otherwise force one CTA per tile)
    small = _plan(300, 300, 512, True, True, "tf32", False, False)
    assert small.splits > 1 and _plan(300, 300, 512, True, True, "tf32", False, True).splits == small.splits

"""The C-ABI boundary without a GPU: the library loads, exports every symbol the header
declares with the arity the ctypes table binds, and validates arguments before touching
CUDA (so these calls are safe on a CPU-only box)."""
import ctypes
import os
import re

import pytest

from conftest import ROOT

HEADER = os.path.join(ROOT, "include", "fuxictr_b200.h")


def header_prototypes():
    text = open(HEADER).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    protos = {}
    for m in re.finditer(r"B2_API\s+([\w\s\*]+?)\s*\b(b2_\w+)\s*\(([^;]*?)\)\s*;", text, flags=re.S):
        args = m.group(3).strip()
        nargs = 0 if args in ("void", "") else len([a for a in args.split(",") if a.strip()])
        protos[m.group(2)] = nargs
    return protos


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__
    __graft_entry__.build()
    from fuxictr_b200 import _lib
    return _lib


def test_header_declares_what_python_binds(lib):
    protos = header_prototypes()
    assert len(protos) >= 17
    assert set(protos) == set(lib.SIGNATURES), set(protos) ^ set(lib.SIGNATURES)
    for name, nargs in protos.items():
        assert len(lib.SIGNATURES[name][1]) == nargs, name


def test_library_exports_every_symbol(lib):
    handle = ctypes.CDLL(lib.LIB_PATH)
    for name in header_prototypes():
        assert hasattr(handle, name), name
    assert lib.version().startswith("fuxictr_b200")


def test_field_struct_layout(lib):
    assert ctypes.sizeof(lib.b2_field) == 64
    assert lib.b2_field.vocab.offset == 24 and lib.b2_field.dim.offset == 48


def test_entry_points_reject_bad_arguments_without_a_gpu(lib):
    L = lib.load()
    null = ctypes.c_void_p(0)
    rc = L.b2_gemm_f32(null, 1, 1, null, 1, 1, null, 1, 4, 4, 4, null, 0, null, null, 0, null)
    assert rc == -1 and b"NULL" in L.b2_last_error()
    rc = L.b2_fm_fwd(ctypes.c_void_p(16), 4, 3, 8, 7, ctypes.c_void_p(16), null)
    assert rc == -1 and b"mode" in L.b2_last_error()
    fields = (lib.b2_field * 1)()
    rc = L.b2_embed_gather_fwd(fields, 0, 4, lib.B2_F64, lib.B2_F32, null, null, 0, null)
    assert rc == -1 and b"nfields" in L.b2_last_error()
    rc = L.b2_embed_gather_fwd(fields, 1, 4, lib.B2_F64, lib.B2_BF16, null, null, 0, null)
    assert rc == -1
    with pytest.raises(lib.B2Error, match="NULL"):
        lib.call("b2_split_tf32", null, null, 8, null)


def test_front_rejects_lr_fields_that_disagree_with_the_embedding(lib):
    """The front kernels bound an LR row by the embedding field's vocab and skip the embedding's padding row in both
    tables, so b2_front_fwd / b2_front_bwd refuse LR fields whose vocab or padding_idx differ.  batch = 0, and the
    pointers are aligned stand-ins that are never dereferenced: nothing reaches a device."""
    L = lib.load()
    null = ctypes.c_void_p(0)
    p = ctypes.c_void_p(1 << 20)

    def packs(lr_vocab, lr_pad):
        emb, lr = (lib.b2_field * 2)(), (lib.b2_field * 2)()
        for i in range(2):
            emb[i].table, emb[i].idx, emb[i].out = p.value, p.value + 64 * i, p.value + 4096 + 64 * i
            emb[i].vocab, emb[i].idx_stride, emb[i].out_stride = 50, 2, 32
            emb[i].dim, emb[i].seq_len, emb[i].pool, emb[i].padding_idx = 16, 1, 0, 0
            lr[i].table, lr[i].idx, lr[i].idx_stride = p.value + 8192, emb[i].idx, 2
            lr[i].vocab, lr[i].dim, lr[i].seq_len, lr[i].padding_idx = 50, 1, 1, 0
        lr[1].vocab, lr[1].padding_idx = lr_vocab, lr_pad
        return emb, lr

    def fwd(emb, lr):
        return L.b2_front_fwd(emb, lr, 2, 0, lib.B2_I64, 1, null, p, p, null, None, null, null)

    def bwd(emb, lr):
        return L.b2_front_bwd(emb, lr, 2, 0, lib.B2_I64, 1, p, p, p, p, null, None, None, null)

    assert fwd(*packs(50, 0)) == 0 and bwd(*packs(50, 0)) == 0          # agreeing packs pass the checks
    for lr_vocab, lr_pad in ((49, 0), (51, 0), (50, -1), (50, 7)):
        for call in (fwd, bwd):
            assert call(*packs(lr_vocab, lr_pad)) == -1, (call.__name__, lr_vocab, lr_pad)
            msg = L.b2_last_error()
            assert b"field 1" in msg and b"vocab and padding_idx" in msg, msg


def test_missing_library_is_a_hard_error(lib, monkeypatch):
    monkeypatch.setattr(lib, "_lib", None)
    monkeypatch.setattr(lib, "LIB_PATH", "/nonexistent/libfuxictr_b200.so")
    with pytest.raises(ImportError):
        lib.load()


def test_metric_entry_points_validate_before_cuda(lib):
    """b2_auc / b2_sort_u32 / b2_logloss_sum reject bad sizes, NULLs, small or misaligned workspaces
    without touching a device; b2_auc_workspace_bytes is pure arithmetic."""
    L = lib.load()
    null = ctypes.c_void_p(0)
    nbytes = ctypes.c_int64(0)
    assert L.b2_auc_workspace_bytes(1000, ctypes.byref(nbytes)) == 0
    small = nbytes.value
    assert small >= 2 * 4 * 1000 + 256 * 4 and small % 256 == 0
    assert L.b2_auc_workspace_bytes(6_000_000, ctypes.byref(nbytes)) == 0 and nbytes.value > 48_000_000
    assert L.b2_auc_workspace_bytes(0, ctypes.byref(nbytes)) == -1
    assert L.b2_auc_workspace_bytes(1 << 31, ctypes.byref(nbytes)) == -1 and b"2^31" in L.b2_last_error()
    ptr = ctypes.c_void_p(4096)
    assert L.b2_auc(null, ptr, 10, ptr, 1 << 20, ptr, null) == -1 and b"NULL" in L.b2_last_error()
    assert L.b2_auc(ptr, ptr, 1000, ptr, small - 1, ptr, null) == -1 and b"workspace" in L.b2_last_error()
    assert L.b2_auc(ptr, ptr, 1000, ctypes.c_void_p(4096 + 8), small, ptr, null) == -1 and b"aligned" in L.b2_last_error()
    assert L.b2_auc(ptr, ptr, 1000, ptr, small, ctypes.c_void_p(4100), null) == -1
    assert L.b2_sort_u32(null, 0, null, 0, null) == 0                     # empty input: nothing to do
    assert L.b2_sort_u32(null, 5, ptr, small, null) == -1
    assert L.b2_logloss_sum(null, null, 0, null, null) == 0
    assert L.b2_logloss_sum(null, ptr, 4, ptr, null) == -1
    assert L.b2_set_l2_fetch_granularity(48) == -1 and b"granularity" in L.b2_last_error()


def _plan(M, N, K, a_mn=False, b_mn=False, mode="tf32x3", epilogue=False, lda=None, ldb=None):
    """b2_gemm_tc_plan for fake (aligned, never dereferenced) operand addresses."""
    from fuxictr_b200 import _lib
    d = _lib.b2_gemm_desc()
    d.a, d.b, d.c = 0x10000000, 0x20000000, 0x30000000
    esz = 2 if mode == "bf16" else 4
    pad = 16 // esz
    d.lda = lda or ((M if a_mn else K) + pad - 1) // pad * pad
    d.ldb = ldb or ((N if b_mn else K) + pad - 1) // pad * pad
    d.ldc = N
    d.M, d.N, d.K = M, N, K
    d.a_mn_major, d.b_mn_major = int(a_mn), int(b_mn)
    d.elem_dtype = _lib.B2_BF16 if mode == "bf16" else _lib.B2_F32
    if mode == "tf32x3":
        d.flags = _lib.B2_GEMM_X3_INLINE
    elif mode == "tf32x3_aux":
        d.a_small, d.b_small = 0x40000000, 0x50000000
    if epilogue:
        d.bias, d.act = 0x60000000, 1
    plan = _lib.b2_gemm_plan()
    _lib.call("b2_gemm_tc_plan", ctypes.byref(d), ctypes.byref(plan))
    return plan


def test_gemm_plans_fit_the_sm():
    """Host-only: for a sweep of shapes, operand majors, arithmetic modes and epilogues the launch plan of
    the wgmma GEMM stays inside one SM — <= 227 KB of dynamic shared memory, rings of >= 2 stages, accumulator
    tiles that fit the registers, one CTA per tile, tiles that cover the problem.  (A 239 KB plan once reached
    the GPU as `invalid argument`; this sweep runs without one.)"""
    import itertools
    shapes = [(4096, 300, 624), (4096, 624, 300), (300, 624, 4096), (8192, 624, 624), (624, 624, 8192), (2048, 500, 432),
              (65536, 64, 415), (64, 415, 65536), (128, 32, 32), (76, 44, 36), (1, 16, 8), (130, 18, 40), (4096, 1024, 1024),
              (100000, 400, 624), (777, 64, 128), (33, 257, 1000), (8192, 256, 256), (8192, 512, 2048)]
    checked = 0
    for (M, N, K), a_mn, b_mn, mode, epi in itertools.product(shapes, (False, True), (False, True),
                                                               ("tf32", "tf32x3", "tf32x3_aux", "bf16"), (False, True)):
        esz = 2 if mode == "bf16" else 4
        if (a_mn and M % (16 // esz)) or (b_mn and N % (16 // esz)):
            continue                      # an MN-major operand needs a 16-byte row pitch over its rows
        p = _plan(M, N, K, a_mn, b_mn, mode, epi)
        tag = (M, N, K, a_mn, b_mn, mode, epi)
        assert 1024 <= p.smem_bytes <= 227 * 1024, tag
        assert 2 <= p.stages <= 4 and 2 <= p.cstages <= 4, tag
        assert p.passes == (3 if mode.startswith("tf32x3") else 1), tag
        assert p.bn in (32, 64, 128), tag
        if p.passes == 3:
            assert p.bn <= 64, tag        # main, partial and correction accumulators: 3 x bn/2 registers a thread
        assert p.tiles_m * 128 >= M and p.tiles_n * p.bn >= N and (p.tiles_n - 1) * p.bn < N, tag
        kb = -(-K // (128 // esz))
        assert p.splits >= 1 and p.splits * p.kb_per_split >= kb and (p.splits - 1) * p.kb_per_split < kb, tag
        if epi:
            assert p.splits == 1, tag     # a non-linear epilogue cannot be split over K
        assert p.grid == p.tiles_m * p.tiles_n * p.splits, tag
        assert p.threads == 384, tag
        checked += 1
    assert checked > 400


def test_gemm_plan_rejects_what_tma_cannot_address():
    from fuxictr_b200 import _lib
    with pytest.raises(_lib.B2Error, match="TMA"):
        _plan(128, 64, 30, lda=30)        # fp32 row pitch of 120 bytes

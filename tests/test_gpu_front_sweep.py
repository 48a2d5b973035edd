"""The embedding front against float64 at every branch of its launch plans.

Fused front (csrc/fused_front.cu): b2_front_fwd (gather + FM product_sum + LR + bias in one launch), b2_front_bwd
(table, LR and bias gradients) and b2_table_mark, called through the C-ABI so that every buffer can start as NaN
and the backward can take a b2_touch over a flat gradient buffer, and once through functional.front (autograd).
Sharded front (csrc/shard.cu): publish, push, reduce, gprep, pull and the ragged evaluation lookup of
`world` virtual ranks on one GPU (sharded.VirtualPeerGroup), driven phase by phase in lock step.

Reference: a plain restatement in torch, run in float64 (the exact answer) and in float32:
    e[b,f]   = T_f[id[b,f]]                      (a zero row for an id outside [0, vocab))
    logit[b] = 1/2 sum_d((sum_f e)^2 - sum_f e^2) + sum_f w_f[id[b,f]] + bias
    table gradients: index_add_ over the live slots (id in range, not padding) of gx + gl * (sum_f e - e)
    LR gradients: index_add_ of gl over the live slots; bias gradient: sum_b gl
The bar, for the logit, the field sums and every gradient:
    err(ours, fp64) <= max(1e-5, 3 * err(fp32 restatement, fp64))          (max-norm, relative)
Copies are held bit-exact: the gathered rows, the rows landed by the push, emb_small against tf32_small(emb), the
LR weights and `status`.  Tables, gx and gl are positive, so no table-gradient sum can cancel to near zero (where
the order of the atomic adds would decide its last digits).

The fused front's lane plan: LPR = 2^next_pow2_log2(dim / 4) lanes per row, 32 / LPR rows per pass, MAX_PASSES =
2 | 5 | 8 by the number of passes, and a loop over chunks of 32 / LPR * MAX_PASSES fields beyond that
(front_branch below; tests/test_front_sweep_host.py checks that FRONT_SHAPES reach every combination)."""
import ctypes
import sys

import pytest
import torch

from conftest import rel_err, ROOT

sys.path.insert(0, ROOT)
pytestmark = pytest.mark.gpu

RTOL = 1e-5
MAX_FIELDS = 128          # B2_MAX_FIELDS
GRID_WARPS = 132 * 8 * 8  # grid_for's cap (132 SMs x 8 CTAs of 256 threads), in warps
GRID_THREADS = GRID_WARPS * 32
GAP = 20                  # floats between the tables of a flat buffer: 16-byte aligned, off the 16-float granules


# ------------------------------------------------------------------ the launch plan, restated on the host
def next_pow2_log2(v):
    l = 0
    while (1 << l) < v:
        l += 1
    return l


def front_branch(dim, F):
    """(LPR, MAX_PASSES, chunk loop) of launch_front_fwd for F fields of dim `dim`."""
    lpr_log2 = next_pow2_log2((dim + 3) // 4)
    rows_per_pass = 32 >> lpr_log2
    passes = -(-F // rows_per_pass)
    max_passes = 2 if passes <= 2 else (5 if passes <= 5 else 8)
    return 1 << lpr_log2, max_passes, F > rows_per_pass * max_passes


def reachable_branches():
    return {front_branch(dim, F) for dim in range(4, 129, 4) for F in range(1, MAX_FIELDS + 1)}


# (dim, F): every reachable (LPR, MAX_PASSES, chunk loop), the comment gives (LPR, passes)
FRONT_SHAPES = [
    (128, 1), (128, 2), (128, 3), (128, 5), (96, 6), (128, 8), (68, 9), (128, 128),   # 32: 1, 2, 3, 5, 6, 8, 9, 128
    (64, 4), (64, 10), (48, 16), (64, 17), (40, 26),                                   # 16: 2, 5, 8, 9, 13
    (32, 8), (32, 20), (24, 32), (32, 33), (20, 39),                                   # 8: 2, 5, 8, 9, 10
    (16, 16), (16, 40), (12, 64), (16, 65), (12, 26),                                  # 4: 2, 5, 8, 9, 4
    (8, 32), (8, 80), (8, 128),                                                        # 2: 2, 5, 8
    (4, 1), (4, 64), (4, 65), (4, 128),                                                # 1: 1, 2, 3, 4
    (100, 7), (124, 17),                                                               # 32 with idle lanes: 7, 17
]

IDX_DTYPES = [torch.float64, torch.int64, torch.int32]


# ------------------------------------------------------------------ helpers
def bar(ours, ref32, ref64, what):
    assert ours.shape == ref64.shape, (what, tuple(ours.shape), tuple(ref64.shape))
    if ref64.numel() == 0:       # the shard of a rank that owns no row of the table
        return
    e_ours, e_ref = rel_err(ours, ref64), rel_err(ref32, ref64)
    assert e_ours <= max(RTOL, 3 * e_ref), (what, e_ours, e_ref)


def tf32_small(x):
    """b2_tf32_small restated: x - big(x) rounded to tf32, to nearest with ties away from zero."""
    big = (x.view(torch.int32) & -8192).view(torch.float32)
    d = x - big
    return ((d.view(torch.int32) + 0x1000) & -8192).view(torch.float32)


def bits_equal(a, b):
    return torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


class Flat(object):
    """Tables laid out one after another in one float32 buffer, GAP floats apart (16-byte aligned starts that
    fall off the 16-float touch granules), so that a touch over the buffer covers them all."""

    def __init__(self, shapes):
        self.offs, off = [], GAP
        for rows, cols in shapes:
            self.offs.append(off)
            off = (off + rows * cols + 3) // 4 * 4 + GAP
        self.shapes, self.n = list(shapes), off

    def buffer(self, tensors=None):
        buf = torch.zeros(self.n, dtype=torch.float32, device="cuda")
        views = [buf[o:o + r * c].view(r, c) for o, (r, c) in zip(self.offs, self.shapes)]
        if tensors is not None:
            for v, t in zip(views, tensors):
                v.copy_(t)
        return buf, views

    def granules(self, spans):
        """Flags of the granules that any (table, first row, rows) span overlaps."""
        g = torch.zeros(-(-self.n // 16), dtype=torch.uint8)
        for t, row, nrows in spans:
            cols = self.shapes[t][1]
            lo = self.offs[t] + row * cols
            g[lo // 16:(lo + nrows * cols - 1) // 16 + 1] = 1
        return g


def touch_of(buf):
    from fuxictr_b200 import _lib
    flags = torch.zeros(-(-buf.numel() // 16), dtype=torch.uint8, device="cuda")
    return flags, _lib.b2_touch(flags.data_ptr(), buf.data_ptr(), buf.numel())


def check_touch(flags, grad_flat, allowed, what):
    """Every granule holding a non-zero gradient is flagged (touched Adam skips the others), and no granule is
    flagged that no referenced row overlaps."""
    flags = flags.cpu()
    g = grad_flat.cpu()
    pad = (-g.numel()) % 16
    nonzero = (torch.cat([g, g.new_zeros(pad)]).view(-1, 16) != 0).any(1)
    assert bool((flags[nonzero] == 1).all()), (what, "unflagged granules", torch.nonzero(nonzero & (flags == 0))[:8])
    stray = (flags == 1) & (allowed == 0)
    assert not bool(stray.any()), (what, "stray flags", torch.nonzero(stray)[:8])


def reference(tables, lr_tables, tab_of, vocab, pads, ids, bias, gx, gl, want_fm, dtype):
    """The front restated in `dtype` on the CPU.  tables[t] (V_t, D); lr_tables[t] (V_t, 1) or None; field f reads
    table tab_of[f] with vocab[f] rows and padding row pads[f] (-1: none); ids (N, F) int64; gx (N, F, D); gl (N,)."""
    N, F = ids.shape
    embs, live, lrsum = [], [], torch.zeros(N, dtype=dtype)
    for f in range(F):
        i = ids[:, f]
        ok = (i >= 0) & (i < vocab[f])
        j = i.clamp(0, vocab[f] - 1)
        embs.append(tables[tab_of[f]].to(dtype)[j] * ok[:, None].to(dtype))
        live.append(ok & (i != pads[f]))
        if lr_tables is not None:
            lrsum = lrsum + lr_tables[tab_of[f]].to(dtype)[j, 0] * ok.to(dtype)
    E = torch.stack(embs, 1)
    S, Q = E.sum(1), (E * E).sum(1)
    logit = torch.zeros(N, dtype=dtype)
    if want_fm:
        logit = logit + 0.5 * (S * S - Q).sum(1)
    if lr_tables is not None:
        logit = logit + lrsum
    if bias is not None:
        logit = logit + bias.to(dtype)
    gl_ = gl.to(dtype)
    g = gx.to(dtype).clone()
    if want_fm:
        g = g + gl_[:, None, None] * (S[:, None, :] - E)
    gT = [torch.zeros(t.shape, dtype=dtype) for t in tables]
    gL = [torch.zeros(t.shape, dtype=dtype) for t in lr_tables] if lr_tables is not None else None
    for f in range(F):
        m = live[f]
        gT[tab_of[f]].index_add_(0, ids[m, f], g[m, f])
        if gL is not None:
            gL[tab_of[f]].index_add_(0, ids[m, f], gl_[m, None])
    return dict(emb=E, sums=S, logit=logit, g=g, gT=gT, gL=gL, gbias=gl_.sum(), live=live)


def make_ids(gen, N, vocab, pads, *, oob_fields=(), zipf=False, same_row_field=None):
    """(N, F) int64 ids: uniform (or Zipf-heavy) in range, every padding row present, and in `oob_fields` ids at
    vocab, vocab + 3 and -1."""
    cols = []
    for f, V in enumerate(vocab):
        u = torch.rand(N, generator=gen, dtype=torch.float64)
        i = (V * (u ** 4 if zipf else u)).long().clamp(max=V - 1)
        if pads[f] >= 0:
            i[3::5] = pads[f]
        if f in oob_fields:
            i[1::7] = V
            i[4::13] = V + 3
            i[2::11] = -1
        if f == same_row_field:
            i[:] = V // 2 if V // 2 != pads[f] else V // 2 + 1
        cols.append(i)
    return torch.stack(cols, 1)


def expected_status(ids, vocab, slot_field=None):
    """max(field + 1) over the slots (columns of ids) holding an out-of-range id, 0 when there is none."""
    bad = [(slot_field[s] if slot_field else s) + 1 for s in range(ids.shape[1])
           if bool(((ids[:, s] < 0) | (ids[:, s] >= vocab[s])).any())]
    return max(bad) if bad else 0


@pytest.fixture(scope="module", autouse=True)
def _built():
    import __graft_entry__
    __graft_entry__.build()
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"


# ------------------------------------------------------------------ fused front through the C-ABI
def front_case(dim, F, B, *, want_fm=True, has_lr=True, with_bias=True, idx_dtype=torch.float64, small=False,
               oob=True, shared=False, zipf=False, same_row=False, emb_grad=True, lr_grad=True, seed=0):
    from fuxictr_b200 import _lib, functional as F2
    gen = torch.Generator().manual_seed(seed * 1009 + dim * 131 + F * 7 + B)
    tab_of = list(range(F))
    if shared and F >= 2:
        tab_of[1] = 0                                   # fields 0 and 1 read one table (one gradient buffer)
    ntab = max(tab_of) + 1
    tvocab = [40 + (7 * t) % 61 for t in range(ntab)]
    vocab = [tvocab[tab_of[f]] for f in range(F)]
    pads = [(3 if f % 2 == 0 else -1) for f in range(F)]          # a padding row other than 0, and none
    tables = [(0.25 + 0.5 * torch.rand(V, dim, generator=gen)) for V in tvocab]
    lr_tables = [(0.1 + 0.2 * torch.rand(V, 1, generator=gen)) for V in tvocab] if has_lr else None
    bias = torch.tensor([0.3]) if with_bias else None
    oob_fields = {f for f in range(F) if f % 3 == 1} | {F - 1} if oob else set()
    ids = make_ids(gen, B, vocab, pads, oob_fields=oob_fields, zipf=zipf, same_row_field=0 if same_row else None)
    gx = 0.5 + torch.rand(B, F, dim, generator=gen)
    gl = 0.25 + torch.rand(B, generator=gen)

    shapes = [tuple(t.shape) for t in tables] + ([tuple(t.shape) for t in lr_tables] if has_lr else [])
    lay = Flat(shapes)
    pflat, pviews = lay.buffer(tables + (lr_tables or []))
    gflat, gviews = lay.buffer()
    ptab, plr = pviews[:ntab], pviews[ntab:]
    gtab, glr = gviews[:ntab], gviews[ntab:]

    # batch matrix (B, F + 1) in the index dtype, as the collator lays it out (a label column at the end)
    mat = torch.cat([ids, torch.zeros(B, 1, dtype=torch.int64)], 1).to(idx_dtype).cuda()
    W = F + 1
    width = F * dim
    stride = width + 4                                  # 4 guard floats after each sample's row
    nan = float("nan")
    arena = torch.full((B + 2, stride), nan, device="cuda")  # guard rows 0 and B + 1
    small_buf = torch.full((B + 2, stride), nan, device="cuda") if small else None
    sums = torch.full((B + 2, dim), nan, device="cuda") if want_fm else None
    logit = torch.full((B + 2,), nan, device="cuda")
    status = torch.zeros(1, dtype=torch.int32, device="cuda")
    bias_d = bias.cuda() if bias is not None else None
    esz, fsz = mat.element_size(), 4

    def descs(tabs, lrs, out_base):
        e = (_lib.b2_field * F)()
        l = (_lib.b2_field * F)() if has_lr else None
        for f in range(F):
            d = e[f]
            d.table = tabs[tab_of[f]].data_ptr() if tabs[tab_of[f]] is not None else 0
            d.idx, d.idx_stride, d.vocab = mat.data_ptr() + f * esz, W, vocab[f]
            d.out, d.out_stride = (out_base + f * dim * fsz, stride) if out_base else (0, 0)
            d.dim, d.seq_len, d.pool, d.padding_idx = dim, 1, 0, pads[f]
            if l is not None:
                d = l[f]
                d.table = lrs[tab_of[f]].data_ptr() if lrs[tab_of[f]] is not None else 0
                d.idx, d.idx_stride, d.vocab = mat.data_ptr() + f * esz, W, vocab[f]
                d.dim, d.seq_len, d.pool, d.padding_idx = 1, 1, 0, pads[f]
        return e, l

    row1 = arena.data_ptr() + stride * fsz
    e, l = descs(ptab, plr, row1)
    code = F2._IDX_CODE[idx_dtype]
    _lib.call("b2_front_fwd", e, l, F, B, code, int(want_fm), F2._ptr(bias_d), ctypes.c_void_p(logit.data_ptr() + 4),
              ctypes.c_void_p(sums.data_ptr() + dim * fsz) if want_fm else None, F2._ptr(status), None,
              ctypes.c_void_p(small_buf.data_ptr() + stride * fsz) if small else None, F2._stream())

    # backward: gx in an arena laid out like the forward's (NaN guards), gradients into the flat buffer
    garena = torch.full((B + 2, stride), nan, device="cuda")
    garena[1:B + 1, :width] = gx.view(B, width).cuda()
    gl_d = gl.cuda()
    gbias = torch.zeros(1, device="cuda") if with_bias else None
    gtabs = [v if emb_grad else None for v in gtab]
    glrs = [v if lr_grad else None for v in glr]
    ge, gle = descs(gtabs, glrs, garena.data_ptr() + stride * fsz)
    flags, touch = touch_of(gflat)
    _lib.call("b2_front_bwd", ge, gle, F, B, code, int(want_fm), ctypes.c_void_p(row1),
              ctypes.c_void_p(garena.data_ptr() + stride * fsz),
              ctypes.c_void_p(sums.data_ptr() + dim * fsz) if want_fm else None,
              F2._ptr(gl_d), F2._ptr(gbias), None, ctypes.byref(touch), F2._stream())
    # table_mark over the parameter buffer (same layout): a superset of the backward's flags
    mflags, mtouch = touch_of(pflat)
    me, ml = descs(ptab, plr, 0)
    _lib.call("b2_table_mark", me, ml, F, B, code, ctypes.byref(mtouch), F2._stream())
    torch.cuda.synchronize()

    r64 = reference(tables, lr_tables, tab_of, vocab, pads, ids, bias, gx, gl, want_fm, torch.float64)
    r32 = reference(tables, lr_tables, tab_of, vocab, pads, ids, bias, gx, gl, want_fm, torch.float32)
    a = arena.cpu()
    # ---- forward
    assert bits_equal(a[1:B + 1, :width], r32["emb"].reshape(B, width)), "gathered rows"
    assert bool(torch.isnan(a[0]).all() and torch.isnan(a[B + 1]).all() and torch.isnan(a[:, width:]).all()), \
        "the forward wrote outside its rows"
    if small:
        s = small_buf.cpu()
        assert bits_equal(s[1:B + 1, :width], tf32_small(a[1:B + 1, :width].contiguous())), "emb_small"
        assert bool(torch.isnan(s[0]).all() and torch.isnan(s[B + 1]).all() and torch.isnan(s[:, width:]).all())
    lg = logit.cpu()
    bar(lg[1:B + 1], r32["logit"], r64["logit"], "logit")
    assert bool(torch.isnan(lg[0]) and torch.isnan(lg[B + 1]))
    if want_fm:
        sm = sums.cpu()
        bar(sm[1:B + 1], r32["sums"], r64["sums"], "sums")
        assert bool(torch.isnan(sm[0]).all() and torch.isnan(sm[B + 1]).all())
    assert int(status.item()) == expected_status(ids, vocab), "status"
    # ---- backward
    gf = gflat.cpu()
    for t in range(ntab):
        got = gtab[t].cpu()
        if not emb_grad:
            assert not bool(got.any()), ("NULL gradient table written", t)
        else:
            bar(got, r32["gT"][t], r64["gT"][t], "gT%d" % t)
            dead = r64["gT"][t].abs().sum(1) == 0       # rows no live slot reaches: padding, out of range, unused
            assert not bool(got[dead].any()), ("gradient in a row without a live slot", t)
        if not has_lr:
            continue
        got = glr[t].cpu()
        if not lr_grad:
            assert not bool(got.any()), ("NULL LR gradient table written", t)
        else:
            bar(got, r32["gL"][t], r64["gL"][t], "gL%d" % t)
            assert not bool(got[r64["gL"][t][:, 0] == 0].any()), ("LR gradient in a row without a live slot", t)
    outside = torch.ones(lay.n, dtype=torch.bool)
    for o, (r, c) in zip(lay.offs, lay.shapes):
        outside[o:o + r * c] = False
    assert not bool(gf[outside].any()), "the backward wrote between the tables"
    if with_bias:
        bar(gbias.cpu()[0], r32["gbias"], r64["gbias"], "gbias")
    # ---- touch flags: referenced = an in-range id of a field whose gradient table is there
    spans, mark_spans = [], []
    for f in range(F):
        for row in torch.unique(ids[:, f][(ids[:, f] >= 0) & (ids[:, f] < vocab[f])]).tolist():
            mark_spans.append((tab_of[f], row, 1))
            if emb_grad:
                spans.append((tab_of[f], row, 1))
            if has_lr:
                mark_spans.append((ntab + tab_of[f], row, 1))
                if lr_grad:
                    spans.append((ntab + tab_of[f], row, 1))
    check_touch(flags, gflat, lay.granules(spans), "b2_front_bwd")
    mf, bf = mflags.cpu(), flags.cpu()
    assert bool((mf >= bf).all()), ("b2_table_mark misses granules the backward flags", torch.nonzero(bf > mf)[:8])
    assert not bool(((mf == 1) & (lay.granules(mark_spans) == 0)).any()), "b2_table_mark flags an unread granule"


@pytest.mark.parametrize("dim,F", FRONT_SHAPES)
def test_front_lane_plans(dim, F):
    """Every (LPR, MAX_PASSES, chunk loop) at B = 257, with out-of-range and -1 ids in several fields, a non-zero
    padding row at index 3, emb_small on every other shape, and the flags and id dtype varying along the list."""
    i = FRONT_SHAPES.index((dim, F))
    front_case(dim, F, 257, want_fm=i % 2 == 0, has_lr=i % 3 != 2, with_bias=i % 4 != 3,
               idx_dtype=IDX_DTYPES[i % 3], small=(i // 2) % 2 == 1, seed=i)


@pytest.mark.parametrize("idx_dtype", IDX_DTYPES, ids=["f64", "i64", "i32"])
@pytest.mark.parametrize("want_fm", [True, False], ids=["fm", "nofm"])
@pytest.mark.parametrize("has_lr", [True, False], ids=["lr", "nolr"])
@pytest.mark.parametrize("with_bias", [True, False], ids=["bias", "nobias"])
def test_front_flags_and_index_dtypes(idx_dtype, want_fm, has_lr, with_bias):
    front_case(40, 26, 255, want_fm=want_fm, has_lr=has_lr, with_bias=with_bias, idx_dtype=idx_dtype,
               small=want_fm, oob=has_lr)


@pytest.mark.parametrize("B", [1, 255, 257])
@pytest.mark.parametrize("dim,F", [(4, 3), (12, 26), (128, 9)])
def test_front_batch_edges(B, dim, F):
    front_case(dim, F, B, idx_dtype=torch.int64, small=True)


def test_front_forward_grid_strides():
    """B = 20000 samples > 8448 warps of the capped grid (the forward's sample loop strides), and B * F * LPR =
    640000 lanes > 270336 threads (the backward's item loop strides)."""
    B, dim, F = 20000, 32, 4
    assert B > GRID_WARPS and B * F * front_branch(dim, F)[0] > GRID_THREADS
    front_case(dim, F, B, idx_dtype=torch.int32, zipf=True)


def test_front_backward_grid_strides():
    """B * F * LPR = 3000 * 26 * 16 > 270336 with fewer samples than warps (the forward does not stride)."""
    B, dim, F = 3000, 64, 26
    assert B < GRID_WARPS and B * F * front_branch(dim, F)[0] > GRID_THREADS
    front_case(dim, F, B, small=True)


@pytest.mark.parametrize("dim,F", [(4, 1), (4, 5), (16, 2), (64, 3), (128, 2)])
def test_front_warp_aggregation(dim, F):
    """Field 0 hits one live row in every sample (a warp of 32 / LPR items that all aggregate into one row at
    LPR = 1), and fields 0 and 1 share one table, so neighbouring items of a sample meet in one gradient row."""
    front_case(dim, F, 257, shared=True, same_row=True)


@pytest.mark.parametrize("zipf", [True, False])
def test_front_shared_table_zipf(zipf):
    front_case(16, 39, 1024, shared=True, zipf=zipf, idx_dtype=torch.int32, small=True)


@pytest.mark.parametrize("emb_grad,lr_grad", [(False, True), (True, False), (False, False)])
def test_front_tables_without_gradients(emb_grad, lr_grad):
    """A table that does not require grad reaches the backward as a NULL gradient table."""
    front_case(24, 11, 257, emb_grad=emb_grad, lr_grad=lr_grad)


def test_front_autograd_wrapper_tf32x3_small_part():
    """functional.front under 3xTF32 with the small parts in HBM (set_x3_inline(False)): the arena's small part is
    tf32_small(arena), bit for bit; the autograd gradients (tables, LR tables, bias) meet the bar."""
    from fuxictr_b200 import functional as F2
    B, dim, F = 300, 20, 6
    gen = torch.Generator().manual_seed(11)
    vocab, pads = [30 + 3 * f for f in range(F)], [0 if f % 2 else -1 for f in range(F)]
    tables = [0.25 + 0.5 * torch.rand(V, dim, generator=gen) for V in vocab]
    lr_tables = [0.1 + 0.2 * torch.rand(V, 1, generator=gen) for V in vocab]
    bias = torch.tensor([0.2])
    ids = make_ids(gen, B, vocab, pads, oob_fields={2})
    gx = 0.5 + torch.rand(B, F, dim, generator=gen)
    gl = 0.25 + torch.rand(B, generator=gen)
    plan = F2.GatherPlan([F2.GatherField("f%d" % f, f, dim, padding_idx=pads[f]) for f in range(F)])
    lr_plan = F2.GatherPlan([F2.GatherField("f%d" % f, f, 1, padding_idx=pads[f]) for f in range(F)])
    et = [t.cuda().requires_grad_(True) for t in tables]
    lt = [t.cuda().requires_grad_(True) for t in lr_tables]
    bd = bias.cuda().requires_grad_(True)
    status = torch.zeros(1, dtype=torch.int32, device="cuda")
    mode, inline = F2.get_matmul_precision(), F2._MATMUL["x3_inline"]
    try:
        F2.set_matmul_precision("tf32x3")
        F2.set_x3_inline(False)
        arena, logit = F2.front(plan, lr_plan, [ids[:, f].double().cuda() for f in range(F)], et, lt, bd, True,
                                status=status)
    finally:
        F2.set_matmul_precision(mode)
        F2.set_x3_inline(inline)
    aux = getattr(arena, "_b2_aux", None)
    assert aux is not None and aux[0] == "tf32x3", "set_x3_inline(False) must make the front write emb_small"
    assert bits_equal(aux[1].cpu(), tf32_small(arena.detach().cpu()))
    ((arena * gx.view(B, -1).cuda()).sum() + (logit.view(-1) * gl.cuda()).sum()).backward()
    r64 = reference(tables, lr_tables, list(range(F)), vocab, pads, ids, bias, gx, gl, True, torch.float64)
    r32 = reference(tables, lr_tables, list(range(F)), vocab, pads, ids, bias, gx, gl, True, torch.float32)
    assert bits_equal(arena.detach().cpu(), r32["emb"].reshape(B, -1))
    bar(logit.detach().cpu().view(-1), r32["logit"], r64["logit"], "logit")
    assert int(status.item()) == 3
    for f in range(F):
        bar(et[f].grad.cpu(), r32["gT"][f], r64["gT"][f], "gT%d" % f)
        bar(lt[f].grad.cpu(), r32["gL"][f], r64["gL"][f], "gL%d" % f)
    bar(bd.grad.cpu()[0], r32["gbias"], r64["gbias"], "gbias")


# ------------------------------------------------------------------ sharded front (virtual ranks, lock step)
def shard_case(world, dim, vocab, B_l, *, seq_lens=None, has_lr=True, want_fm=True, with_bias=True,
               idx_dtype=torch.float64, oob=True, zipf=False, seed=0):
    """Push, reduce, gprep, pull (with a touch over each rank's flat gradient buffer) and an evaluation round of
    `world` virtual ranks, each against the float64 restatement over the global batch.  Field f's padding row is
    None, 0 or vocab - 1 by f % 3; owner of global row r = r % world (no power-of-two assumption)."""
    from fuxictr_b200 import _lib, functional as F2, sharded as SH
    gen = torch.Generator().manual_seed(seed * 7919 + world * 101 + dim)
    F = len(vocab)
    seq_lens = list(seq_lens) if seq_lens is not None else [1] * F
    slot_field = [f for f in range(F) for _ in range(seq_lens[f])]
    S = len(slot_field)
    pads = [(-1, 0, vocab[f] - 1)[(f + seed) % 3] for f in range(F)]
    tables = [0.25 + 0.5 * torch.rand(V, dim, generator=gen) for V in vocab]
    lr_tables = [0.1 + 0.2 * torch.rand(V, 1, generator=gen) for V in vocab] if has_lr else None
    bias = torch.tensor([-0.4]) if with_bias else None
    N = world * B_l
    svocab, spads = [vocab[f] for f in slot_field], [pads[f] for f in slot_field]
    oob_slots = {s for s in range(S) if s % 3 == 2} if oob else set()
    ids = make_ids(gen, N, svocab, spads, oob_fields=oob_slots, zipf=zipf)
    gx = 0.5 + torch.rand(N, S, dim, generator=gen)
    gl = 0.25 + torch.rand(N, generator=gen)
    W = S + 1                                            # the fields' columns, then a label column
    mat = torch.cat([ids, torch.zeros(N, 1, dtype=torch.int64)], 1).to(idx_dtype).cuda()
    columns = [sum(seq_lens[:f]) for f in range(F)]

    registry, fronts, lays, flats = {}, [], [], []
    for r in range(world):
        et = [SH.shard_rows(t, r, world).cuda() for t in tables]
        lt = [SH.shard_rows(t, r, world).cuda() for t in lr_tables] if has_lr else None
        fronts.append(SH.ShardedFront(SH.VirtualPeerGroup(r, world, registry), ["f%d" % f for f in range(F)], et, lt,
                                      vocab, columns, [None if p < 0 else p for p in pads], dim, B_l, W, idx_dtype,
                                      bias=bias.cuda() if with_bias else None, want_fm=want_fm, seq_lens=seq_lens))
        lay = Flat([tuple(t.shape) for t in et] + ([tuple(t.shape) for t in lt] if has_lr else []))
        lays.append(lay)
        flats.append(lay.buffer())
    for r, fr in enumerate(fronts):
        fr.phase_ids(mat[r * B_l:(r + 1) * B_l])
    for fr in fronts:
        fr.phase_push()
    outs = [fr.phase_reduce() for fr in fronts]
    torch.cuda.synchronize()
    slot_tables = [tables[f] for f in slot_field]
    slot_lr = [lr_tables[f] for f in slot_field] if has_lr else None
    r64 = reference(slot_tables, slot_lr, list(range(S)), svocab, spads, ids, bias, gx, gl, want_fm, torch.float64)
    r32 = reference(slot_tables, slot_lr, list(range(S)), svocab, spads, ids, bias, gx, gl, want_fm, torch.float32)
    live = torch.stack(r64["live"], 1)                   # (N, S)
    owner = ids.remainder(world)
    for r, fr in enumerate(fronts):
        rows = slice(r * B_l, (r + 1) * B_l)
        assert bits_equal(fr.emb.cpu(), r32["emb"][rows].reshape(B_l, S * dim)), ("landed rows", r)
        if has_lr:
            lr_ref = torch.stack([slot_lr[s][ids[rows, s].clamp(0, svocab[s] - 1), 0] *
                                  ((ids[rows, s] >= 0) & (ids[rows, s] < svocab[s])).float() for s in range(S)], 1)
            assert bits_equal(fr.lrw.cpu(), lr_ref), ("landed LR weights", r)
        if has_lr or want_fm:
            bar(outs[r][1].cpu().view(-1), r32["logit"][rows], r64["logit"][rows], "logit rank %d" % r)
        if want_fm:
            bar(outs[r][2].cpu(), r32["sums"][rows], r64["sums"][rows], "sums rank %d" % r)
        status_r = expected_status(ids[rows], svocab, slot_field)      # this rank's own samples only
        assert int(fr.status.item()) == status_r, ("status", r, int(fr.status.item()), status_r)
        assert int(fr.owned_count.item()) == int((live & (owner == r)).sum()), ("owned_count", r)

    # ---- backward: gprep (bias gradient pre-zeroed on even ranks, NaN and reset on odd ones), then the pull
    needs_logit = has_lr or want_fm
    gbiases = []
    for r, fr in enumerate(fronts):
        rows = slice(r * B_l, (r + 1) * B_l)
        gx_r = gx[rows].reshape(B_l, -1).cuda()
        gl_r = gl[rows].cuda() if needs_logit else None
        gb = None
        if with_bias:
            gb = torch.zeros(1, device="cuda") if r % 2 == 0 else torch.full((1,), float("nan"), device="cuda")
        gbiases.append((gb, gx_r, gl_r))
        _lib.call("b2_front_gprep", F2._ptr(gx_r), F2._ptr(fr.emb), F2._ptr(outs[r][2]), F2._ptr(gl_r), B_l, S, dim,
                  int(want_fm), F2._ptr(fr.gemb), F2._ptr(fr.glogit) if gl_r is not None else None, F2._ptr(gb),
                  1 if (gb is not None and r % 2 == 0) else 0, F2._stream())
    touches = []
    for r, fr in enumerate(fronts):
        flat, views = flats[r]
        egr, lgr = views[:F], (views[F:] if has_lr else None)
        flags, touch = touch_of(flat)
        touches.append(flags)
        lr = fr._descs(lgr, 1) if lgr else None
        _lib.call("b2_shard_pull", fr._descs(egr, dim), lr, F, B_l, world, r, SH._ptr_array(fr.gemb_ptrs),
                  SH._ptr_array(fr.glogit_ptrs) if lr is not None else None, fr.pull_scale, F2._ptr(fr.owned),
                  F2._ptr(fr.owned_count), fr.owned_cap, None, ctypes.byref(touch), F2._stream())
    torch.cuda.synchronize()
    for r, fr in enumerate(fronts):
        rows = slice(r * B_l, (r + 1) * B_l)
        bar(fr.gemb.cpu(), r32["g"][rows].reshape(B_l, -1), r64["g"][rows].reshape(B_l, -1), "gemb rank %d" % r)
        if needs_logit:
            assert bits_equal(fr.glogit.cpu(), gl[rows]), ("published logit gradient", r)
        if with_bias:
            bar(gbiases[r][0].cpu()[0], gl[rows].float().sum(), gl[rows].double().sum(), "gbias rank %d" % r)
    # gradients: each field's table sums its slots; the pull scales every row by 1 / world
    for r, fr in enumerate(fronts):
        flat, views = flats[r]
        lay = lays[r]
        for f in range(F):
            ss = [s for s in range(S) if slot_field[s] == f]
            want = {}
            for dt, ref in ((torch.float64, r64), (torch.float32, r32)):
                full = sum(ref["gT"][s] for s in ss) * torch.tensor(1.0 / world, dtype=dt)
                want[dt] = SH.shard_rows(full, r, world)
            got = views[f].cpu()
            bar(got, want[torch.float32], want[torch.float64], "gT field %d rank %d" % (f, r))
            assert not bool(got[want[torch.float64].abs().sum(1) == 0].any()), ("gradient in a dead row", f, r)
            if has_lr:
                full64 = r64["gL"][f] * (1.0 / world)
                full32 = r32["gL"][f] * torch.tensor(1.0 / world)
                got = views[F + f].cpu()
                bar(got, SH.shard_rows(full32, r, world), SH.shard_rows(full64, r, world), "gL %d rank %d" % (f, r))
                assert not bool(got[SH.shard_rows(full64, r, world)[:, 0] == 0].any()), ("LR gradient, dead row", f, r)
        outside = torch.ones(lay.n, dtype=torch.bool)
        for o, (nr, c) in zip(lay.offs, lay.shapes):
            outside[o:o + nr * c] = False
        assert not bool(flat.cpu()[outside].any()), ("the pull wrote between the tables", r)
        spans = []
        for s in range(S):
            f = slot_field[s]
            i = ids[:, s]
            mine = (i >= 0) & (i < svocab[s]) & (i.remainder(world) == r)
            for row in torch.unique(i[mine]).tolist():
                spans.append((f, row // world, 1))
                if has_lr:
                    spans.append((F + f, row // world, 1))
        check_touch(touches[r], flat, lay.granules(spans), "b2_shard_pull rank %d" % r)

    # ---- an evaluation round: rank r serves rows_all[r] in {batch_local, 0, some} of new ids
    eids = make_ids(gen, N, svocab, spads, oob_fields=oob_slots)
    emat = torch.cat([eids, torch.zeros(N, 1, dtype=torch.int64)], 1).to(idx_dtype).cuda()
    nrows = [(B_l, 0, 1 + (5 * r) % B_l)[r % 3] for r in range(world)]
    owned_before = [(fr.owned.clone(), fr.owned_count.clone()) for fr in fronts]
    for fr in fronts:
        fr.status.zero_()
    for r, fr in enumerate(fronts):
        assert fr.eval_phase_ids(emat[r * B_l:r * B_l + nrows[r]]) == nrows[r]
    for fr in fronts:
        fr.eval_phase_lookup()
    landed = [fr.eval_phase_reduce() for fr in fronts]
    torch.cuda.synchronize()
    e64 = reference(slot_tables, slot_lr, list(range(S)), svocab, spads, eids, bias, gx, gl, want_fm, torch.float64)
    e32 = reference(slot_tables, slot_lr, list(range(S)), svocab, spads, eids, bias, gx, gl, want_fm, torch.float32)
    for r, fr in enumerate(fronts):
        n = nrows[r]
        rows = slice(r * B_l, r * B_l + n)
        assert torch.equal(fr.owned, owned_before[r][0]) and torch.equal(fr.owned_count, owned_before[r][1]), \
            ("the evaluation lookup touched the owned list", r)
        status_r = expected_status(eids[rows], svocab, slot_field) if n else 0
        assert int(fr.status.item()) == status_r, ("evaluation status", r)
        if n == 0:
            assert landed[r] is None
            continue
        assert bits_equal(fr.emb[:n].cpu(), e32["emb"][rows].reshape(n, S * dim)), ("evaluation rows", r)
        if needs_logit:
            bar(landed[r][1].cpu().view(-1), e32["logit"][rows], e64["logit"][rows], "evaluation logit %d" % r)


# (world, dim, vocabularies, batch_local, idx dtype): vocabularies below the world leave ranks without rows
SHARD_CASES = [
    (1, 16, [37, 50, 9, 64, 21, 40], 33, torch.float64),
    (2, 8, [45, 12, 30, 77, 18, 25, 60], 40, torch.float64),
    (3, 40, [41, 29, 100, 7, 55], 33, torch.int64),
    (5, 128, [23, 61, 4], 31, torch.int32),
    (8, 4, [3, 5, 7, 100, 64, 9, 8, 33, 250], 35, torch.float64),
    (16, 12, [2, 9, 16, 300], 17, torch.int64),
]


@pytest.mark.parametrize("world,dim,vocab,B_l,idx_dtype", SHARD_CASES,
                         ids=["w%d-d%d" % (c[0], c[1]) for c in SHARD_CASES])
def test_sharded_front(world, dim, vocab, B_l, idx_dtype):
    shard_case(world, dim, vocab, B_l, idx_dtype=idx_dtype, want_fm=world != 2, with_bias=world != 3,
               seed=world)


def test_sharded_front_zipf_lr_only():
    shard_case(3, 24, [200, 31, 17, 90], 64, want_fm=False, zipf=True, seed=1)


def test_sharded_push_more_chunks_than_the_grid():
    """world * batch_local * slots = 3 * 2304 * 40 = 276480 candidates > 270336 = 1056 CTAs x 256 (the push's chunk
    loop runs twice in some CTAs), and ~92k owned entries per rank > the 67584 lane groups of the pull's grid."""
    vocab = [50 + 13 * f for f in range(40)]
    assert 3 * 2304 * 40 > GRID_THREADS
    shard_case(3, 16, vocab, 2304, has_lr=False, with_bias=False, oob=True, seed=2)


@pytest.mark.parametrize("world,dim,seq_lens,vocab", [(3, 16, [1, 4, 1, 3], [40, 70, 5, 33]),
                                                      (16, 32, [5, 1, 2], [100, 3, 20])],
                         ids=["w3", "w16"])
def test_sharded_embedding_only_sequences(world, dim, seq_lens, vocab):
    """DLRM / DIN-style fronts: embeddings only, unpooled sequence fields as consecutive slots (ALL_LEN1 = false)."""
    shard_case(world, dim, vocab, 29, seq_lens=seq_lens, has_lr=False, want_fm=False, with_bias=False,
               idx_dtype=torch.float64, seed=world)

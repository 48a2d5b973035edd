"""torch.autograd bindings of the C-ABI kernels (device pointers in, device pointers out).

PyTorch is plumbing here: it owns device memory, the current stream and the autograd
tape; all arithmetic happens in libfuxictr_b200.so.  Every function requires CUDA
tensors and raises otherwise — there is no eager/CPU fallback on this path.
"""
import ctypes
import math
import os
import weakref

import torch

from . import _lib
from ._lib import (B2_F32, B2_BF16, B2_F64, B2_I32, B2_I64, B2_POOL_NONE, B2_POOL_SUM, B2_POOL_MEAN,
                   B2_ACT_NONE, B2_ACT_RELU, B2_ACT_SIGMOID, B2_PREP_MUL, b2_field)

_IDX_CODE = {torch.float64: B2_F64, torch.int64: B2_I64, torch.int32: B2_I32}
ACT_CODE = {None: B2_ACT_NONE, "none": B2_ACT_NONE, "relu": B2_ACT_RELU, "sigmoid": B2_ACT_SIGMOID}


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else ctypes.c_void_p(0)


def _require_cuda(*tensors):
    for t in tensors:
        if t is not None and not t.is_cuda:
            raise RuntimeError("fuxictr_b200 kernels need CUDA tensors (got device=%s); "
                               "there is no CPU path" % t.device)


def _f32c(t):
    """Contiguous fp32 view/copy of an activation (no-op in the steady state)."""
    if t.dtype != torch.float32:
        t = t.float()
    return t if t.is_contiguous() else t.contiguous()


# --------------------------------------------------------------------------------------
# Gradient arena hook: a parameter whose gradient should be produced in place inside a
# flat arena carries `_b2_grad_view` (set by fuxictr_b200.arena.ParamArena).  Backward
# kernels write there (no extra copy, no per-tensor allocation) the first time the
# parameter is hit in a step; a second hit falls back to a fresh tensor so autograd can
# accumulate.
# --------------------------------------------------------------------------------------
def _grad_buffer(param, zero, marks=False):
    """marks: the caller's kernel flags every granule it writes (ParamArena.touched, passed as _touch());
    any other writer into the arena's table prefix gets the whole slot flagged here."""
    slot = getattr(param, "_b2_slot", None)
    if slot is not None:
        arena = slot.arena
        if param.grad is None and slot.step_mark != arena.step_id:  # first hit this step
            slot.step_mark = arena.step_id
            view = arena.grad_view(slot)  # a fresh view object, so AccumulateGrad can steal it
            if zero and not arena.grads_are_zero:
                view.zero_()
            if not marks:
                arena.mark_slot(slot)
            return view
        # the buffer below reaches the arena through AccumulateGrad's in-place add or the step's p.grad copy
        arena.mark_slot(slot)
        # ... and that add or copy reads the first gradient, which a deferred side stream may still be writing
        arena.join_grads()
    return torch.zeros_like(param) if zero else torch.empty_like(param)


def _touch(bufs):
    """byref(b2_touch) of the arena the gradient buffers `bufs` live in, or None (no flags to set)."""
    for b in bufs:
        base = b._base if b is not None else None
        arena = getattr(base, "_b2_arena", None) if base is not None else None
        if arena is not None and arena.touch is not None:
            return ctypes.byref(arena.touch)
    return None


def _is_zeroed(buf):
    """True when `buf` is a gradient-arena slice that the optimizer pass left all-zero (so a kernel that
    accumulates into it needs no memset node of its own)."""
    base = buf._base if buf is not None else None
    arena = getattr(base, "_b2_arena", None) if base is not None else None
    return arena is not None and arena.grads_are_zero


# --------------------------------------------------------------------------------------
# Fused multi-field embedding gather
# --------------------------------------------------------------------------------------
class GatherField(object):
    """Static description of one feature of a fused gather (see struct b2_field)."""
    __slots__ = ("name", "table_slot", "dim", "seq_len", "pool", "padding_idx", "out_offset",
                 "out_width")

    def __init__(self, name, table_slot, dim, seq_len=1, pool=B2_POOL_NONE, padding_idx=-1,
                 out_offset=0):
        self.name = name
        self.table_slot = table_slot  # index into the de-duplicated weight tuple
        self.dim = dim
        self.seq_len = seq_len
        self.pool = pool
        self.padding_idx = -1 if padding_idx is None else int(padding_idx)
        self.out_offset = out_offset  # element offset inside one sample's arena row
        pooled = seq_len > 1 and pool != B2_POOL_NONE
        self.out_width = dim if (seq_len == 1 or pooled) else seq_len * dim


class GatherPlan(object):
    """Layout of one fused launch: fields, arena width, persistent descriptor array."""

    def __init__(self, fields):
        self.fields = list(fields)
        if not 1 <= len(self.fields) <= _lib.B2_MAX_FIELDS:
            raise ValueError("a fused gather takes 1..%d fields, got %d"
                             % (_lib.B2_MAX_FIELDS, len(self.fields)))
        off = 0
        for f in self.fields:
            f.out_offset = off
            off += f.out_width
        self.width = off
        self.hot_rows = 0       # > 0: stage that many leading (most frequent) rows of every table in shared memory
        self.needs_count = any(f.seq_len > 1 and f.pool == B2_POOL_MEAN for f in self.fields)
        self.widths = [f.out_width for f in self.fields]
        self._descs = (b2_field * len(self.fields))()
        for d, f in zip(self._descs, self.fields):
            d.dim, d.seq_len, d.pool, d.padding_idx = f.dim, f.seq_len, f.pool, f.padding_idx

    def fill(self, tables, idx_list, arena, batch):
        """Point the descriptors at this call's tables / index views / arena rows."""
        esz = 4
        base = arena.data_ptr()
        for d, f, idx in zip(self._descs, self.fields, idx_list):
            t = tables[f.table_slot]
            d.table = t.data_ptr()
            d.vocab = t.shape[0]
            d.idx = idx.data_ptr()
            d.idx_stride = idx.stride(0) if batch > 0 else 0
            d.out = base + f.out_offset * esz
            d.out_stride = self.width
        return self._descs


def _prep_indices(idx_list, fields):
    """Validate/normalise the per-feature index views; returns (list, dtype code)."""
    dtype = idx_list[0].dtype
    if dtype not in _IDX_CODE or any(t.dtype != dtype for t in idx_list):
        # mixed or exotic dtypes: fall back to the reference's own cast (.long())
        idx_list = [t.long() for t in idx_list]
        dtype = torch.int64
    out = []
    for t, f in zip(idx_list, fields):
        if f.seq_len > 1:
            if t.dim() != 2 or t.shape[1] != f.seq_len:
                raise ValueError("feature %s: expected (B, %d) indices, got %s"
                                 % (f.name, f.seq_len, tuple(t.shape)))
            if t.stride(1) != 1:
                t = t.contiguous()
        else:
            if t.dim() == 2 and t.shape[1] == 1:
                t = t[:, 0]
            if t.dim() != 1:
                raise ValueError("feature %s: expected (B,) indices, got %s" % (f.name, tuple(t.shape)))
        out.append(t)
    return out, _IDX_CODE[dtype]


class _EmbedGather(torch.autograd.Function):
    """arena[b, off_f : off_f + w_f] = rows of table_f (one launch for all features).

    Reference: FeatureEmbeddingDict.forward + dict2tensor
    (fuxictr/pytorch/layers/embeddings/feature_embedding.py:261-297, 230-259).
    """

    @staticmethod
    def forward(ctx, plan, idx_list, status, *tables):
        batch = idx_list[0].shape[0]
        dev = tables[0].device
        arena = torch.empty((batch, plan.width), dtype=torch.float32, device=dev)
        count = (torch.empty((len(plan.fields), max(batch, 1)), dtype=torch.float32, device=dev)
                 if plan.needs_count else None)
        descs = plan.fill(tables, idx_list, arena, batch)
        _lib.call("b2_embed_gather_fwd", descs, len(plan.fields), batch, ctx_code(idx_list),
                  B2_F32, _ptr(count), _ptr(status), int(plan.hot_rows), _stream())
        ctx.plan, ctx.idx_list, ctx.count, ctx.tables = plan, idx_list, count, tables
        return arena

    @staticmethod
    def backward(ctx, garena):
        plan, idx_list, tables = ctx.plan, ctx.idx_list, ctx.tables
        batch = idx_list[0].shape[0]
        garena = _f32c(garena)
        grads = [None] * len(tables)
        for slot, t in enumerate(tables):
            if t.requires_grad:
                grads[slot] = _grad_buffer(t, zero=True, marks=True)
        live = [(f, idx) for f, idx in zip(plan.fields, idx_list) if grads[f.table_slot] is not None]
        if live and batch > 0:
            descs = (b2_field * len(live))()
            base = garena.data_ptr()
            for d, (f, idx) in zip(descs, live):
                g = grads[f.table_slot]
                d.table, d.vocab = g.data_ptr(), g.shape[0]
                d.idx, d.idx_stride = idx.data_ptr(), idx.stride(0)
                d.out, d.out_stride = base + f.out_offset * 4, plan.width
                d.dim, d.seq_len, d.pool, d.padding_idx = f.dim, f.seq_len, f.pool, f.padding_idx
            count = ctx.count
            if count is not None:
                # mean_count is indexed by the position in the *backward* field list
                rows = [plan.fields.index(f) for f, _ in live]
                count = count[rows].contiguous()
            _lib.call("b2_embed_scatter_bwd", descs, len(live), batch, ctx_code(idx_list), B2_F32,
                      _ptr(count), _touch(grads), _stream())
        return (None, None, None) + tuple(grads)


def ctx_code(idx_list):
    return _IDX_CODE[idx_list[0].dtype]


def embed_gather(plan, idx_list, tables, status=None):
    """Run the fused gather; returns the (B, plan.width) arena (differentiable w.r.t. tables)."""
    _require_cuda(*tables)
    _require_cuda(*idx_list)
    for t in tables:
        if t.dtype != torch.float32 or not t.is_contiguous():
            raise RuntimeError("embedding tables must be contiguous float32")
    idx_list, _ = _prep_indices(list(idx_list), plan.fields)
    return _EmbedGather.apply(plan, idx_list, status, *tables)


# --------------------------------------------------------------------------------------
# LogisticRegression gather-reduce
# --------------------------------------------------------------------------------------
class _LRForward(torch.autograd.Function):
    """out[b,0] = sum_f w_f[idx_f[b]] (+ bias).  logistic_regression.py:55-58."""

    @staticmethod
    def forward(ctx, plan, idx_list, status, bias, *tables):
        batch = idx_list[0].shape[0]
        out = torch.empty((batch, 1), dtype=torch.float32, device=tables[0].device)
        descs = plan._descs
        for d, f, idx in zip(descs, plan.fields, idx_list):
            t = tables[f.table_slot]
            d.table, d.vocab = t.data_ptr(), t.shape[0]
            d.idx, d.idx_stride = idx.data_ptr(), (idx.stride(0) if batch > 0 else 0)
            d.out, d.out_stride = 0, 0
        _lib.call("b2_lr_fwd", descs, len(plan.fields), batch, ctx_code(idx_list), _ptr(bias),
                  _ptr(out), _ptr(status), _stream())
        ctx.plan, ctx.idx_list, ctx.tables, ctx.bias = plan, idx_list, tables, bias
        return out

    @staticmethod
    def backward(ctx, gout):
        plan, idx_list, tables, bias = ctx.plan, ctx.idx_list, ctx.tables, ctx.bias
        batch = idx_list[0].shape[0]
        gout = _f32c(gout).view(-1)
        grads = [None] * len(tables)
        for slot, t in enumerate(tables):
            if t.requires_grad:
                grads[slot] = _grad_buffer(t, zero=True, marks=True)
        gbias = None
        if bias is not None and bias.requires_grad:
            gbias = _grad_buffer(bias, zero=True)
        live = [(f, idx) for f, idx in zip(plan.fields, idx_list) if grads[f.table_slot] is not None]
        if batch > 0 and (live or gbias is not None):
            if live:
                descs = (b2_field * len(live))()
                for d, (f, idx) in zip(descs, live):
                    g = grads[f.table_slot]
                    d.table, d.vocab = g.data_ptr(), g.shape[0]
                    d.idx, d.idx_stride = idx.data_ptr(), idx.stride(0)
                    d.dim, d.seq_len, d.pool, d.padding_idx = 1, f.seq_len, f.pool, f.padding_idx
                _lib.call("b2_lr_bwd", descs, len(live), batch, ctx_code(idx_list), _ptr(gout),
                          _ptr(gbias), _touch(grads), _stream())
            else:
                gbias.copy_(gout.sum().view(1))
        return (None, None, None, gbias) + tuple(grads)


def lr_forward(plan, idx_list, tables, bias=None, status=None):
    _require_cuda(*tables)
    _require_cuda(*idx_list)
    idx_list, _ = _prep_indices(list(idx_list), plan.fields)
    return _LRForward.apply(plan, idx_list, status, bias, *tables)


# --------------------------------------------------------------------------------------
# InnerProductInteraction
# --------------------------------------------------------------------------------------
class _FMInteraction(torch.autograd.Function):
    """inner_product.py:55-66 (product_sum / bi_interaction / inner_product)."""

    @staticmethod
    def forward(ctx, emb, mode):
        emb = _f32c(emb)
        B, F, D = emb.shape
        if mode == _lib.FM_PRODUCT_SUM:
            out = torch.empty((B, 1), dtype=torch.float32, device=emb.device)
        elif mode == _lib.FM_BI_INTERACTION:
            out = torch.empty((B, D), dtype=torch.float32, device=emb.device)
        else:
            out = torch.empty((B, F * (F - 1) // 2), dtype=torch.float32, device=emb.device)
        _lib.call("b2_fm_fwd", _ptr(emb), B, F, D, mode, _ptr(out), _stream())
        ctx.save_for_backward(emb)
        ctx.mode = mode
        return out

    @staticmethod
    def backward(ctx, gout):
        (emb,) = ctx.saved_tensors
        B, F, D = emb.shape
        gout = _f32c(gout)
        gemb = torch.empty_like(emb)
        _lib.call("b2_fm_bwd", _ptr(emb), _ptr(gout), B, F, D, ctx.mode, _ptr(gemb), _stream())
        return gemb, None


def fm_interaction(emb, mode):
    _require_cuda(emb)
    if emb.dim() != 3:
        raise ValueError("feature_emb must be (batch, num_fields, embedding_dim)")
    return _FMInteraction.apply(emb, mode)


# --------------------------------------------------------------------------------------
# CrossNet (rank-1)
# --------------------------------------------------------------------------------------
class _CrossNet(torch.autograd.Function):
    """cross_net.py:80-92 with all layers fused; w, b are (L, d)."""

    @staticmethod
    def forward(ctx, x0, w, b):
        x0, w, b = _f32c(x0), _f32c(w), _f32c(b)
        B, d = x0.shape
        L = w.shape[0]
        out = torch.empty_like(x0)
        s = torch.empty((B, L), dtype=torch.float32, device=x0.device)
        _lib.call("b2_crossnet_fwd", _ptr(x0), _ptr(w), _ptr(b), B, d, L, _ptr(out), _ptr(s), _stream())
        ctx.save_for_backward(x0, w, b, s)
        return out

    @staticmethod
    def backward(ctx, gout):
        x0, w, b, s = ctx.saved_tensors
        B, d = x0.shape
        L = w.shape[0]
        gout = _f32c(gout)
        gx0 = torch.empty_like(x0)
        gw = torch.zeros_like(w)
        gb = torch.zeros_like(b)
        if L > 0:
            _lib.call("b2_crossnet_bwd", _ptr(x0), _ptr(w), _ptr(b), _ptr(s), _ptr(gout), B, d, L,
                      _ptr(gx0), _ptr(gw), _ptr(gb), _stream())
        else:
            gx0.copy_(gout)
        return gx0, gw, gb


def crossnet(x0, w, b):
    _require_cuda(x0, w, b)
    return _CrossNet.apply(x0, w, b)


# --------------------------------------------------------------------------------------
# Dense layer (fp32 parity path)
# --------------------------------------------------------------------------------------
def gemm_f32(a, b, out, a_t=False, b_t=False, bias=None, act=B2_ACT_NONE, mul=None, add=None,
             accumulate=False):
    """out (M,N) = epi(op(a) @ op(b)); a is (M,K) [or (K,M) if a_t], b is (K,N) [or (N,K) if b_t]."""
    if a_t:
        K, M = a.shape
        a_rs, a_cs = a.stride(1), a.stride(0)
    else:
        M, K = a.shape
        a_rs, a_cs = a.stride(0), a.stride(1)
    if b_t:
        N, K2 = b.shape
        b_rs, b_cs = b.stride(1), b.stride(0)
    else:
        K2, N = b.shape
        b_rs, b_cs = b.stride(0), b.stride(1)
    if K != K2 or tuple(out.shape) != (M, N) or out.stride(1) != 1:
        raise ValueError("gemm shape mismatch: a%s b%s out%s" % (tuple(a.shape), tuple(b.shape), tuple(out.shape)))
    for t in (mul, add):        # the kernel reads them at out's element offsets
        if t is not None and (tuple(t.shape) != (M, N) or t.stride() != out.stride()):
            raise ValueError("gemm_f32: mul and add must share out's shape and leading dimension")
    _lib.call("b2_gemm_f32", _ptr(a), a_rs, a_cs, _ptr(b), b_rs, b_cs, _ptr(out), out.stride(0), M, N, K,
              _ptr(bias), act, _ptr(mul), _ptr(add), 1 if accumulate else 0, _stream())
    return out


# Matmul arithmetic of the dense layers:
#   "fp32"   FFMA SIMT kernel (b2_gemm_f32)                       — bit-for-bit the reference's class
#   "tf32x3" wgmma tensor cores, error-compensated 3xTF32         — fp32-class accuracy (1e-5 parity)
#   "tf32"   wgmma tensor cores, single TF32 pass (10-bit mantissa, >= the bf16 of BASELINE configs[1])
#   "bf16"   wgmma .bf16 on bf16 copies of the operands, fp32 accumulation (BASELINE configs[1] "bf16");
#            activations / weights / gradients stay fp32 in HBM, every producer also emits the bf16 operand
#            3xTF32 reads the fp32 operands alone and derives the small parts in shared memory inside the
#            GEMM (B2_GEMM_X3_INLINE, default); set_x3_inline(False) / B2_X3_INLINE=0 exercises the ABI's other
#            3xTF32 form: producers also write small parts to HBM and pass them as a_small / b_small, which the
#            GEMM does not read — extra launches and traffic for identical results, kept for testing that form
_MATMUL = {"mode": "fp32", "x3_inline": os.environ.get("B2_X3_INLINE", "1") != "0"}


def set_x3_inline(on):
    _MATMUL["x3_inline"] = bool(on)


def _x3_aux():
    """True when 3xTF32 wants auxiliary small-part tensors in HBM (the non-inline layout)."""
    return _MATMUL["mode"] == "tf32x3" and not _MATMUL["x3_inline"]


def set_matmul_precision(mode):
    if mode not in ("fp32", "tf32x3", "tf32", "bf16"):
        raise ValueError("matmul precision must be 'fp32', 'tf32x3', 'tf32' or 'bf16'")
    _MATMUL["mode"] = mode


def get_matmul_precision():
    return _MATMUL["mode"]


def _tc_operand_ok(t):
    return t.dim() == 2 and t.stride(1) == 1 and t.stride(0) % 4 == 0 and t.data_ptr() % 16 == 0 \
        and t.stride(0) >= t.shape[1]


def split_tf32(t):
    """small part of a contiguous fp32 tensor for 3xTF32."""
    small = torch.empty_like(t)
    _lib.call("b2_split_tf32", _ptr(t), _ptr(small), t.numel(), _stream())
    return small


def gemm_ex(a, b, out, a_mn=False, b_mn=False, a_small=None, b_small=None, bias=None, act=B2_ACT_NONE,
            mul=None, add=None, ybwd=None, act_bwd=B2_ACT_NONE, out_small=None, colsum=None, accumulate=False,
            out_pre=None, out_is_zero=False, backfill=False, drop=None):
    """out (M,N) = epi(sum_k A(m,k) B(n,k)) on the wgmma kernel (b2_gemm_tc_ex).  a is (M,K), or (K,M) when
    a_mn (MN-major: the tensor is consumed as it lies, no transpose); b is (N,K), or (K,N) when b_mn.
    a_small / b_small: the operands' 3xTF32 small parts (both or neither).  Epilogue extras: ybwd/act_bwd
    (activation backward of the gradient's producer), out_small (3xTF32 small part of out), colsum (N).
    backfill: the launch runs beside a chain of launches on another stream (B2_GEMM_BACKFILL: short split-K CTAs).
    drop: (snapshot, layer, thresh, scale), the dropout mask of out's (M, N) elements (see dropout_snapshot)."""
    d = _lib.b2_gemm_desc()
    K, M = (a.shape if a_mn else a.shape[::-1])
    K2, N = (b.shape if b_mn else b.shape[::-1])
    if K != K2 or tuple(out.shape) != (M, N) or out.stride(1) != 1 or a.stride(1) != 1 or b.stride(1) != 1:
        raise ValueError("gemm_ex shape mismatch: a%s b%s out%s" % (tuple(a.shape), tuple(b.shape), tuple(out.shape)))
    for t in (mul, add, ybwd, out_pre) + ((out_small,) if (out_small is not None and out_small.dtype == torch.float32) else ()):
        if t is not None and (tuple(t.shape) != (M, N) or t.stride(0) != out.stride(0) or t.stride(1) != 1):
            raise ValueError("gemm_ex: epilogue tensors must share out's shape and leading dimension")
    bf16 = a_small is not None and a_small.dtype == torch.bfloat16
    if bf16:        # the auxiliary tensors ARE the operands (bf16 copies, row pitch padded to 16 bytes)
        if b_small is None or b_small.dtype != torch.bfloat16 or a_small.shape != a.shape or b_small.shape != b.shape:
            raise ValueError("gemm_ex: bf16 mode needs bf16 copies of both operands")
        a, b, a_small, b_small = a_small, b_small, None, None
        d.elem_dtype = B2_BF16
    for t, ref in ((a_small, a), (b_small, b)):
        if t is not None and (t.shape != ref.shape or t.stride() != ref.stride()):
            raise ValueError("gemm_ex: small parts must share their operand's layout")
    d.a, d.b = a.data_ptr(), b.data_ptr()
    d.a_small = a_small.data_ptr() if a_small is not None else None
    d.b_small = b_small.data_ptr() if b_small is not None else None
    d.c = out.data_ptr()
    d.c_small = out_small.data_ptr() if out_small is not None else None
    if out_small is not None:
        if (out_small.dtype == torch.bfloat16) != bf16:
            raise ValueError("gemm_ex: out_small dtype does not match the operand mode")
        d.ld_aux = out_small.stride(0)
    d.c_pre = out_pre.data_ptr() if out_pre is not None else None
    d.bias = bias.data_ptr() if bias is not None else None
    d.mul = mul.data_ptr() if mul is not None else None
    d.add = add.data_ptr() if add is not None else None
    d.ybwd = ybwd.data_ptr() if ybwd is not None else None
    d.colsum = colsum.data_ptr() if colsum is not None else None
    d.lda, d.ldb, d.ldc = a.stride(0), b.stride(0), out.stride(0)
    d.M, d.N, d.K = M, N, K
    d.a_mn_major, d.b_mn_major = int(bool(a_mn)), int(bool(b_mn))
    d.act, d.act_bwd = act, (act_bwd if ybwd is not None else B2_ACT_NONE)
    d.beta_accumulate = 1 if accumulate else 0
    d.flags = (_lib.B2_GEMM_C_IS_ZERO if out_is_zero else 0) | (_lib.B2_GEMM_COLSUM_IS_ZERO if _is_zeroed(colsum) else 0) \
        | (_lib.B2_GEMM_BACKFILL if backfill else 0)
    if a_small is None and not bf16 and _MATMUL["mode"] == "tf32x3" and _MATMUL["x3_inline"]:
        d.flags |= _lib.B2_GEMM_X3_INLINE
    if drop is not None:
        d.drop_rng, d.drop_layer, d.drop_thresh, d.drop_scale = drop[0].data_ptr(), drop[1], drop[2], drop[3]
    _lib.call("b2_gemm_tc_ex", ctypes.byref(d), _stream())
    return out


def gemm_nt(a, b, out, bias=None, act=B2_ACT_NONE, mul=None, add=None, accumulate=False,
            a_small=None, b_small=None):
    """out (M,N) = epi(a (M,K) @ b (N,K)^T) in the configured matmul precision."""
    mode = _MATMUL["mode"]
    N = b.shape[0]
    use_tc = (mode != "fp32" and N >= 16 and _tc_operand_ok(a) and _tc_operand_ok(b) and out.stride(1) == 1)
    if not use_tc:
        return gemm_f32(a, b, out, b_t=True, bias=bias, act=act, mul=mul, add=add, accumulate=accumulate)
    if mode in ("tf32x3", "bf16"):
        if a_small is None:
            a_small = make_aux(a)
        if b_small is None:
            b_small = make_aux(b)
    else:
        a_small = b_small = None
    return gemm_ex(a, b, out, a_small=a_small, b_small=b_small, bias=bias, act=act, mul=mul, add=add,
                   accumulate=accumulate)


# ---- 3xTF32 small parts of WEIGHTS: one split per weight per optimizer step -------------------
# A weight changes once per step; its small part is cached until the weight's version changes.
# torch bumps `_version` for in-place ops; updates through raw pointers (the fused arena optimizer,
# CUDA-graph replays of it) are announced with bump_weight_epoch().
_WEIGHT_EPOCH = [0]
_SMALL_CACHE = {}      # id(weight) -> (key, aux, weakref to the weight)


def bump_weight_epoch():
    _WEIGHT_EPOCH[0] += 1


def _pad8(n):
    return (n + 7) // 8 * 8


def empty_aux(rows, cols, device):
    """Uninitialised auxiliary operand of a (rows, cols) fp32 tensor for the current precision: its 3xTF32
    small part (fp32, same layout), or its bf16 copy (row pitch padded to 16 bytes for TMA); None otherwise."""
    mode = _MATMUL["mode"]
    if _x3_aux():
        return torch.empty((rows, cols), dtype=torch.float32, device=device)
    if mode == "bf16":
        return torch.empty((rows, _pad8(cols)), dtype=torch.bfloat16, device=device)[:, :cols]
    return None


def make_aux(t):
    """The auxiliary operand of a contiguous-row fp32 matrix `t` (see empty_aux), computed in one launch."""
    mode = _MATMUL["mode"]
    if mode == "tf32x3" and not _x3_aux():
        return None
    base = t._base if t._base is not None else t
    hint = getattr(base, "_b2_aux", None)       # the producer already emitted it (fused front -> first MLP layer)
    if hint is not None and hint[0] == mode and hint[2] == base._version and t.is_contiguous() \
            and t.data_ptr() == base.data_ptr() and hint[1].numel() == t.numel():
        return hint[1].view(t.shape)
    if mode == "tf32x3":
        return split_tf32(t if t.is_contiguous() else t.contiguous())
    if mode == "bf16":
        rows, cols = t.shape
        out = empty_aux(rows, cols, t.device)
        _lib.call("b2_to_bf16", _ptr(t), rows, cols, t.stride(0), _ptr(out), out.stride(0), _stream())
        return out
    return None


def weight_aux(w):
    """Auxiliary operand of a WEIGHT, cached until the weight changes (see bump_weight_epoch)."""
    mode = _MATMUL["mode"]
    if mode != "bf16" and not _x3_aux():
        return None
    if not w.is_contiguous():
        raise RuntimeError("tensor-core GEMM weights must be contiguous")
    slot = getattr(w, "_b2_slot", None)
    if mode == "tf32x3" and slot is not None and slot.offset >= slot.arena.tail_offset > 0:
        # the dense parameters of an arena are one contiguous slice: ONE split launch per optimizer step
        # serves every Linear of the model (the small part has the operand's own layout)
        arena = slot.arena
        key = (_WEIGHT_EPOCH[0], arena.P.data_ptr(), tuple(p._version for p in arena.tail_params))
        ent = getattr(arena, "_tail_small", None)
        if ent is None or ent[0] != key:
            ent = (key, split_tf32(arena.P[arena.tail_offset:arena.numel]))
            arena._tail_small = ent
        off = slot.offset - arena.tail_offset
        return ent[1][off:off + slot.numel].view(slot.shape)
    key = (mode, w.data_ptr(), w._version, _WEIGHT_EPOCH[0], tuple(w.shape))
    ent = _SMALL_CACHE.get(id(w))
    if ent is not None and ent[0] == key and ent[2]() is w:
        return ent[1]
    aux = make_aux(w.detach())
    wid = id(w)
    _SMALL_CACHE[wid] = (key, aux, weakref.ref(w, lambda _r, wid=wid: _SMALL_CACHE.pop(wid, None)))
    return aux


def prep_operand(x, y=None, act=B2_ACT_NONE, want_out=False, want_small=False, want_t=False,
                 want_t_small=False, colsum=None, drop=None):
    """One pass over x (R, C): [dropout mask (drop = (snapshot, layer, thresh, scale)), act-backward with y]
    -> out / out_small / out^T / out^T_small / column sums."""
    R, C = x.shape
    dev = x.device
    out = torch.empty((R, C), dtype=torch.float32, device=dev) if want_out else None
    small = torch.empty((R, C), dtype=torch.float32, device=dev) if want_small else None
    out_t = torch.empty((C, R), dtype=torch.float32, device=dev) if want_t else None
    t_small = torch.empty((C, R), dtype=torch.float32, device=dev) if want_t_small else None
    snap, layer, thresh, scale = drop if drop is not None else (None, 0, 0, 0.0)
    _lib.call("b2_prep_operand", _ptr(x), _ptr(y), act, R, C, _ptr(out), _ptr(small), _ptr(out_t), _ptr(t_small),
              _ptr(colsum), _ptr(snap), layer, thresh, scale, _stream())
    return out, small, out_t, t_small


def _grad_operand(g, y, act, tc, colsum=None, drop=None):
    """The gradient g of a layer's output as the dZ operand of its dgrad and wgrad, in one pass over g
    (prep_operand): the dropout mask `drop` regenerated, the backward of `act` with the output y (B2_PREP_MUL:
    g * y), the column sums (bias gradient) added to `colsum`.  Returns (dZ, its auxiliary operand): dZ is g
    itself when the pass changes no value; the auxiliary operand is what the matmul precision wants of a
    tensor-core operand (see empty_aux, None without `tc`), written by the same pass where the kernel can."""
    if act == B2_ACT_NONE:
        y = None
    keep = y is not None or drop is not None
    out, aux, _, _ = prep_operand(g, y, act, want_out=keep, want_small=tc and _x3_aux(), colsum=colsum, drop=drop)
    gz = out if keep else g
    if tc and aux is None:
        aux = make_aux(gz)          # bf16 mode (None for single-pass TF32 and in-kernel 3xTF32)
    return gz, aux


# ---- dropout masks of MLP chains (include/fuxictr_b200.h "Dropout masks", csrc/philox.cuh) -------------------
# One {seed, offset} int64 pair per device.  Its seed is drawn from torch's generator of that device on first eager
# use, and drawn again on the first eager use after torch.manual_seed (so seed_everything governs the masks as it
# governs nn.Dropout).  Every chain forward with dropout snapshots it on the device and advances its offset, so a
# CUDA graph replay reads and advances the device state: fresh masks every replay, no host value in the graph.
_DROPOUT = {}       # device -> [state tensor, torch.initial_seed() it was drawn under]


def dropout_consts(p):
    """(thresh, scale) of a dropout probability 0 < p < 1: keep iff the Philox word < thresh; kept x -> x * scale."""
    if not 0.0 < p < 1.0:
        raise ValueError("dropout probability must lie in (0, 1), got %r" % (p,))
    thresh = min(int(round((1.0 - p) * 4294967296.0)), 4294967295)
    return thresh, float(ctypes.c_float(1.0 / (1.0 - p)).value)


def dropout_state(dev):
    """The device's {seed, offset} state (int64[2]), drawn when absent or torch.manual_seed changed it.  Never
    drawn inside a CUDA graph capture: an eager forward (TrainPipeline's warm-up steps) must create it first."""
    dev = torch.device(dev)
    capturing = dev.type == "cuda" and torch.cuda.is_current_stream_capturing()
    ent = _DROPOUT.get(dev)
    seed_now = torch.initial_seed()
    if ent is not None and (ent[1] == seed_now or capturing):
        return ent[0]
    if capturing:
        raise RuntimeError("the dropout RNG state of %s is created by an eager forward; run one before capturing "
                           "a CUDA graph" % dev)
    seed = torch.randint(0, 1 << 62, (1,), dtype=torch.int64, device=dev)
    state = torch.cat([seed, torch.zeros(1, dtype=torch.int64, device=dev)])
    _DROPOUT[dev] = [state, seed_now]
    return state


def dropout_snapshot(dev, n_layers):
    """Snapshot the device's dropout state and advance its offset by n_layers (one launch); layer l of the
    forward draws its mask at offset snapshot.offset + l."""
    state = dropout_state(dev)
    snap = torch.empty(2, dtype=torch.int64, device=state.device)
    _lib.call("b2_dropout_rng_take", _ptr(state), _ptr(snap), n_layers, _stream())
    return snap


def dropout_apply(x, snap, layer, p, out=None):
    """out (M, N) = keep ? x * scale : 0 with the mask of layer `layer` of snapshot `snap` (out may be x)."""
    thresh, scale = dropout_consts(p)
    M, N = x.shape
    if out is None:
        out = torch.empty_like(x)
    if x.stride(1) != 1 or out.stride() != x.stride():
        raise ValueError("dropout_apply: x and out must share one row-major layout")
    _lib.call("b2_dropout_apply", _ptr(x), _ptr(out), M, N, x.stride(0), _ptr(snap), layer, thresh, scale, _stream())
    return out


def _tc_layer_ok(weight):
    """nn.Linear weight (N, K) usable by the tensor-core kernel in all three contractions
    (Y = X W^T, dX = dZ W, dW = dZ^T X): TMA needs 16-byte bases and leading dimensions % 4."""
    N, K = weight.shape
    return (_MATMUL["mode"] != "fp32" and N >= 16 and K >= 16 and N % 4 == 0 and K % 4 == 0
            and weight.is_contiguous() and weight.data_ptr() % 16 == 0)


def _head_ok(weight):
    """nn.Linear weight (1, K) that the N = 1 head kernels take: contiguous, K within the backward's
    shared-memory staging (B2_HEAD_MAX_K).  A wider one runs as a general GEMM."""
    return weight.shape[0] == 1 and weight.shape[1] <= _lib.B2_HEAD_MAX_K and weight.is_contiguous()


def _linear_fwd(tc, a, a_aux, W, out, w_aux=None, **epilogue):
    """out = epi(a W^T), W (N, K) as nn.Linear keeps it: on the tensor cores (a_aux, w_aux: the operands' auxiliary
    ones; w_aux None: weight_aux(W), a parameter's cached one, itself None in a precision that has none) or,
    without tc, on the SIMT GEMM.  The epilogue keywords are gemm_ex's or gemm_f32's."""
    if tc:
        return gemm_ex(a, W, out, a_small=a_aux, b_small=weight_aux(W) if w_aux is None else w_aux, **epilogue)
    return gemm_f32(a, W, out, b_t=True, **epilogue)


def _linear_dgrad(tc, gz, gz_aux, W, gx, w_aux=None, **epilogue):
    """dX = epi(dZ W): W is consumed as it lies in memory (MN-major), no transpose in HBM."""
    if tc:
        return gemm_ex(gz, W, gx, b_mn=True, a_small=gz_aux, b_small=weight_aux(W) if w_aux is None else w_aux,
                       **epilogue)
    return gemm_f32(gz, W, gx, **epilogue)


def _linear_wgrad(tc, gz, gz_aux, a, a_aux, gw, fork=None, ready=None, backfill=False):
    """dW = dZ^T X, dZ and X (the forward's `a`, with the auxiliary operand the forward made) both MN-major.
    ready: fork.ready() recorded before the dgrad was launched; the GEMM then runs on the fork's side stream."""
    if ready is not None:
        return fork.gemm(ready, gz, gz_aux, a, a_aux, gw)
    if tc:
        return gemm_ex(gz, a, gw, a_mn=True, b_mn=True, a_small=gz_aux, b_small=a_aux, out_is_zero=_is_zeroed(gw),
                       backfill=backfill)
    return gemm_f32(gz, a, gw, a_t=True)


class _LinearAct(torch.autograd.Function):
    """y = act(x W^T + b): nn.Linear (+ReLU/Sigmoid) of MLP_Block (mlp_block.py:74-80).

    Three arithmetic paths: the N = 1 output head (GEMV kernels), the wgmma tensor-core GEMM
    (TF32 / 3xTF32; dX and dW consume W, dZ and X as they lie in memory as MN-major operands —
    no transposes in HBM), and the fp32 SIMT GEMM.  The backward fuses activation-backward,
    the 3xTF32 split and the bias gradient into a single pass over dY."""

    @staticmethod
    def forward(ctx, x, weight, bias, act):
        x = _f32c(x)
        M, K = x.shape
        N = weight.shape[0]
        y = torch.empty((M, N), dtype=torch.float32, device=x.device)
        ctx.act, ctx.bias, ctx.has_bias = act, bias, bias is not None
        if _head_ok(weight):
            ctx.kind = "head"
            _lib.call("b2_head_fwd", _ptr(x), _ptr(weight), _ptr(bias), M, K, act, _ptr(y), _stream())
        else:
            tc = _tc_layer_ok(weight) and x.data_ptr() % 16 == 0
            ctx.kind = "tc" if tc else "simt"
            ctx.x_small = make_aux(x) if tc else None
            _linear_fwd(tc, x, ctx.x_small, weight, y, bias=bias, act=act)
        ctx.save_for_backward(x, weight, y if act != B2_ACT_NONE else None)
        return y

    @staticmethod
    def backward(ctx, gy):
        x, weight, y = ctx.saved_tensors
        gy = _f32c(gy)
        M, K = x.shape
        act = ctx.act
        need_x, need_w = ctx.needs_input_grad[0], ctx.needs_input_grad[1]
        need_b = ctx.has_bias and ctx.needs_input_grad[2]
        gx = gw = gb = None
        if ctx.kind == "head":
            gx = torch.empty((M, K), dtype=torch.float32, device=x.device) if need_x else None
            gw = _grad_buffer(weight, zero=False)
            gb = _grad_buffer(ctx.bias, zero=False) if need_b else None
            _lib.call("b2_head_bwd", _ptr(x), _ptr(weight), _ptr(y), _ptr(gy), M, K, act, _ptr(gx), _ptr(gw),
                      _ptr(gb), _stream())
            return gx, gw, gb, None
        gb = _grad_buffer(ctx.bias, zero=False) if need_b else None
        tc = ctx.kind == "tc"
        gz, gz_aux = gy, None
        if tc or act != B2_ACT_NONE or gb is not None:      # a SIMT layer with nothing to undo or to sum takes dY as it is
            gz, gz_aux = _grad_operand(gy, y, act, tc, colsum=gb)
        if need_x:
            gx = torch.empty((M, K), dtype=torch.float32, device=x.device)
            _linear_dgrad(tc, gz, gz_aux, weight, gx)
        if need_w:
            gw = _grad_buffer(weight, zero=False)
            _linear_wgrad(tc, gz, gz_aux, x, ctx.x_small, gw)
        return gx, gw, gb, None


_FORK = {"on": True, "side": {}}     # the weight-gradient side stream of each device


def set_backward_fork(on):
    """on (default): an MLP chain's backward runs its weight-gradient GEMMs on a side stream (see _WgradFork);
    off: every launch on the current stream, one after another (the reference order the fork is tested against)."""
    _FORK["on"] = bool(on)


class _WgradFork(object):
    """The weight-gradient GEMMs of a chain backward on a side stream.  The data-gradient chain (head backward,
    then each dgrad) stays on the current stream; a wgrad waits only for the launch that produced its dZ, so it
    fills the SMs a dgrad's last wave leaves idle.  Launched as backfill (B2_GEMM_BACKFILL): split over K into
    short CTAs, so that none holds an SM for long when the next dgrad wants it.  (A launch priority does not
    help: the wgrads already run at the lowest, and raising the dgrads above them made the backward slower.)

    Everything is an event record / wait, so the fork and the join are captured into a CUDA graph as edges.
    The operands the side stream reads stay referenced until the join, after which the current stream can
    reuse their memory.  The join: the current stream waits for the side stream at the end of the backward,
    unless every weight gradient lives in a ParamArena whose fused optimizer defers it (ParamArena.defer_join):
    then the optimizer joins where it first reads the dense gradients."""

    def __init__(self, dev):
        side = _FORK["side"].get(dev)
        if side is None:
            side = _FORK["side"][dev] = torch.cuda.Stream(device=dev)
        self.main, self.side = torch.cuda.current_stream(dev), side
        self.keep, self.arenas = [], set()
        self.defer = True

    def ready(self):
        """Record, on the current stream, that dZ (and its auxiliary operand) are written: before the dgrad launch."""
        ev = torch.cuda.Event()
        ev.record(self.main)
        return ev

    def gemm(self, ready, gz, gz_small, h, h_small, gw):
        self.side.wait_event(ready)
        with torch.cuda.stream(self.side):
            _linear_wgrad(True, gz, gz_small, h, h_small, gw, backfill=True)
        self.keep += [gz, gz_small, h, h_small]
        base = gw._base
        arena = getattr(base, "_b2_arena", None) if base is not None else None
        if arena is None or not arena.defer_join:
            self.defer = False
        else:
            self.arenas.add(arena)

    def join(self):
        done = torch.cuda.Event()
        done.record(self.side)
        if self.defer and len(self.arenas) == 1:
            self.arenas.pop().pending.append((done, self.keep))
        else:
            self.main.wait_event(done)


class _MLPChain(torch.autograd.Function):
    """A whole Linear(+ReLU/Sigmoid) chain of MLP_Block (mlp_block.py:64-85) as ONE autograd node, so that
    work can move across layer boundaries: the forward epilogue of layer i writes the 3xTF32 small part
    layer i+1 consumes; the dgrad GEMM of layer i+1 applies layer i's activation backward in its
    epilogue and emits dZ_i, its small part and layer i's bias gradient directly (the N = 1 head does
    the same in its fused backward).  Launches per 3-hidden-layer MLP step: 15 (was 26).

    Dropout (drops: per-layer p, or None): layer i's output is act(z_i) * keep_i * scale_i, the mask applied by
    whichever launch writes it (the forward epilogue; b2_dropout_apply after a head or SIMT layer), so h_{i+1} holds
    the dropped value.  The forward takes one snapshot of the dropout state (dropout_snapshot) and keeps it for
    the backward, which regenerates each mask where it folds that layer's activation backward: the next layer's
    dgrad epilogue, the head backward, or the explicit pass (b2_prep_operand) at the top or below a SIMT layer."""

    @staticmethod
    def forward(ctx, x, acts, drops, *params):
        x = _f32c(x)
        M = x.shape[0]
        L = len(acts)
        Ws, bs = params[0::2], params[1::2]
        dl = [None] * L                 # per layer: (snapshot, ordinal, thresh, scale) of its dropout, or None
        n_drop = sum(1 for p in (drops or ()) if p > 0)
        snap = dropout_snapshot(x.device, n_drop) if n_drop else None
        for i, p in enumerate(drops or ()):
            if p > 0:
                dl[i] = (snap, sum(1 for q in drops[:i] if q > 0)) + dropout_consts(p)
        kinds = []
        for W in Ws:
            if _head_ok(W):
                kinds.append("head")
            elif _tc_layer_ok(W):
                kinds.append("tc")
            else:
                kinds.append("simt")
        hs = [x]
        smalls = [make_aux(x) if kinds[0] == "tc" else None]
        for i in range(L):
            W, b, act = Ws[i], bs[i], acts[i]
            N, K = W.shape
            h = hs[-1]
            y = torch.empty((M, N), dtype=torch.float32, device=x.device)
            want_small = i + 1 < L and kinds[i + 1] == "tc"
            y_small = None
            if kinds[i] == "head":
                _lib.call("b2_head_fwd", _ptr(h), _ptr(W), _ptr(b), M, K, act, _ptr(y), _stream())
            elif kinds[i] == "tc" and h.data_ptr() % 16 == 0:
                y_small = empty_aux(M, N, x.device) if want_small else None
                _linear_fwd(True, h, smalls[-1], W, y, bias=b, act=act, out_small=y_small, drop=dl[i])
            else:
                kinds[i] = "simt"
                _linear_fwd(False, h, None, W, y, bias=b, act=act)
            if dl[i] is not None and kinds[i] != "tc":
                dropout_apply(y, snap, dl[i][1], drops[i], out=y)
            if want_small and y_small is None:
                y_small = make_aux(y)
            hs.append(y)
            smalls.append(y_small)
        ctx.acts, ctx.kinds, ctx.smalls, ctx.params, ctx.dl = acts, kinds, smalls, params, dl
        ctx.save_for_backward(*hs)
        return hs[-1]

    @staticmethod
    def backward(ctx, gy):
        hs = ctx.saved_tensors
        acts, kinds, smalls, params, dl = ctx.acts, ctx.kinds, ctx.smalls, ctx.params, ctx.dl
        Ws, bs = params[0::2], params[1::2]
        L = len(acts)
        M = hs[0].shape[0]
        dev = hs[0].device
        grads = [None] * len(params)

        def bias_buf(i):
            b = bs[i]
            return _grad_buffer(b, zero=False) if (b is not None and b.requires_grad) else None

        g, g_small, g_is_dz = _f32c(gy), None, False     # g: gradient w.r.t. y_i; g_is_dz: already dZ_i (+ db_i done)
        fork = None                                      # _WgradFork: the wgrads run beside the dgrad chain
        for i in range(L - 1, -1, -1):
            W, act, h, y = Ws[i], acts[i], hs[i], hs[i + 1]
            N, K = W.shape
            need_gx = i > 0 or ctx.needs_input_grad[0]
            fuse_prev = i > 0                       # fold layer i-1's activation backward / bias grad into this dgrad
            prev_small = fuse_prev and kinds[i - 1] == "tc"
            gx = torch.empty((M, K), dtype=torch.float32, device=dev) if need_gx else None
            gx_small = empty_aux(M, K, dev) if (prev_small and gx is not None) else None
            gb_prev = None
            if kinds[i] == "head":
                if dl[i] is not None and not g_is_dz:   # a width-1 dropout layer: its mask in the explicit pass
                    gb = bias_buf(i)
                    g, _ = _grad_operand(g, y, act, False, colsum=gb, drop=dl[i])
                    grads[2 * i + 1] = gb
                    g_is_dz = True
                gw = _grad_buffer(W, zero=False)
                gb = None if g_is_dz else bias_buf(i)          # g already dZ_i: activation backward and db_i are done
                gb_prev = bias_buf(i - 1) if fuse_prev else None
                fp32_small = gx_small if (gx_small is not None and gx_small.dtype == torch.float32) else None
                pdrop = dl[i - 1] if fuse_prev else None
                _lib.call("b2_head_bwd_ex", _ptr(h), _ptr(W), None if g_is_dz else _ptr(y), _ptr(g), M, K,
                          B2_ACT_NONE if g_is_dz else act, _ptr(gx), _ptr(gw), _ptr(gb),
                          acts[i - 1] if fuse_prev else B2_ACT_NONE, _ptr(fp32_small), _ptr(gb_prev),
                          1 if (_is_zeroed(gw) and (gb is None or _is_zeroed(gb))
                                and (gb_prev is None or _is_zeroed(gb_prev))) else 0,
                          *((_ptr(pdrop[0]),) + pdrop[1:] if pdrop is not None else (_ptr(None), 0, 0, 0.0)),
                          _stream())
                if gx_small is not None and fp32_small is None:     # bf16 mode: the head kernel emits fp32 only
                    gx_small = make_aux(gx)
                grads[2 * i] = gw
                if not g_is_dz:
                    grads[2 * i + 1] = gb
                if fuse_prev:
                    grads[2 * (i - 1) + 1] = gb_prev
                g, g_small, g_is_dz = gx, gx_small, fuse_prev
                continue
            tc = kinds[i] == "tc"       # else an fp32 SIMT layer inside a chain (odd shapes)
            if not g_is_dz:     # top of the chain (or below a non-fusing layer): one explicit pass over dY
                gb = bias_buf(i)
                gz, gz_small = _grad_operand(g, y, act, tc, colsum=gb, drop=dl[i])
                grads[2 * i + 1] = gb
            else:
                gz, gz_small = g, g_small
            ready = None
            if tc:
                if fork is None and W.requires_grad and _FORK["on"] and gz.is_cuda:
                    fork = _WgradFork(dev)
                if fork is not None and W.requires_grad:
                    ready = fork.ready()
                if gx is not None:
                    prev_act = acts[i - 1] if fuse_prev else B2_ACT_NONE
                    gb_prev = bias_buf(i - 1) if fuse_prev else None
                    _linear_dgrad(True, gz, gz_small, W, gx,
                                  ybwd=hs[i] if (fuse_prev and prev_act != B2_ACT_NONE) else None, act_bwd=prev_act,
                                  out_small=gx_small, colsum=gb_prev,
                                  drop=dl[i - 1] if fuse_prev else None)                          # dX (= dZ_{i-1})
                if fuse_prev:
                    grads[2 * (i - 1) + 1] = gb_prev
            elif gx is not None:
                _linear_dgrad(False, gz, None, W, gx)
            if W.requires_grad:
                gw = _grad_buffer(W, zero=False)
                _linear_wgrad(tc, gz, gz_small, h, smalls[i], gw, fork, ready)
                grads[2 * i] = gw
            # below a SIMT layer, layer i-1 takes the explicit pass (its own db)
            g, g_small, g_is_dz = (gx, gx_small, fuse_prev) if tc else (gx, None, False)
        if fork is not None:
            fork.join()
        return (g if ctx.needs_input_grad[0] else None, None, None) + tuple(grads)


def _cross_step_fwd(a, a_aux, W, w_aux, bias, x0, add, tc):
    """The CrossNetV2 step out = add + x0 * lin, lin = a W^T + bias: returns (out, lin).  On the tensor cores the
    GEMM epilogue applies `add + mul * (acc + bias)` and keeps lin for the backward — no elementwise pass."""
    out, lin = torch.empty_like(add), torch.empty_like(add)
    if tc:
        _linear_fwd(True, a, a_aux, W, out, w_aux, bias=bias, mul=x0, add=add, out_pre=lin)
    else:
        _linear_fwd(False, a, None, W, lin, bias=bias)
        torch.addcmul(add, x0, lin, out=out)
    return out, lin


def _cross_step_bwd(g, x0, a, a_aux, W, w_aux, bias, gw, tc, add_g):
    """Backward of _cross_step_fwd but for dx_0 = g * lin, which the caller takes: dlin = g * x_0 (one pass: value,
    auxiliary operand, bias gradient), d_a = dlin W (+ g in the GEMM's epilogue when add_g: `a` was also `add`),
    dW = dlin^T a into gw (None: not wanted).  Returns (d_a, the bias gradient or None)."""
    gb = _grad_buffer(bias, zero=False) if (bias is not None and bias.requires_grad) else None
    dlin, dlin_aux = _grad_operand(g, x0, B2_PREP_MUL, tc, colsum=gb)
    d_a = torch.empty_like(a)
    _linear_dgrad(tc, dlin, dlin_aux, W, d_a, w_aux, add=g if add_g else None)
    if gw is not None:
        _linear_wgrad(tc, dlin, dlin_aux, a, a_aux, gw)
    return d_a, gb


class _CrossV2Layer(torch.autograd.Function):
    """One CrossNetV2 layer, x_next = x_i + x_0 * (x_i W^T + b) (cross_net.py:126-129): the GEMM epilogue
    applies `add + mul * (acc + bias)` and keeps lin = acc + bias for the backward — no elementwise pass.
    Backward: dlin = g * x_0 (one pass: value, 3xTF32 small part, bias gradient), dW = dlin^T x_i,
    dx_i = g + dlin W (epilogue add), dx_0 = g * lin."""

    @staticmethod
    def forward(ctx, x0, xi, weight, bias):
        x0, xi = _f32c(x0), _f32c(xi)
        ctx.tc = (_tc_layer_ok(weight) and weight.shape[0] == weight.shape[1] == xi.shape[1]
                  and xi.data_ptr() % 16 == 0 and x0.data_ptr() % 16 == 0)
        ctx.xi_small = make_aux(xi) if ctx.tc else None
        out, lin = _cross_step_fwd(xi, ctx.xi_small, weight, None, bias, x0, xi, ctx.tc)
        ctx.save_for_backward(x0, xi, lin, weight)
        ctx.bias = bias
        return out

    @staticmethod
    def backward(ctx, g):
        x0, xi, lin, weight = ctx.saved_tensors
        g = _f32c(g)
        gw = _grad_buffer(weight, zero=False) if weight.requires_grad else None
        gxi, gb = _cross_step_bwd(g, x0, xi, ctx.xi_small, weight, None, ctx.bias, gw, ctx.tc, add_g=True)
        gx0 = g * lin if ctx.needs_input_grad[0] else None
        return gx0, gxi, gw, gb


def cross_v2_layer(x0, xi, weight, bias):
    _require_cuda(x0, xi, weight, bias)
    return _CrossV2Layer.apply(x0, xi, weight, bias)


def crossnet_mix_bound(low_rank, num_experts):
    """None when the CrossNetMix kernels cover (low_rank, num_experts), else the bound it breaks."""
    if not 1 <= low_rank <= _lib.B2_CROSSMIX_MAX_RANK:
        return "low_rank must lie in [1, %d], got %d" % (_lib.B2_CROSSMIX_MAX_RANK, low_rank)
    if num_experts < 1 or num_experts * low_rank > _lib.B2_CROSSMIX_MAX_COLS:
        return "num_experts * low_rank must lie in [1, %d], got %d" % (_lib.B2_CROSSMIX_MAX_COLS,
                                                                     num_experts * low_rank)
    return None


def _aux_args(aux):
    """(pointer, dtype code, row pitch) of an auxiliary operand written by a row kernel (see empty_aux)."""
    if aux is None:
        return _ptr(None), B2_F32, 0
    return _ptr(aux), (B2_BF16 if aux.dtype == torch.bfloat16 else B2_F32), aux.stride(0)


class _CrossMixLayer(torch.autograd.Function):
    """One CrossNetMix layer (cross_net.py:168-198) as two GEMMs around a per-row expert kernel
    (include/fuxictr_b200.h "CrossNetMix"): P = x_l W1^T (the E rank-r projections and the E gate logits in
    one GEMM), A2 = [p_e tanh(tanh(h_e) C_e^T)] (b2_crossmix_fwd), x_next = x_l + x_0 * (A2 W2^T + b) (the
    CrossNetV2 epilogue, lin kept).  W1, W2 are packed from U, V and the gating weights each forward.
    Backward: dlin = g * x_0 (+ bias gradient), dA2 = dlin W2, dW2 = dlin^T A2, the row kernel back to
    dA1 = dP (+ dC), dx_l = g + dA1 W1, dW1 = dA1^T x_l, and one unpack of dW1, dW2 into U, V, gating."""

    @staticmethod
    def forward(ctx, x0, xl, U, V, C, G, bias):
        x0, xl = _f32c(x0), _f32c(xl)
        U, V, C, G = _f32c(U), _f32c(V), _f32c(C), _f32c(G)
        B, d = xl.shape
        E, _, r = U.shape
        n1, k2 = (E * r + E + 3) // 4 * 4, (E * r + 3) // 4 * 4
        dev = xl.device
        W1 = torch.empty((n1, d), dtype=torch.float32, device=dev)
        W2 = torch.empty((d, k2), dtype=torch.float32, device=dev)
        _lib.call("b2_crossmix_pack", _ptr(U), _ptr(V), _ptr(G), d, r, E, _ptr(W1), _ptr(W2), _stream())
        tc = _tc_layer_ok(W1) and _tc_layer_ok(W2) and xl.data_ptr() % 16 == 0 and x0.data_ptr() % 16 == 0
        P = torch.empty((B, n1), dtype=torch.float32, device=dev)
        A2 = torch.empty((B, k2), dtype=torch.float32, device=dev)
        xl_aux = a2_aux = w1_aux = w2_aux = None
        if tc:
            xl_aux, w1_aux, w2_aux = make_aux(xl), make_aux(W1), make_aux(W2)
            a2_aux = empty_aux(B, k2, dev)
        _linear_fwd(tc, xl, xl_aux, W1, P, w1_aux)
        _lib.call("b2_crossmix_fwd", _ptr(P), _ptr(C), B, r, E, _ptr(A2), *_aux_args(a2_aux), _stream())
        out, lin = _cross_step_fwd(A2, a2_aux, W2, w2_aux, bias.view(-1), x0, xl, tc)
        ctx.save_for_backward(x0, xl, lin, P, A2, W1, W2, C)
        ctx.tc, ctx.aux, ctx.r, ctx.bias = tc, (xl_aux, a2_aux, w1_aux, w2_aux), r, bias
        return out

    @staticmethod
    def backward(ctx, g):
        x0, xl, lin, P, A2, W1, W2, C = ctx.saved_tensors
        g = _f32c(g)
        xl_aux, a2_aux, w1_aux, w2_aux = ctx.aux
        tc, r, bias = ctx.tc, ctx.r, ctx.bias
        B, d = xl.shape
        E = C.shape[0]
        n1, k2 = W1.shape[0], W2.shape[1]
        dev = xl.device
        dW2 = torch.empty((d, k2), dtype=torch.float32, device=dev)
        dA1 = torch.empty((B, n1), dtype=torch.float32, device=dev)
        dW1 = torch.empty((n1, d), dtype=torch.float32, device=dev)
        gxl = torch.empty_like(xl)
        gC = torch.zeros_like(C)
        da1_aux = empty_aux(B, n1, dev) if tc else None
        dA2, gb = _cross_step_bwd(g, x0, A2, a2_aux, W2, w2_aux, bias, dW2, tc, add_g=False)
        _lib.call("b2_crossmix_bwd", _ptr(P), _ptr(C), _ptr(dA2), B, r, E, _ptr(dA1), *_aux_args(da1_aux),
                  _ptr(gC), _stream())
        _linear_dgrad(tc, dA1, da1_aux, W1, gxl, w1_aux, add=g)                                    # dx_l = g + dA1 W1
        _linear_wgrad(tc, dA1, da1_aux, xl, xl_aux, dW1)                                           # dW1 = dA1^T x_l
        gU = torch.empty((E, d, r), dtype=torch.float32, device=dev)
        gV = torch.empty_like(gU)
        gG = torch.empty((E, d), dtype=torch.float32, device=dev)
        _lib.call("b2_crossmix_unpack", _ptr(dW1), _ptr(dW2), d, r, E, _ptr(gU), _ptr(gV), _ptr(gG), _stream())
        gx0 = g * lin if ctx.needs_input_grad[0] else None
        return gx0, gxl, gU, gV, gC, gG, gb


def crossnet_mix_layer(x0, xl, U, V, C, gating_weights, bias):
    """x_next of one CrossNetMix layer: U, V (E, d, r), C (E, r, r) and bias (d, 1) are the layer's
    U_list[i], V_list[i], C_list[i], bias[i]; gating_weights the (E, d) rows of every gating[e].weight
    (a tensor, or the E (1, d) weights, which are concatenated)."""
    if isinstance(gating_weights, (list, tuple)):
        gating_weights = torch.cat([w.reshape(1, -1) for w in gating_weights], dim=0)
    _require_cuda(x0, xl, U, V, C, gating_weights, bias)
    E, d, r = U.shape
    if xl.dim() != 2 or xl.shape[1] != d or tuple(V.shape) != (E, d, r) or tuple(C.shape) != (E, r, r) \
            or tuple(gating_weights.shape) != (E, d) or bias.numel() != d:
        raise ValueError("crossnet_mix_layer: shapes x%s U%s V%s C%s gating%s bias%s do not match"
                         % tuple(tuple(t.shape) for t in (xl, U, V, C, gating_weights, bias)))
    bound = crossnet_mix_bound(r, E)
    if bound is not None:
        raise NotImplementedError("CrossNetMix kernels: " + bound)
    return _CrossMixLayer.apply(x0, xl, U, V, C, gating_weights, bias)


class _GatedCrossLayer(torch.autograd.Function):
    """One GDCN gated cross layer, x_next = x_0 * (x_i W^T + b) * sigmoid(x_i Wg^T) + x_i (GDCN.py,
    GateCorssLayer.forward), as one GEMM and one row kernel (include/fuxictr_b200.h "GDCN"): Wp = [W; Wg]
    (b2_gdcn_pack), P = x_i Wp^T, x_next from P (b2_gdcn_fwd, which also writes x_next's auxiliary operand for the
    next layer's GEMM).  Backward: dP, dx_0 and the bias gradient from P (b2_gdcn_bwd), dx_i = g + dP Wp (one
    dgrad, K = 2d, epilogue add), dWp = dP^T x_i (one wgrad) and one b2_gdcn_unpack into the gradients of W, Wg."""

    @staticmethod
    def forward(ctx, x0, xi, w, wg, b):
        ctx.w, ctx.wg, ctx.b = w, wg, b             # the parameters: their gradients may live in an arena
        x0, xi, w, wg, b = _f32c(x0), _f32c(xi), _f32c(w), _f32c(wg), _f32c(b)
        B, d = xi.shape
        dev = xi.device
        Wp = torch.empty((2 * d, d), dtype=torch.float32, device=dev)
        _lib.call("b2_gdcn_pack", _ptr(w), _ptr(wg), d, _ptr(Wp), _stream())
        tc = _tc_layer_ok(Wp) and xi.data_ptr() % 16 == 0 and x0.data_ptr() % 16 == 0
        xi_aux = make_aux(xi) if tc else None
        wp_aux = make_aux(Wp) if tc else None
        P = torch.empty((B, 2 * d), dtype=torch.float32, device=dev)
        _linear_fwd(tc, xi, xi_aux, Wp, P, wp_aux)
        out = torch.empty_like(xi)
        out_aux = empty_aux(B, d, dev) if tc else None
        _lib.call("b2_gdcn_fwd", _ptr(P), _ptr(b), _ptr(x0), _ptr(xi), B, d, _ptr(out), *_aux_args(out_aux),
                  _stream())
        if out_aux is not None:         # the next layer's (or the MLP's) make_aux finds it
            out._b2_aux = (_MATMUL["mode"], out_aux, out._version)
        ctx.save_for_backward(x0, xi, P, Wp, b)
        ctx.tc, ctx.aux = tc, (xi_aux, wp_aux)
        return out

    @staticmethod
    def backward(ctx, g):
        x0, xi, P, Wp, b = ctx.saved_tensors
        g = _f32c(g)
        xi_aux, wp_aux = ctx.aux
        tc = ctx.tc
        B, d = xi.shape
        dev = xi.device
        _, _, w_grad, wg_grad, b_grad = ctx.needs_input_grad
        dP = torch.empty((B, 2 * d), dtype=torch.float32, device=dev)
        dp_aux = empty_aux(B, 2 * d, dev) if tc else None
        gx0 = torch.empty_like(x0)
        gb = _grad_buffer(ctx.b, zero=True) if b_grad else torch.zeros_like(b)
        _lib.call("b2_gdcn_bwd", _ptr(P), _ptr(b), _ptr(x0), _ptr(g), B, d, _ptr(dP), *_aux_args(dp_aux), _ptr(gx0),
                  _ptr(gb), _stream())
        gxi = torch.empty_like(xi)
        _linear_dgrad(tc, dP, dp_aux, Wp, gxi, wp_aux, add=g)                               # dx_i = g + dP Wp
        gw = gwg = None
        if w_grad or wg_grad:
            dWp = torch.empty_like(Wp)
            _linear_wgrad(tc, dP, dp_aux, xi, xi_aux, dWp)                                 # dWp = dP^T x_i
            gw = _grad_buffer(ctx.w, zero=False) if w_grad else torch.empty_like(ctx.w)
            gwg = _grad_buffer(ctx.wg, zero=False) if wg_grad else torch.empty_like(ctx.wg)
            _lib.call("b2_gdcn_unpack", _ptr(dWp), d, _ptr(gw), _ptr(gwg), _stream())
        return (gx0 if ctx.needs_input_grad[0] else None, gxi, gw if w_grad else None, gwg if wg_grad else None,
                gb if b_grad else None)


def gated_cross_layer(x0, xi, w, wg, b):
    """x_next of one GDCN gated cross layer: w, wg (d, d) are the layer's w[i].weight and wg[i].weight, b (d,) its
    b[i]; x0 and xi (B, d)."""
    _require_cuda(x0, xi, w, wg, b)
    if xi.dim() != 2 or tuple(x0.shape) != tuple(xi.shape):
        raise ValueError("gated_cross_layer: x0%s and xi%s must be the same (B, d)" % (tuple(x0.shape), tuple(xi.shape)))
    d = xi.shape[1]
    if tuple(w.shape) != (d, d) or tuple(wg.shape) != (d, d) or tuple(b.shape) != (d,):
        raise ValueError("gated_cross_layer: shapes x%s w%s wg%s b%s do not match"
                         % tuple(tuple(t.shape) for t in (xi, w, wg, b)))
    return _GatedCrossLayer.apply(x0, xi, w, wg, b)


# --------------------------------------------------------------------------------------
# MaskNet (include/fuxictr_b200.h "MaskNet")
# --------------------------------------------------------------------------------------
def masknet_width_bound(n, what="width"):
    """None when the MaskNet row kernels cover a row of n values, else the bound it breaks."""
    if not 1 <= n <= _lib.B2_MASKNET_MAX_WIDTH:
        return "%s must lie in [1, %d], got %d" % (what, _lib.B2_MASKNET_MAX_WIDTH, n)
    return None


class EmbeddingGrad(object):
    """The gradient of MaskNet's flattened embedding V_emb, ONE buffer: every mask block's first mask Linear adds its
    dgrad into it (GEMM accumulate), and so do the embedding LayerNorm's backward and, when V_hidden is V_emb itself,
    the blocks' v_in gradients.  shared_grad() hands it to autograd once all of them have run.  It also keeps V_emb's
    GEMM operand copy, made once per forward for all blocks."""

    def __init__(self):
        self.buf = None
        self._aux = None

    def target(self, like):
        """(buffer, accumulate): the first writer of a backward gets an uninitialised buffer to overwrite."""
        if self.buf is None:
            self.buf = torch.empty_like(like)
            return self.buf, False
        return self.buf, True

    def emb_aux(self, v_emb):
        key = (_MATMUL["mode"], _MATMUL["x3_inline"], v_emb.data_ptr(), v_emb._version, tuple(v_emb.shape))
        if self._aux is None or self._aux[0] != key:
            self._aux = (key, make_aux(v_emb))
        return self._aux[1]


class _SharedGrad(torch.autograd.Function):
    """x -> x (a view), whose backward returns the EmbeddingGrad buffer the consumers of the view added into (they
    return no gradient for it themselves).  Autograd runs this backward after every consumer's."""

    @staticmethod
    def forward(ctx, x, sink):
        ctx.set_materialize_grads(False)
        ctx.sink = sink
        sink.buf = None
        return x.view_as(x)

    @staticmethod
    def backward(ctx, g):
        if g is not None:
            raise RuntimeError("shared_grad: the view's consumers must add into the EmbeddingGrad buffer")
        buf, ctx.sink.buf = ctx.sink.buf, None
        return buf, None


def shared_grad(v_emb):
    """(V_emb view, EmbeddingGrad) for field_layernorm and mask_blocks, which add V_emb's gradient into one buffer."""
    _require_cuda(v_emb)
    sink = EmbeddingGrad()
    return _SharedGrad.apply(_f32c(v_emb), sink), sink


def field_param_layout(weights, biases):
    """(gamma_0, beta_0, pstride) when the F LayerNorms' weights and biases lie at one stride (weight f at
    &weight_0 + f pstride, bias f at &bias_0 + f pstride, as pack_field_params and the fused optimizer's arena place
    them), else None."""
    F = len(weights)
    w0, b0 = weights[0], biases[0]
    if any(not t.is_contiguous() or t.dtype != torch.float32 for t in list(weights) + list(biases)):
        return None
    if F == 1:
        return w0, b0, 0
    step = weights[1].data_ptr() - w0.data_ptr()
    if step <= 0 or step % 4:
        return None
    for f in range(F):
        if weights[f].data_ptr() != w0.data_ptr() + f * step or biases[f].data_ptr() != b0.data_ptr() + f * step:
            return None
    if step // 4 < w0.numel():
        return None
    return w0, b0, step // 4


def pack_field_params(norms):
    """Re-home the weights and biases of the LayerNorms `norms` (one per field) into one buffer,
    [weight_0 | bias_0 | weight_1 | ...] with every slice 16-byte aligned, the layout the fused optimizer's arena gives
    them: the embedding LayerNorm then reads all F of them at one stride.  The Parameter objects stay (only their .data
    moves), so optimizers and state_dict keys are unchanged."""
    params = [p for m in norms for p in (m.weight, m.bias)]
    D = params[0].numel()
    pitch = (D + 3) // 4 * 4
    buf = torch.zeros(len(params) * pitch, dtype=torch.float32, device=params[0].device)
    with torch.no_grad():
        for i, p in enumerate(params):
            dst = buf[i * pitch:i * pitch + D].view(p.shape)
            dst.copy_(p.data)
            p.data = dst


def _strided_grads(params, pstride):
    """Zeroed gradient buffers of params (the weights then the biases of F LayerNorms at one stride) that lie at
    that same stride: the fused optimizer's arena views when they do, else views of one fresh buffer."""
    F = len(params) // 2
    grads = [_grad_buffer(p, zero=True) for p in params]
    layout = field_param_layout(grads[:F], grads[F:])
    if layout is not None and layout[2] == pstride and \
            grads[F].data_ptr() - grads[0].data_ptr() == params[F].data_ptr() - params[0].data_ptr():
        return grads
    base = min(p.data_ptr() for p in params)
    span = (max(p.data_ptr() for p in params) - base) // 4 + params[0].numel()
    buf = torch.zeros(span, dtype=torch.float32, device=params[0].device)
    out = []
    for p in params:
        o = (p.data_ptr() - base) // 4
        out.append(buf[o:o + p.numel()].view(p.shape))
    return out


class _FieldLayerNorm(torch.autograd.Function):
    """MaskNet's embedding LayerNorm, V_hidden = cat_f LayerNorm_f(V_emb[:, f]) (MaskNet.py, MaskNet.forward), one
    launch each way for all F fields (b2_field_ln_fwd / _bwd).  The backward adds the input gradient into the
    EmbeddingGrad buffer and the weight and bias gradients into buffers at the parameters' stride."""

    @staticmethod
    def forward(ctx, x, sink, F, D, eps, *params):
        gamma, beta, pstride = field_param_layout(params[:F], params[F:])
        B = x.shape[0]
        out = torch.empty_like(x)
        ctx.sink, ctx.F, ctx.D, ctx.pstride, ctx.params = sink, F, D, pstride, params
        if B == 0:          # nothing to normalise: no launch (an empty tensor has no device address)
            ctx.save_for_backward(x, None, None)
            return out
        mean = torch.empty((B, F), dtype=torch.float32, device=x.device)
        rstd = torch.empty_like(mean)
        _lib.call("b2_field_ln_fwd", _ptr(x), B, F, D, _ptr(gamma), _ptr(beta), pstride, eps, _ptr(out), _ptr(mean),
                  _ptr(rstd), _stream())
        ctx.save_for_backward(x, mean, rstd)
        return out

    @staticmethod
    def backward(ctx, g):
        x, mean, rstd = ctx.saved_tensors
        F, D, params = ctx.F, ctx.D, ctx.params
        grads = _strided_grads(params, ctx.pstride)
        dx, acc = ctx.sink.target(x)
        if x.shape[0] == 0:
            return (None, None, None, None, None) + tuple(grads)
        _lib.call("b2_field_ln_bwd", _ptr(x), _ptr(mean), _ptr(rstd), _ptr(_f32c(g)), x.shape[0], F, D,
                  _ptr(params[0]), ctx.pstride, _ptr(dx), 1 if acc else 0, _ptr(grads[0]), _ptr(grads[F]), _stream())
        return (None, None, None, None, None) + tuple(grads)


def field_layernorm(x, sink, weights, biases, eps=1e-5):
    """cat_f LayerNorm_f(x[:, f D:(f + 1) D]) of a shared_grad view x (B, F D): the F LayerNorms' weights and biases
    (D) must lie at one stride (field_param_layout; pack_field_params places them so)."""
    F = len(weights)
    _require_cuda(x, *weights)
    if F < 1 or len(biases) != F:
        raise ValueError("field_layernorm: one weight and one bias per field")
    D = weights[0].numel()
    bound = masknet_width_bound(D, "embedding_dim")
    if bound:
        raise ValueError("field_layernorm: " + bound)
    if x.dim() != 2 or x.shape[1] != F * D:
        raise ValueError("field_layernorm: x%s is not (B, %d * %d)" % (tuple(x.shape), F, D))
    if field_param_layout(weights, biases) is None:
        raise ValueError("field_layernorm: the LayerNorms' weights and biases do not lie at one stride; "
                         "re-home them with pack_field_params")
    return _FieldLayerNorm.apply(x, sink, F, D, float(eps), *weights, *biases)


_MASK_PARAMS = 7        # per block: W1, b1, W2, b2, W3, gamma, beta (gamma, beta None without LayerNorm)


class _MaskBlocks(torch.autograd.Function):
    """nb MaskBlocks on one (V_emb, v_in) (MaskNet.py, MaskBlock.forward), their outputs side by side in one
    (B, nb n) tensor: ParallelMaskNet's concatenation without a copy (nb = 1: one block of SerialMaskNet).  Block k:
      h = ReLU(V_emb W1^T + b1)                    GEMM, bias + ReLU epilogue
      u = V_mask * v_in,  V_mask = h W2^T + b2     GEMM, bias + mul epilogue keeping V_mask (out_pre)
      z = u W3^T                                   GEMM
      out[:, k n:(k + 1) n] = drop(act(LN(z)))     b2_mask_row_fwd (+ the operand copy a GEMM consumer wants)
    Backward of block k: dz (b2_mask_row_bwd, with the LayerNorm weight and bias gradients), dV_mask = v_in * (dz W3)
    with du = dz W3 kept (one dgrad, mul epilogue, out_pre, colsum = the b2 gradient), dW3, dv_in += du * V_mask
    (b2_mask_mul), dh = ReLU'(h) * (dV_mask W2) (one dgrad, colsum = the b1 gradient), dW2, and V_emb's gradient added
    into the EmbeddingGrad buffer (dgrad, accumulate), dW1.  v_in None: v_in is V_emb, its gradient goes to the
    buffer too.  Where the tensor cores cannot take a Linear it runs on the SIMT GEMM, and the product the mul
    epilogue would form takes one b2_mask_mul (its sum one b2_prep_operand)."""

    @staticmethod
    def forward(ctx, v_emb, v_in, sink, cfg, *params):
        act, eps, drops, want_aux = cfg
        nb = len(params) // _MASK_PARAMS
        x = v_in if v_in is not None else v_emb
        B = v_emb.shape[0]
        dev = v_emb.device
        n = params[4].shape[0]
        out = torch.empty((B, nb * n), dtype=torch.float32, device=dev)
        ctx.sink, ctx.cfg, ctx.params, ctx.nb = sink, cfg, params, nb
        if B == 0:          # no rows: no launch (an empty tensor has no device address)
            ctx.save_for_backward(v_emb, v_in)
            return out
        out_aux = empty_aux(B, nb * n, dev) if want_aux else None
        emb_aligned = v_emb.data_ptr() % 16 == 0 and x.data_ptr() % 16 == 0
        saved, meta = [], []
        for k in range(nb):
            W1, b1, W2, b2, W3, gamma, beta = params[k * _MASK_PARAMS:(k + 1) * _MASK_PARAMS]
            r, hd = W1.shape[0], W2.shape[0]
            tc = [_tc_layer_ok(W) and emb_aligned for W in (W1, W2, W3)]
            emb_aux = sink.emb_aux(v_emb) if tc[0] else None
            h = torch.empty((B, r), dtype=torch.float32, device=dev)
            h_aux = empty_aux(B, r, dev) if (tc[1] and tc[0]) else None
            _linear_fwd(tc[0], v_emb, emb_aux, W1, h, bias=b1, act=B2_ACT_RELU,
                        **({"out_small": h_aux} if tc[0] else {}))
            if tc[1] and h_aux is None:
                h_aux = make_aux(h)
            vmask = torch.empty((B, hd), dtype=torch.float32, device=dev)
            u = torch.empty_like(vmask)
            u_aux = empty_aux(B, hd, dev) if (tc[2] and tc[1]) else None
            if tc[1]:
                _linear_fwd(True, h, h_aux, W2, u, bias=b2, mul=x, out_pre=vmask, out_small=u_aux)
            else:
                _linear_fwd(False, h, None, W2, vmask, bias=b2)
                _lib.call("b2_mask_mul", _ptr(vmask), _ptr(x), B * hd, _ptr(u), 0, _stream())
            if tc[2] and u_aux is None:
                u_aux = make_aux(u)
            z = torch.empty((B, n), dtype=torch.float32, device=dev)
            _linear_fwd(tc[2], u, u_aux, W3, z)
            ln = gamma is not None
            mean = torch.empty(B, dtype=torch.float32, device=dev) if ln else None
            rstd = torch.empty(B, dtype=torch.float32, device=dev) if ln else None
            dl = drops[k] if drops is not None else None
            seg_aux = out_aux[:, k * n:] if out_aux is not None else None
            _lib.call("b2_mask_row_fwd", _ptr(z), B, n, _ptr(gamma), _ptr(beta), eps, act,
                      *_drop_args(dl), ctypes.c_void_p(out.data_ptr() + 4 * k * n), nb * n,
                      *_aux_args(seg_aux), _ptr(mean), _ptr(rstd), _stream())
            saved += [h, vmask, u, z, mean, rstd]
            meta.append((tc, emb_aux, h_aux, u_aux, dl))
        if out_aux is not None:
            out._b2_aux = (_MATMUL["mode"], out_aux, out._version)
        ctx.save_for_backward(v_emb, v_in, *saved)
        ctx.meta = meta
        return out

    @staticmethod
    def backward(ctx, g):
        v_emb, v_in = ctx.saved_tensors[:2]
        saved = ctx.saved_tensors[2:]
        act = ctx.cfg[0]
        nb, params, sink = ctx.nb, ctx.params, ctx.sink
        x = v_in if v_in is not None else v_emb
        g = _f32c(g)
        B = v_emb.shape[0]
        dev = v_emb.device
        grads = [None] * len(params)
        gx = None
        if B == 0:          # every gradient is zero; V_emb's buffer is left to the other writers
            grads = [_grad_buffer(p, zero=True) if p is not None else None for p in params]
            return (None, torch.zeros_like(v_in) if v_in is not None else None, None, None) + tuple(grads)
        for k in range(nb):
            W1, b1, W2, b2, W3, gamma, beta = params[k * _MASK_PARAMS:(k + 1) * _MASK_PARAMS]
            h, vmask, u, z, mean, rstd = saved[6 * k:6 * k + 6]
            tc, emb_aux, h_aux, u_aux, dl = ctx.meta[k]
            r, hd, n = W1.shape[0], W2.shape[0], W3.shape[0]
            base = k * _MASK_PARAMS
            # the block's tail: dz (+ its operand copy for W3's dgrad and wgrad) and the LayerNorm's gradients
            dz = torch.empty((B, n), dtype=torch.float32, device=dev)
            dz_aux = empty_aux(B, n, dev) if tc[2] else None
            dgamma = dbeta = None
            if gamma is not None:
                dgamma, dbeta = _grad_buffer(gamma, zero=True), _grad_buffer(beta, zero=True)
                grads[base + 5], grads[base + 6] = dgamma, dbeta
            _lib.call("b2_mask_row_bwd", _ptr(z), _ptr(mean), _ptr(rstd), _ptr(gamma), _ptr(beta), act,
                      *_drop_args(dl), ctypes.c_void_p(g.data_ptr() + 4 * k * n), g.stride(0), B, n, _ptr(dz),
                      *_aux_args(dz_aux), _ptr(dgamma), _ptr(dbeta), _stream())
            if tc[2] and dz_aux is None:
                dz_aux = make_aux(dz)
            # hidden Linear: du = dz W3, dV_mask = v_in * du (+ b2's gradient), dW3
            gb2 = _grad_buffer(b2, zero=False)
            du = torch.empty((B, hd), dtype=torch.float32, device=dev)
            dvm = torch.empty_like(du)
            dvm_aux = empty_aux(B, hd, dev) if (tc[1] and tc[2]) else None
            if tc[2]:
                _linear_dgrad(True, dz, dz_aux, W3, dvm, mul=x, out_pre=du, out_small=dvm_aux, colsum=gb2)
                if tc[1] and dvm_aux is None:
                    dvm_aux = make_aux(dvm)
            else:
                _linear_dgrad(False, dz, None, W3, du)
                dvm, dvm_aux = _grad_operand(du, x, B2_PREP_MUL, tc[1], colsum=gb2)
            grads[base + 3] = gb2
            gw3 = _grad_buffer(W3, zero=False)
            _linear_wgrad(tc[2], dz, dz_aux, u, u_aux, gw3)
            grads[base + 4] = gw3
            # v_in's gradient, du * V_mask: summed over the blocks (V_emb's buffer when v_in is V_emb)
            if v_in is not None:
                if gx is None:
                    gx, acc = torch.empty_like(v_in), False
                else:
                    acc = True
            else:
                gx, acc = sink.target(v_emb)
            _lib.call("b2_mask_mul", _ptr(du), _ptr(vmask), B * hd, _ptr(gx), 1 if acc else 0, _stream())
            # mask MLP: dh = ReLU'(h) * (dV_mask W2) (+ b1's gradient), dW2, V_emb's gradient, dW1
            gb1 = _grad_buffer(b1, zero=False)
            dh = torch.empty((B, r), dtype=torch.float32, device=dev)
            if tc[1]:
                dh_aux = empty_aux(B, r, dev) if tc[0] else None
                _linear_dgrad(True, dvm, dvm_aux, W2, dh, ybwd=h, act_bwd=B2_ACT_RELU, out_small=dh_aux, colsum=gb1)
                if tc[0] and dh_aux is None:
                    dh_aux = make_aux(dh)
            else:
                _linear_dgrad(False, dvm, None, W2, dh)
                dh, dh_aux = _grad_operand(dh, h, B2_ACT_RELU, tc[0], colsum=gb1)
            grads[base + 1] = gb1
            gw2 = _grad_buffer(W2, zero=False)
            _linear_wgrad(tc[1], dvm, dvm_aux, h, h_aux, gw2)
            grads[base + 2] = gw2
            gemb, acc = sink.target(v_emb)
            _linear_dgrad(tc[0], dh, dh_aux, W1, gemb, accumulate=acc)
            gw1 = _grad_buffer(W1, zero=False)
            _linear_wgrad(tc[0], dh, dh_aux, v_emb, emb_aux, gw1)
            grads[base] = gw1
        return (None, gx if v_in is not None else None, None, None) + tuple(grads)


def _drop_args(dl):
    """The (drop_rng, drop_layer, drop_thresh, drop_scale) arguments of a (snapshot, layer, thresh, scale) or None."""
    if dl is None:
        return _ptr(None), 0, 0, 0.0
    return _ptr(dl[0]), dl[1], dl[2], dl[3]


def mask_blocks(v_emb, sink, v_in, blocks, act, eps=1e-5, dropout=0.0, snapshot=None, first_layer=0, want_aux=False):
    """The outputs of the MaskBlocks `blocks` on one (V_emb, v_in), side by side in one (B, nb n) tensor.  v_emb and
    sink come from shared_grad; v_in None: the blocks' input is V_emb itself.  A block is (W1, b1, W2, b2, W3,
    gamma, beta) (gamma, beta None: no LayerNorm): its mask_layer.0, mask_layer.2 and hidden_layer Linear weights
    and biases, and its LayerNorm's.  act: B2_ACT_RELU or B2_ACT_SIGMOID.  dropout > 0: block k draws the mask of
    layer first_layer + k of `snapshot` (dropout_snapshot).  want_aux: also write the output's GEMM operand copy for
    a GEMM consumer."""
    _require_cuda(v_emb, v_in)
    if act not in (B2_ACT_RELU, B2_ACT_SIGMOID, B2_ACT_NONE):
        raise NotImplementedError("mask_blocks: activation code %r" % (act,))
    x = v_in if v_in is not None else v_emb
    B, d = v_emb.shape
    params = []
    n = blocks[0][4].shape[0]
    for blk in blocks:
        W1, b1, W2, b2, W3, gamma, beta = blk
        r, hd = W1.shape[0], W2.shape[0]
        if (tuple(W1.shape) != (r, d) or tuple(b1.shape) != (r,) or tuple(W2.shape) != (hd, r)
                or tuple(b2.shape) != (hd,) or tuple(W3.shape) != (n, hd) or x.shape != (B, hd)
                or (gamma is None) != (beta is None)
                or (gamma is not None and (tuple(gamma.shape) != (n,) or tuple(beta.shape) != (n,)))):
            raise ValueError("mask_blocks: shapes V_emb%s v_in%s W1%s W2%s W3%s do not match"
                             % tuple(tuple(t.shape) for t in (v_emb, x, W1, W2, W3)))
        params += [W1, b1, W2, b2, W3, gamma, beta]
    bound = masknet_width_bound(n, "output_dim")
    if bound:
        raise ValueError("mask_blocks: " + bound)
    drops = None
    if dropout > 0:
        consts = dropout_consts(dropout)
        drops = [(snapshot, first_layer + k) + consts for k in range(len(blocks))]
    return _MaskBlocks.apply(v_emb, None if v_in is None else _f32c(v_in), sink, (act, float(eps), drops, want_aux),
                             *params)


# --------------------------------------------------------------------------------------
# AutoInt (include/fuxictr_b200.h "AutoInt")
# --------------------------------------------------------------------------------------
def autoint_bound(fields, attention_dim, heads):
    """None when the AutoInt row kernels cover F fields, attention_dim A and `heads` heads, else the bound it breaks."""
    if not 1 <= fields <= _lib.B2_AUTOINT_MAX_FIELDS:
        return "the number of fields must lie in [1, %d], got %d" % (_lib.B2_AUTOINT_MAX_FIELDS, fields)
    if not 1 <= attention_dim <= _lib.B2_AUTOINT_MAX_DIM:
        return "attention_dim must lie in [1, %d], got %d" % (_lib.B2_AUTOINT_MAX_DIM, attention_dim)
    if heads < 1 or attention_dim % heads:
        return "num_heads=%d does not divide attention_dim=%d" % (heads, attention_dim)
    return None


class _SelfAttentionLayer(torch.autograd.Function):
    """One AutoInt MultiHeadSelfAttention layer (AutoInt.py, MultiHeadSelfAttention.forward) on X (B, F, d_in) as one
    GEMM and one row kernel (include/fuxictr_b200.h "AutoInt"): Wp = [W_q; W_k; W_v (; W_res)] (b2_autoint_pack),
    P = X Wp^T, out = ReLU(LN(attention(P) + residual)) (b2_autoint_fwd, which also writes out's auxiliary operand for
    the next layer's GEMM when asked).  Backward: dP with the residual's and the LayerNorm's gradients
    (b2_autoint_bwd), dX = dP Wp (+ dR for an identity residual, as the dgrad's epilogue add), dWp = dP^T X and one
    b2_autoint_unpack into the gradients of W_q, W_k, W_v (, W_res)."""

    @staticmethod
    def forward(ctx, x, cfg, wq, wk, wv, wres, gamma, beta):
        heads, scale, eps, res_mode, drop, want_aux = cfg
        ctx.params = (wq, wk, wv, wres, gamma, beta)     # their gradients may live in an arena
        B, F, din = x.shape
        A = wq.shape[0]
        dev = x.device
        x2 = _f32c(x).view(B * F, din)
        parts = 4 if wres is not None else 3
        NP = parts * A
        out = torch.empty((B, F, A), dtype=torch.float32, device=dev)
        ctx.cfg, ctx.shape = cfg, (B, F, din, A, NP)
        if B == 0:          # no rows: no launch (an empty tensor has no device address)
            ctx.tc = False
            return out
        Wp = torch.empty((NP, din), dtype=torch.float32, device=dev)
        _lib.call("b2_autoint_pack", _ptr(_f32c(wq)), _ptr(_f32c(wk)), _ptr(_f32c(wv)),
                  _ptr(_f32c(wres) if wres is not None else None), din, A, _ptr(Wp), _stream())
        tc = _tc_layer_ok(Wp) and x2.data_ptr() % 16 == 0
        x_aux = make_aux(x2) if tc else None
        wp_aux = make_aux(Wp) if tc else None
        P = torch.empty((B * F, NP), dtype=torch.float32, device=dev)
        _linear_fwd(tc, x2, x_aux, Wp, P, wp_aux)
        out_aux = empty_aux(B * F, A, dev) if want_aux else None
        smax = torch.empty((B, heads, F), dtype=torch.float32, device=dev)
        ssum = torch.empty_like(smax)
        ln = gamma is not None
        mean = torch.empty(B * F, dtype=torch.float32, device=dev) if ln else None
        rstd = torch.empty_like(mean) if ln else None
        _lib.call("b2_autoint_fwd", _ptr(P), _ptr(x2), B, F, din, A, heads, res_mode, scale, _ptr(gamma), _ptr(beta),
                  eps, *_drop_args(drop), _ptr(out), *_aux_args(out_aux), _ptr(smax), _ptr(ssum), _ptr(mean),
                  _ptr(rstd), _stream())
        if out_aux is not None:         # the next layer's make_aux finds it
            out._b2_aux = (_MATMUL["mode"], out_aux, out._version)
        ctx.save_for_backward(x2, P, Wp, out, smax, ssum, mean, rstd)
        ctx.tc, ctx.aux = tc, (x_aux, wp_aux)
        return out

    @staticmethod
    def backward(ctx, g):
        heads, scale, _, res_mode, drop, _ = ctx.cfg
        B, F, din, A, NP = ctx.shape
        wq, wk, wv, wres, gamma, beta = ctx.params
        need = ctx.needs_input_grad
        ln = gamma is not None
        dgamma = _grad_buffer(gamma, zero=True) if ln and need[6] else (torch.zeros_like(gamma) if ln else None)
        dbeta = _grad_buffer(beta, zero=True) if ln and need[7] else (torch.zeros_like(beta) if ln else None)
        ws = [w for w in (wq, wk, wv, wres) if w is not None]
        if B == 0:
            gws = [_grad_buffer(w, zero=True) for w in ws] + [None] * (4 - len(ws))
            return (torch.zeros((B, F, din), dtype=torch.float32, device=g.device), None) + tuple(gws) + (dgamma, dbeta)
        x2, P, Wp, out, smax, ssum, mean, rstd = ctx.saved_tensors
        x_aux, wp_aux = ctx.aux
        tc = ctx.tc
        dev = x2.device
        g = _f32c(g)
        dP = torch.empty((B * F, NP), dtype=torch.float32, device=dev)
        dp_aux = empty_aux(B * F, NP, dev) if tc else None
        gres = torch.empty((B * F, A), dtype=torch.float32, device=dev) if res_mode == 1 else None
        _lib.call("b2_autoint_bwd", _ptr(P), _ptr(x2), _ptr(out), _ptr(g), _ptr(smax), _ptr(ssum), _ptr(mean),
                  _ptr(rstd), B, F, din, A, heads, res_mode, scale, _ptr(gamma), *_drop_args(drop), _ptr(dP),
                  *_aux_args(dp_aux), _ptr(gres), _ptr(dgamma), _ptr(dbeta), _stream())
        gx = torch.empty((B * F, din), dtype=torch.float32, device=dev)
        _linear_dgrad(tc, dP, dp_aux, Wp, gx, wp_aux, **({"add": gres} if gres is not None else {}))   # dX = dP Wp
        dWp = torch.empty_like(Wp)
        _linear_wgrad(tc, dP, dp_aux, x2, x_aux, dWp)                                                   # dWp = dP^T X
        gws = [_grad_buffer(w, zero=False) if need[2 + k] else torch.empty_like(w)
               for k, w in enumerate((wq, wk, wv, wres)) if w is not None]
        _lib.call("b2_autoint_unpack", _ptr(dWp), din, A, _ptr(gws[0]), _ptr(gws[1]), _ptr(gws[2]),
                  _ptr(gws[3] if wres is not None else None), _stream())
        gws += [None] * (4 - len(gws))
        gws = [gw if need[2 + k] else None for k, gw in enumerate(gws)]
        return (gx.view(B, F, din), None) + tuple(gws) + (dgamma if ln and need[6] else None,
                                                          dbeta if ln and need[7] else None)


def self_attention_layer(x, w_q, w_k, w_v, w_res=None, num_heads=1, use_residual=True, use_scale=False, gamma=None,
                         beta=None, eps=1e-5, dropout=0.0, snapshot=None, layer=0, want_aux=False):
    """out (B, F, A) of one AutoInt MultiHeadSelfAttention layer on x (B, F, d_in): w_q, w_k, w_v (and w_res, when
    use_residual and d_in != A) the (A, d_in) weights of W_q, W_k, W_v (and W_res); gamma, beta (A) the LayerNorm's
    weight and bias (None: no LayerNorm).  dropout > 0: the attention weights take the mask of layer `layer` of
    `snapshot` (dropout_snapshot; None: a snapshot of its own).  want_aux: also write out's GEMM operand copy for a
    following layer's projection GEMM."""
    _require_cuda(x, w_q, w_k, w_v, w_res, gamma, beta)
    if x.dim() != 3:
        raise ValueError("self_attention_layer: x%s is not (B, F, d_in)" % (tuple(x.shape),))
    B, F, din = x.shape
    A = w_q.shape[0]
    bound = autoint_bound(F, A, num_heads)
    if bound is not None:
        raise NotImplementedError("AutoInt kernels: " + bound)
    if any(tuple(w.shape) != (A, din) for w in (w_q, w_k, w_v) + ((w_res,) if w_res is not None else ())):
        raise ValueError("self_attention_layer: x%s and the projection weights %s do not match"
                         % (tuple(x.shape), [tuple(w.shape) for w in (w_q, w_k, w_v, w_res) if w is not None]))
    if (gamma is None) != (beta is None) or (gamma is not None and (gamma.numel() != A or beta.numel() != A)):
        raise ValueError("self_attention_layer: the LayerNorm needs a weight and a bias of %d" % A)
    if use_residual and w_res is None and din != A:
        raise ValueError("self_attention_layer: a residual with input_dim %d != attention_dim %d needs w_res"
                         % (din, A))
    res_mode = (2 if w_res is not None else 1) if use_residual else 0
    if not use_residual:
        w_res = None
    drop = None
    if dropout > 0:
        if snapshot is None:
            snapshot, layer = dropout_snapshot(x.device, 1), 0
        drop = (snapshot, layer) + dropout_consts(dropout)
    scale = float((A // num_heads) ** 0.5) if use_scale else 0.0
    cfg = (num_heads, scale, float(eps), res_mode, drop, want_aux)
    return _SelfAttentionLayer.apply(x, cfg, w_q, w_k, w_v, w_res, gamma, beta)


# --------------------------------------------------------------------------------------
# BST (include/fuxictr_b200.h "BST")
# --------------------------------------------------------------------------------------
BST_POOL = {"mean": _lib.B2_BST_POOL_MEAN, "sum": _lib.B2_BST_POOL_SUM, "target": _lib.B2_BST_POOL_TARGET}


def bst_bound(seq_len, model_dim, num_heads, parts=1, heads_apply=True):
    """None when the BST kernels cover L = seq_len tokens of width model_dim in num_heads heads, built from `parts`
    fields per token; else the bound it breaks.  heads_apply=False: the kernels that see no heads (tokens, pooling)."""
    if not 2 <= seq_len <= _lib.B2_BST_MAX_LEN:
        return "max_len + 1 must lie in [2, %d], got %d" % (_lib.B2_BST_MAX_LEN, seq_len)
    if not 1 <= model_dim <= _lib.B2_BST_MAX_DIM:
        return "model_dim must lie in [1, %d], got %d" % (_lib.B2_BST_MAX_DIM, model_dim)
    if not 1 <= parts <= _lib.B2_BST_MAX_PARTS:
        return "a token takes 1 to %d fields, got %d" % (_lib.B2_BST_MAX_PARTS, parts)
    if not heads_apply:
        return None
    if not 1 <= num_heads <= _lib.B2_BST_MAX_HEADS:
        return "num_heads must lie in [1, %d], got %d" % (_lib.B2_BST_MAX_HEADS, num_heads)
    if model_dim % num_heads:
        return "num_heads=%d does not divide model_dim=%d" % (num_heads, model_dim)
    if model_dim // num_heads > _lib.B2_BST_MAX_HEAD_DIM:
        return "the head width model_dim / num_heads must be at most %d, got %d" % (_lib.B2_BST_MAX_HEAD_DIM,
                                                                                 model_dim // num_heads)
    return None


def _set_aux_hint(out, aux):
    """The next GEMM's make_aux(out) finds the operand copy its producer wrote."""
    if aux is not None:
        out._b2_aux = (_MATMUL["mode"], aux, out._version)


def _arr(ctype, values):
    return (ctype * len(values))(*values)


class _BstTokens(torch.autograd.Function):
    """X (B L, md): per sample the L - 1 history tokens [seq_0[b, t] .. | pos[t]] and the target token
    [tgt_0[b] .. | pos[L - 1]] (b2_bst_tokens_fwd).  Backward: each view's gradient and the position table's batch sum
    in one launch (b2_bst_tokens_bwd)."""

    @staticmethod
    def forward(ctx, cfg, pos, *views):
        want_aux, = cfg
        nf = len(views) // 2
        # a view's samples may lie at any pitch (an arena slice, a sharded front's landed rows); within a sample
        # the tokens must be contiguous
        seqs = [v if (v.dtype == torch.float32 and v.stride(2) == 1 and v.stride(1) == v.shape[2]) else
                v.float().contiguous() for v in views[:nf]]
        tgts = [v if (v.dtype == torch.float32 and v.stride(1) == 1) else v.float().contiguous() for v in views[nf:]]
        B, Lm1, D = seqs[0].shape
        L = Lm1 + 1
        md = D * (nf + (pos is not None))
        dev = seqs[0].device
        out = torch.empty((B * L, md), dtype=torch.float32, device=dev)
        ctx.shape = (B, L, D, nf, pos is not None)
        ctx.pos = pos
        if B == 0:
            return out
        aux = empty_aux(B * L, md, dev) if want_aux else None
        _lib.call("b2_bst_tokens_fwd", _arr(ctypes.c_void_p, [v.data_ptr() for v in seqs]),
                  _arr(ctypes.c_int64, [v.stride(0) for v in seqs]), _arr(ctypes.c_void_p, [v.data_ptr() for v in tgts]),
                  _arr(ctypes.c_int64, [v.stride(0) for v in tgts]), nf, _ptr(_f32c(pos) if pos is not None else None),
                  B, L, D, _ptr(out), *_aux_args(aux), _stream())
        _set_aux_hint(out, aux)
        return out

    @staticmethod
    def backward(ctx, g):
        B, L, D, nf, use_pos = ctx.shape
        dev = g.device
        dseq = [torch.empty((B, L - 1, D), dtype=torch.float32, device=dev) for _ in range(nf)]
        dtgt = [torch.empty((B, D), dtype=torch.float32, device=dev) for _ in range(nf)]
        dpos = None
        if use_pos:
            dpos = _grad_buffer(ctx.pos, zero=True) if ctx.needs_input_grad[1] else torch.zeros_like(ctx.pos)
        if B > 0:
            _lib.call("b2_bst_tokens_bwd", _ptr(_f32c(g)), None, B, L, D, nf, int(use_pos),
                      _arr(ctypes.c_void_p, [t.data_ptr() for t in dseq]), _arr(ctypes.c_void_p, [t.data_ptr() for t in dtgt]),
                      _ptr(dpos), _stream())
        return (None, dpos if use_pos and ctx.needs_input_grad[1] else None) + tuple(dseq) + tuple(dtgt)


def bst_tokens(sequence_embs, target_embs, position_emb=None, want_aux=False):
    """The (B L, model_dim) token matrix of one (target, sequence) pair: sequence_embs nf views (B, L - 1, D),
    target_embs nf views (B, D) (a tuple of fields: their embeddings side by side), position_emb (L, D) or None.
    want_aux: also write the matrix's GEMM operand copy for the in-projection."""
    seqs, tgts = list(sequence_embs), list(target_embs)
    _require_cuda(*(seqs + tgts + [position_emb]))
    if len(seqs) != len(tgts) or not seqs:
        raise ValueError("bst_tokens: %d sequence fields and %d target fields" % (len(seqs), len(tgts)))
    B, Lm1, D = seqs[0].shape
    for v in seqs:
        if v.dim() != 3 or tuple(v.shape) != (B, Lm1, D):
            raise ValueError("bst_tokens: sequence embeddings %s differ" % [tuple(t.shape) for t in seqs])
    for v in tgts:
        if tuple(v.shape) != (B, D):
            raise ValueError("bst_tokens: target embeddings %s are not (%d, %d)" % ([tuple(t.shape) for t in tgts], B, D))
    if position_emb is not None and tuple(position_emb.shape) != (Lm1 + 1, D):
        raise ValueError("bst_tokens: position_emb%s is not (%d, %d)" % (tuple(position_emb.shape), Lm1 + 1, D))
    md = D * (len(seqs) + (position_emb is not None))
    bound = bst_bound(Lm1 + 1, md, 1, len(seqs), heads_apply=False)
    if bound is not None:
        raise NotImplementedError("BST kernels: " + bound)
    return _BstTokens.apply((want_aux,), position_emb, *(seqs + tgts))


class _BstAttention(torch.autograd.Function):
    """ctx (B L, md) of the masked multi-head self-attention on QKV (B L, 3 md) (b2_bst_attn_fwd), the probabilities
    never stored; backward: dQKV in one launch (b2_bst_attn_bwd), which feeds the in-projection's dgrad and wgrad."""

    @staticmethod
    def forward(ctx, qkv, valid, cfg):
        B, L, md, heads, causal, scale, drop, want_aux = cfg
        dev = qkv.device
        out = torch.empty((B * L, md), dtype=torch.float32, device=dev)
        ctx.cfg = cfg
        if B == 0:
            return out
        qkv = _f32c(qkv)
        aux = empty_aux(B * L, md, dev) if want_aux else None
        smax = torch.empty((B, heads, L), dtype=torch.float32, device=dev)
        ssum = torch.empty_like(smax)
        _lib.call("b2_bst_attn_fwd", _ptr(qkv), _ptr(valid), B, L, md, heads, int(causal), scale, *_drop_args(drop),
                  _ptr(out), *_aux_args(aux), _ptr(smax), _ptr(ssum), _stream())
        _set_aux_hint(out, aux)
        ctx.save_for_backward(qkv, valid, out, smax, ssum)
        return out

    @staticmethod
    def backward(ctx, g):
        B, L, md, heads, causal, scale, drop, _ = ctx.cfg
        if B == 0:
            return torch.zeros((0, 3 * md), dtype=torch.float32, device=g.device), None, None
        qkv, valid, out, smax, ssum = ctx.saved_tensors
        dqkv = torch.empty_like(qkv)
        _lib.call("b2_bst_attn_bwd", _ptr(qkv), _ptr(valid), _ptr(out), _ptr(_f32c(g)), _ptr(smax), _ptr(ssum), B, L,
                  md, heads, int(causal), scale, *_drop_args(drop), _ptr(dqkv), *_aux_args(None), _stream())
        return dqkv, None, None


def bst_attention(qkv, valid, batch, seq_len, num_heads, causal=False, dropout=0.0, snapshot=None, layer=0,
                  want_aux=False):
    """torch's nn.MultiheadAttention core on the in-projection's output qkv (B L, 3 md) = [Q | K | V]: per head
    softmax((q sqrt(1 / dh)) k^T + mask) v with BST's mask: key j hidden from query i != j when j is a padded history
    slot (valid (B, L - 1) uint8, 0 = padding) or, causal, j > i.  dropout > 0: the weights take the mask of layer
    `layer` of `snapshot` (dropout_snapshot; None: one of its own).  Returns (B L, md), before out_proj."""
    _require_cuda(qkv, valid)
    B, L = batch, seq_len
    md = qkv.shape[1] // 3 if qkv.dim() == 2 else 0
    if qkv.dim() != 2 or qkv.shape[0] != B * L or qkv.shape[1] != 3 * md:
        raise ValueError("bst_attention: qkv%s is not (%d, 3 model_dim)" % (tuple(qkv.shape), B * L))
    if valid.dtype != torch.uint8 or tuple(valid.shape) != (B, L - 1) or not valid.is_contiguous():
        raise ValueError("bst_attention: valid must be a contiguous (%d, %d) uint8 mask" % (B, L - 1))
    bound = bst_bound(L, md, num_heads)
    if bound is not None:
        raise NotImplementedError("BST kernels: " + bound)
    drop = None
    if dropout > 0:
        if snapshot is None:
            snapshot, layer = dropout_snapshot(qkv.device, 1), 0
        drop = (snapshot, layer) + dropout_consts(dropout)
    scale = float(ctypes.c_float(math.sqrt(1.0 / (md // num_heads))).value)
    return _BstAttention.apply(qkv, valid, (B, L, md, num_heads, bool(causal), scale, drop, want_aux))


class _BstAddNorm(torch.autograd.Function):
    """out = LN(res + dropout(a)) (b2_bst_addnorm_fwd), each stage optional; backward in one launch
    (b2_bst_addnorm_bwd): d(res) is dz itself, da the masked dz."""

    @staticmethod
    def forward(ctx, a, res, cfg, gamma, beta):
        eps, drop, want_aux = cfg
        a = _f32c(a)
        res = _f32c(res) if res is not None else None
        R, n = a.shape
        dev = a.device
        out = torch.empty((R, n), dtype=torch.float32, device=dev)
        ln = gamma is not None
        mean = torch.empty(R, dtype=torch.float32, device=dev) if ln else None
        rstd = torch.empty_like(mean) if ln else None
        ctx.cfg, ctx.ln_params = cfg, (gamma, beta)
        ctx.has_res = res is not None
        if R > 0:
            aux = empty_aux(R, n, dev) if want_aux else None
            _lib.call("b2_bst_addnorm_fwd", _ptr(a), _ptr(res), R, n, _ptr(gamma), _ptr(beta), eps, *_drop_args(drop),
                      _ptr(out), *_aux_args(aux), _ptr(mean), _ptr(rstd), _stream())
            _set_aux_hint(out, aux)
        ctx.save_for_backward(a if ln else None, res if ln else None, mean, rstd)
        return out

    @staticmethod
    def backward(ctx, g):
        eps, drop, _ = ctx.cfg
        gamma, beta = ctx.ln_params
        a, res, mean, rstd = ctx.saved_tensors
        need = ctx.needs_input_grad
        ln = gamma is not None
        R, n = g.shape
        dev = g.device
        dgamma = (_grad_buffer(gamma, zero=True) if need[3] else torch.zeros_like(gamma)) if ln else None
        dbeta = (_grad_buffer(beta, zero=True) if need[4] else torch.zeros_like(beta)) if ln else None
        da = torch.empty((R, n), dtype=torch.float32, device=dev)
        dres = torch.empty_like(da) if (ctx.has_res and drop is not None) else None
        if R > 0:
            _lib.call("b2_bst_addnorm_bwd", _ptr(a), _ptr(res), _ptr(_f32c(g)), None, R, n, _ptr(gamma), _ptr(mean),
                      _ptr(rstd), *_drop_args(drop), _ptr(da), *_aux_args(None), _ptr(dres), _ptr(dgamma),
                      _ptr(dbeta), _stream())
        if ctx.has_res and dres is None:
            dres = da                   # no dropout: the residual's gradient is the same dz
        return (da, dres if ctx.has_res else None, None, dgamma if ln and need[3] else None,
                dbeta if ln and need[4] else None)


def bst_add_norm(a, res=None, gamma=None, beta=None, eps=1e-5, dropout=0.0, snapshot=None, layer=0, want_aux=False):
    """LN(res + dropout(a)) on (rows, n): TransformerBlock's `s = LN1(x + dropout1(attn))` and
    `LN2(s + dropout2(ffn))`; res None: no residual; gamma, beta None: no LayerNorm.  dropout > 0: the mask of layer
    `layer` of `snapshot`.  want_aux: also write the output's GEMM operand copy."""
    _require_cuda(a, res, gamma, beta)
    if a.dim() != 2 or (res is not None and res.shape != a.shape):
        raise ValueError("bst_add_norm: a%s and res%s" % (tuple(a.shape), None if res is None else tuple(res.shape)))
    n = a.shape[1]
    if not 1 <= n <= _lib.B2_BST_MAX_DIM:
        raise NotImplementedError("BST kernels: model_dim must lie in [1, %d], got %d" % (_lib.B2_BST_MAX_DIM, n))
    if (gamma is None) != (beta is None) or (gamma is not None and (gamma.numel() != n or beta.numel() != n)):
        raise ValueError("bst_add_norm: the LayerNorm needs a weight and a bias of %d" % n)
    drop = None
    if dropout > 0:
        if snapshot is None:
            snapshot, layer = dropout_snapshot(a.device, 1), 0
        drop = (snapshot, layer) + dropout_consts(dropout)
    return _BstAddNorm.apply(a, res, (float(eps), drop, want_aux), gamma, beta)


class _BstPool(torch.autograd.Function):
    """(B, md) pooling of the L tokens of x (B L, md) (b2_bst_pool_fwd / _bwd)."""

    @staticmethod
    def forward(ctx, x, valid, cfg):
        B, L, mode = cfg
        md = x.shape[1]
        out = torch.empty((B, md), dtype=torch.float32, device=x.device)
        ctx.cfg = cfg
        ctx.save_for_backward(valid)
        if B > 0:
            _lib.call("b2_bst_pool_fwd", _ptr(_f32c(x)), _ptr(valid), B, L, md, mode, _ptr(out), md, _stream())
        return out

    @staticmethod
    def backward(ctx, g):
        B, L, mode = ctx.cfg
        valid, = ctx.saved_tensors
        md = g.shape[1]
        dx = torch.empty((B * L, md), dtype=torch.float32, device=g.device)
        if B > 0:
            g = _f32c(g)
            _lib.call("b2_bst_pool_bwd", _ptr(g), g.stride(0), _ptr(valid), B, L, md, mode, _ptr(dx), _stream())
        return dx, None, None


def bst_pooling(x, valid, batch, seq_len, pooling="mean"):
    """BST.sequence_pooling of the transformer output x (B L, md): "mean" / "sum" over the real history slots and the
    target (mean divides by their count + 1e-12), "target" the last token, "concat" all L tokens flattened (a view)."""
    _require_cuda(x, valid)
    B, L = batch, seq_len
    if x.dim() != 2 or x.shape[0] != B * L:
        raise ValueError("bst_pooling: x%s is not (%d, model_dim)" % (tuple(x.shape), B * L))
    if pooling == "concat":
        return x.reshape(B, L * x.shape[1])
    if pooling not in BST_POOL:
        raise ValueError("seq_pooling_type={} not supported.".format(pooling))
    if valid.dtype != torch.uint8 or tuple(valid.shape) != (B, L - 1) or not valid.is_contiguous():
        raise ValueError("bst_pooling: valid must be a contiguous (%d, %d) uint8 mask" % (B, L - 1))
    bound = bst_bound(L, x.shape[1], 1, heads_apply=False)
    if bound is not None:
        raise NotImplementedError("BST kernels: " + bound)
    return _BstPool.apply(x, valid, (B, L, BST_POOL[pooling]))


# --------------------------------------------------------------------------------------
# TransAct (include/fuxictr_b200.h "TransAct")
# --------------------------------------------------------------------------------------
_IDS_DTYPE = {torch.float64: _lib.B2_F64, torch.int64: _lib.B2_I64, torch.int32: _lib.B2_I32,
              torch.float32: _lib.B2_F32}


def transact_bound(seq_len, model_dim, num_heads, parts=2, heads_apply=True):
    """None when the TransAct kernels cover L = seq_len tokens of width model_dim in num_heads heads, built from
    `parts` fields per token (sequence and target fields together); else the bound it breaks.  heads_apply=False: the
    kernels that see no heads (tokens, output)."""
    if not 1 <= seq_len <= _lib.B2_TRANSACT_MAX_LEN:
        return "max_len must lie in [1, %d], got %d" % (_lib.B2_TRANSACT_MAX_LEN, seq_len)
    if not 1 <= model_dim <= _lib.B2_TRANSACT_MAX_DIM:
        return "model_dim must lie in [1, %d], got %d" % (_lib.B2_TRANSACT_MAX_DIM, model_dim)
    if not 2 <= parts <= _lib.B2_TRANSACT_MAX_PARTS:
        return "a token takes 2 to %d fields, got %d" % (_lib.B2_TRANSACT_MAX_PARTS, parts)
    if not heads_apply:
        return None
    if not 1 <= num_heads <= _lib.B2_TRANSACT_MAX_HEADS:
        return "num_heads must lie in [1, %d], got %d" % (_lib.B2_TRANSACT_MAX_HEADS, num_heads)
    if model_dim % num_heads:
        return "num_heads=%d does not divide model_dim=%d" % (num_heads, model_dim)
    if model_dim // num_heads > _lib.B2_TRANSACT_MAX_HEAD_DIM:
        return "the head width model_dim / num_heads must be at most %d, got %d" % (_lib.B2_TRANSACT_MAX_HEAD_DIM,
                                                                                 model_dim // num_heads)
    return None


class _TransActTokens(torch.autograd.Function):
    """(X (B L, md), valid (B, L) uint8): token t of sample b is [seq_0[b, t] .. | tgt_0[b] ..], valid is ids != 0 with
    an empty history's last slot set (b2_transact_tokens_fwd, one launch).  Backward: the sequence views' gradients and
    the targets' sums over t in one launch (b2_transact_tokens_bwd)."""

    @staticmethod
    def forward(ctx, cfg, ids, *views):
        ns, want_aux = cfg
        seqs = [v if (v.dtype == torch.float32 and v.stride(2) == 1 and v.stride(1) == v.shape[2]) else
                v.float().contiguous() for v in views[:ns]]
        tgts = [v if (v.dtype == torch.float32 and v.stride(1) == 1) else v.float().contiguous() for v in views[ns:]]
        nt = len(tgts)
        B, L, D = seqs[0].shape
        md = D * (ns + nt)
        dev = seqs[0].device
        out = torch.empty((B * L, md), dtype=torch.float32, device=dev)
        valid = torch.empty((B, L), dtype=torch.uint8, device=dev)
        ctx.shape = (B, L, D, ns, nt)
        ctx.mark_non_differentiable(valid)
        if B == 0:
            return out, valid
        if ids.dtype not in _IDS_DTYPE:
            ids = ids.long()
        if ids.stride(1) != 1:
            ids = ids.contiguous()
        aux = empty_aux(B * L, md, dev) if want_aux else None
        _lib.call("b2_transact_tokens_fwd", _arr(ctypes.c_void_p, [v.data_ptr() for v in seqs]),
                  _arr(ctypes.c_int64, [v.stride(0) for v in seqs]), ns,
                  _arr(ctypes.c_void_p, [v.data_ptr() for v in tgts]), _arr(ctypes.c_int64, [v.stride(0) for v in tgts]),
                  nt, _ptr(ids), _IDS_DTYPE[ids.dtype], ids.stride(0), B, L, D, _ptr(out), *_aux_args(aux),
                  _ptr(valid), _stream())
        _set_aux_hint(out, aux)
        return out, valid

    @staticmethod
    def backward(ctx, g, _gvalid):
        B, L, D, ns, nt = ctx.shape
        dev = g.device
        dseq = [torch.empty((B, L, D), dtype=torch.float32, device=dev) for _ in range(ns)]
        dtgt = [torch.empty((B, D), dtype=torch.float32, device=dev) for _ in range(nt)]
        if B > 0:
            _lib.call("b2_transact_tokens_bwd", _ptr(_f32c(g)), B, L, D, ns, nt,
                      _arr(ctypes.c_void_p, [t.data_ptr() for t in dseq]),
                      _arr(ctypes.c_void_p, [t.data_ptr() for t in dtgt]), _stream())
        return (None, None) + tuple(dseq) + tuple(dtgt)


def transact_tokens(sequence_embs, target_embs, ids, want_aux=False):
    """TransAct's early-fusion tokens of one (target, sequence) pair and its key-padding mask: sequence_embs ns views
    (B, L, D), target_embs nt views (B, D) (a tuple of fields: their embeddings side by side), ids (B, L) the first
    sequence field's ids.  Returns (X (B L, D (ns + nt)), valid (B, L) uint8): valid is ids != 0, with the last slot of
    an all-padding sample set (TransActTransformer.adjust_mask).  want_aux: also write X's GEMM operand copy."""
    seqs, tgts = list(sequence_embs), list(target_embs)
    _require_cuda(*(seqs + tgts + [ids]))
    if not seqs or not tgts:
        raise ValueError("transact_tokens: %d sequence fields and %d target fields" % (len(seqs), len(tgts)))
    B, L, D = seqs[0].shape
    for v in seqs:
        if v.dim() != 3 or tuple(v.shape) != (B, L, D):
            raise ValueError("transact_tokens: sequence embeddings %s differ" % [tuple(t.shape) for t in seqs])
    for v in tgts:
        if tuple(v.shape) != (B, D):
            raise ValueError("transact_tokens: target embeddings %s are not (%d, %d)"
                             % ([tuple(t.shape) for t in tgts], B, D))
    if tuple(ids.shape) != (B, L):
        raise ValueError("transact_tokens: ids%s are not (%d, %d)" % (tuple(ids.shape), B, L))
    bound = transact_bound(L, D * (len(seqs) + len(tgts)), 1, len(seqs) + len(tgts), heads_apply=False)
    if bound is not None:
        raise NotImplementedError("TransAct kernels: " + bound)
    return _TransActTokens.apply((len(seqs), want_aux), ids, *(seqs + tgts))


class _TransActAttention(torch.autograd.Function):
    """ctx (B L, md) of the key-tiled masked self-attention on QKV (B L, 3 md) (b2_transact_attn_fwd), the
    probabilities never stored; backward: dQKV in two deterministic launches (b2_transact_attn_bwd)."""

    @staticmethod
    def forward(ctx, qkv, valid, cfg):
        B, L, md, heads, scale, drop, want_aux = cfg
        dev = qkv.device
        out = torch.empty((B * L, md), dtype=torch.float32, device=dev)
        ctx.cfg = cfg
        if B == 0:
            return out
        qkv = _f32c(qkv)
        aux = empty_aux(B * L, md, dev) if want_aux else None
        smax = torch.empty((B, heads, L), dtype=torch.float32, device=dev)
        ssum = torch.empty_like(smax)
        _lib.call("b2_transact_attn_fwd", _ptr(qkv), _ptr(valid), B, L, md, heads, scale, *_drop_args(drop),
                  _ptr(out), *_aux_args(aux), _ptr(smax), _ptr(ssum), _stream())
        _set_aux_hint(out, aux)
        ctx.save_for_backward(qkv, valid, out, smax, ssum)
        return out

    @staticmethod
    def backward(ctx, g):
        B, L, md, heads, scale, drop, _ = ctx.cfg
        if B == 0:
            return torch.zeros((0, 3 * md), dtype=torch.float32, device=g.device), None, None
        qkv, valid, out, smax, ssum = ctx.saved_tensors
        dqkv = torch.empty_like(qkv)
        delta = torch.empty_like(smax)
        _lib.call("b2_transact_attn_bwd", _ptr(qkv), _ptr(valid), _ptr(out), _ptr(_f32c(g)), _ptr(smax), _ptr(ssum),
                  B, L, md, heads, scale, *_drop_args(drop), _ptr(delta), _ptr(dqkv), *_aux_args(None), _stream())
        return dqkv, None, None


def transact_attention(qkv, valid, batch, seq_len, num_heads, dropout=0.0, snapshot=None, layer=0, want_aux=False):
    """nn.MultiheadAttention's core with a key-padding mask on the in-projection's output qkv (B L, 3 md) =
    [Q | K | V]: per head softmax((q sqrt(1 / dh)) k^T + mask) v, key j hidden iff valid[b, j] == 0 (valid (B, L)
    uint8, never all 0 in a row).  Rows of padded queries come out 0.  dropout > 0: the weights take the mask of layer
    `layer` of `snapshot` (dropout_snapshot; None: one of its own).  Returns (B L, md), before out_proj."""
    _require_cuda(qkv, valid)
    B, L = batch, seq_len
    md = qkv.shape[1] // 3 if qkv.dim() == 2 else 0
    if qkv.dim() != 2 or qkv.shape[0] != B * L or qkv.shape[1] != 3 * md:
        raise ValueError("transact_attention: qkv%s is not (%d, 3 model_dim)" % (tuple(qkv.shape), B * L))
    if valid.dtype != torch.uint8 or tuple(valid.shape) != (B, L) or not valid.is_contiguous():
        raise ValueError("transact_attention: valid must be a contiguous (%d, %d) uint8 mask" % (B, L))
    bound = transact_bound(L, md, num_heads)
    if bound is not None:
        raise NotImplementedError("TransAct kernels: " + bound)
    drop = None
    if dropout > 0:
        if snapshot is None:
            snapshot, layer = dropout_snapshot(qkv.device, 1), 0
        drop = (snapshot, layer) + dropout_consts(dropout)
    scale = float(ctypes.c_float(math.sqrt(1.0 / (md // num_heads))).value)
    return _TransActAttention.apply(qkv, valid, (B, L, md, num_heads, scale, drop, want_aux))


class _TransActOut(torch.autograd.Function):
    """The last k slots of y (B L, md), zeroed where padded, flattened to (B, k md), and (max_pool) the max over L with
    padded slots at -1e9, its winning slot per column saved (b2_transact_out_fwd); backward: dy "=" in one launch
    (b2_transact_out_bwd)."""

    @staticmethod
    def forward(ctx, y, valid, cfg):
        B, L, k, pool, want_aux = cfg
        md = y.shape[1]
        dev = y.device
        last = torch.empty((B, k * md), dtype=torch.float32, device=dev)
        maxv = torch.empty((B, md), dtype=torch.float32, device=dev) if pool else None
        arg = torch.empty((B, md), dtype=torch.int32, device=dev) if pool else None
        ctx.cfg = cfg
        ctx.save_for_backward(valid, arg)
        if B > 0:
            aux = empty_aux(B, md, dev) if (pool and want_aux) else None
            _lib.call("b2_transact_out_fwd", _ptr(_f32c(y)), _ptr(valid), B, L, md, k, _ptr(last), _ptr(maxv),
                      _ptr(arg), *_aux_args(aux), _stream())
            if aux is not None:
                _set_aux_hint(maxv, aux)
        return (last, maxv) if pool else last

    @staticmethod
    def backward(ctx, glast, gmax=None):
        B, L, k, pool, _ = ctx.cfg
        valid, arg = ctx.saved_tensors
        md = glast.shape[1] // k
        dy = torch.empty((B * L, md), dtype=torch.float32, device=glast.device)
        if B > 0:
            if pool and gmax is None:
                gmax = torch.zeros((B, md), dtype=torch.float32, device=glast.device)
            _lib.call("b2_transact_out_bwd", _ptr(_f32c(glast)), _ptr(_f32c(gmax) if pool else None),
                      _ptr(arg), _ptr(valid), B, L, md, k, _ptr(dy), _stream())
        return dy, None, None


def transact_output(y, valid, batch, seq_len, first_k_cols=1, max_pool=True, want_aux=False):
    """TransActTransformer's head on the encoder output y (B L, md): (last, maxv) with last (B, k md) the last k slots,
    zeroed where padded, and maxv (B, md) the max over L with padded slots at -1e9 (ties: the first slot), or last
    alone when not max_pool.  want_aux: also write maxv's GEMM operand copy for out_linear."""
    _require_cuda(y, valid)
    B, L = batch, seq_len
    if y.dim() != 2 or y.shape[0] != B * L:
        raise ValueError("transact_output: y%s is not (%d, model_dim)" % (tuple(y.shape), B * L))
    if valid.dtype != torch.uint8 or tuple(valid.shape) != (B, L) or not valid.is_contiguous():
        raise ValueError("transact_output: valid must be a contiguous (%d, %d) uint8 mask" % (B, L))
    if not 1 <= first_k_cols <= L:
        raise ValueError("transact_output: first_k_cols=%d outside [1, %d]" % (first_k_cols, L))
    bound = transact_bound(L, y.shape[1], 1, heads_apply=False)
    if bound is not None:
        raise NotImplementedError("TransAct kernels: " + bound)
    return _TransActOut.apply(y, valid, (B, L, int(first_k_cols), bool(max_pool), want_aux))


# --------------------------------------------------------------------------------------
# DIEN (include/fuxictr_b200.h "DIEN")
# --------------------------------------------------------------------------------------
DIEN_CELL = {"GRU": _lib.B2_DIEN_GRU, "AUGRU": _lib.B2_DIEN_AUGRU, "AGRU": _lib.B2_DIEN_AGRU}


def dien_bound(model_dim, seq_len):
    """None when the DIEN kernels cover a GRU of width model_dim over seq_len positions, else the bound it breaks."""
    if not 1 <= model_dim <= _lib.B2_DIEN_MAX_DIM:
        return "the GRU width model_dim must lie in [1, %d], got %d" % (_lib.B2_DIEN_MAX_DIM, model_dim)
    if not 1 <= seq_len <= _lib.B2_DIEN_MAX_LEN:
        return "the sequence's max_len must lie in [1, %d], got %d" % (_lib.B2_DIEN_MAX_LEN, seq_len)
    return None


def _dien_seq(x):
    """x (B, L, H) as the kernels read it: fp32, each sample's tokens contiguous, samples at any pitch."""
    if x.dtype == torch.float32 and x.stride(2) == 1 and x.stride(1) == x.shape[2] and x.stride(0) >= x.shape[1] * x.shape[2]:
        return x
    return x.float().contiguous()


def _param_grad(param, need):
    return _grad_buffer(param, zero=True) if need else torch.zeros_like(param)


class _GruSequence(torch.autograd.Function):
    """(h_seq (B, L, H), h_last (B, H)) of one GRU over the sequence (b2_gru_fwd); backward: the reverse-time
    recurrence in one launch (b2_gru_bwd).  With a sink, x's gradient goes into the sink's buffer (x is a shared_grad
    view) and none is returned."""

    @staticmethod
    def forward(ctx, x, mask, att, cfg, W_ih, b_ih, W_hh, b_hh):
        cell, sink = cfg
        ctx.set_materialize_grads(False)
        x = _dien_seq(x)
        B, L, H = x.shape
        dev = x.device
        a = _f32c(att) if att is not None else None
        h_seq = torch.empty((B, L, H), dtype=torch.float32, device=dev)
        h_last = torch.empty((B, H), dtype=torch.float32, device=dev)
        if B > 0:       # an empty batch makes no launch
            _lib.call("b2_gru_fwd", _ptr(x), x.stride(0), _ptr(mask), _ptr(W_ih), _ptr(b_ih), _ptr(W_hh), _ptr(b_hh),
                      _ptr(a), cell, B, L, H, _ptr(h_seq), _ptr(h_last), _stream())
        ctx.cfg = cfg
        ctx.params = (W_ih, b_ih, W_hh, b_hh)
        ctx.save_for_backward(x, mask, a, h_seq)
        return h_seq, h_last

    @staticmethod
    def backward(ctx, dh_seq, dh_last):
        cell, sink = ctx.cfg
        x, mask, a, h_seq = ctx.saved_tensors
        W_ih, b_ih, W_hh, b_hh = ctx.params
        need = ctx.needs_input_grad
        B, L, H = x.shape
        if sink is not None:
            dx, acc = sink.target(h_seq)
        else:
            dx, acc = torch.empty((B, L, H), dtype=torch.float32, device=x.device), False
        da = torch.empty((B, L), dtype=torch.float32, device=x.device) if a is not None else None
        gW_ih, gb_ih, gW_hh, gb_hh = (_param_grad(p, need[4 + i]) for i, p in enumerate(ctx.params))
        if B > 0:       # an empty batch makes no launch
            _lib.call("b2_gru_bwd", _ptr(x), x.stride(0), _ptr(mask), _ptr(W_ih), _ptr(b_ih), _ptr(W_hh), _ptr(b_hh),
                      _ptr(a), cell, B, L, H, _ptr(h_seq), _ptr(_f32c(dh_seq) if dh_seq is not None else None),
                      _ptr(_f32c(dh_last) if dh_last is not None else None), _ptr(dx), int(acc), _ptr(da), _ptr(gW_ih),
                      _ptr(gb_ih), _ptr(gW_hh), _ptr(gb_hh), _stream())
        grads = tuple(g if need[4 + i] else None for i, g in enumerate((gW_ih, gb_ih, gW_hh, gb_hh)))
        return (dx if sink is None else None, None, da if a is not None and need[2] else None, None) + grads


def _dien_mask(mask, B, L):
    if mask.dtype != torch.uint8 or tuple(mask.shape) != (B, L) or not mask.is_contiguous():
        raise ValueError("DIEN: the mask must be a contiguous (%d, %d) uint8 tensor" % (B, L))
    return mask


def gru_sequence(x, mask, W_ih, b_ih, W_hh, b_hh, cell="GRU", att=None, sink=None):
    """One GRU over x (B, L, H) from h = 0: (h_seq (B, L, H), h_last (B, H)).  mask (B, L) uint8: a sample's length is
    its number of non-zero bytes (pad_mask.sum(1)), the recurrence runs over positions [0, len) and h_seq is zero from
    len on; h_last is the state after step len - 1, zero for an empty history (pack_padded_sequence, nn.GRU,
    pad_packed_sequence and DIEN.get_unmasked_tensor).  cell: "GRU" (nn.GRU's gates r, z, n), "AUGRU" or "AGRU"
    (DIEN's AUGRUCell / AGRUCell, chunks u, r, n of x2h / h2h, with the attention att (B, L)).  sink: x is a
    shared_grad view whose gradient this adds into the sink's buffer."""
    _require_cuda(x, mask, W_ih, b_ih, W_hh, b_hh, att)
    if cell not in DIEN_CELL:
        raise ValueError("gru_sequence: cell must be one of %s, got %r" % (sorted(DIEN_CELL), cell))
    if x.dim() != 3:
        raise ValueError("gru_sequence: x%s is not (B, L, H)" % (tuple(x.shape),))
    B, L, H = x.shape
    bound = dien_bound(H, L)
    if bound is not None:
        raise NotImplementedError("DIEN kernels: " + bound)
    _dien_mask(mask, B, L)
    if tuple(W_ih.shape) != (3 * H, H) or tuple(W_hh.shape) != (3 * H, H) or b_ih.numel() != 3 * H \
            or b_hh.numel() != 3 * H:
        raise ValueError("gru_sequence: the weights must be (3H, H) and the biases (3H,) for H = %d" % H)
    if (cell == "GRU") != (att is None) or (att is not None and tuple(att.shape) != (B, L)):
        raise ValueError("gru_sequence: AUGRU and AGRU take an attention (%d, %d), GRU none" % (B, L))
    return _GruSequence.apply(x, mask, att, (DIEN_CELL[cell], sink), W_ih, b_ih, W_hh, b_hh)


class _DienScores(torch.autograd.Function):
    """s (B, L) = <h_t, W t> mask (bilinear) or <h_t, t> mask (dot) (b2_dien_scores_fwd); backward: dh added into the
    sink's buffer (or returned), dt, and dW = dq^T t on the SIMT GEMM."""

    @staticmethod
    def forward(ctx, h, target, mask, sink, W):
        B, L, H = h.shape
        dev = h.device
        t = target if (target.dtype == torch.float32 and target.stride(1) == 1) else target.float().contiguous()
        q = torch.empty((B, H), dtype=torch.float32, device=dev)
        s = torch.empty((B, L), dtype=torch.float32, device=dev)
        Wc = _f32c(W) if W is not None else None
        if B > 0:       # an empty batch makes no launch
            _lib.call("b2_dien_scores_fwd", _ptr(h), _ptr(t), t.stride(0), _ptr(Wc), _ptr(mask), B, L, H, _ptr(q), _ptr(s),
                      _stream())
        ctx.sink, ctx.W = sink, W
        ctx.save_for_backward(h, t, mask, q)
        return s

    @staticmethod
    def backward(ctx, ds):
        h, t, mask, q = ctx.saved_tensors
        sink, W = ctx.sink, ctx.W
        B, L, H = h.shape
        if sink is not None:
            dh, acc = sink.target(h)
        else:
            dh, acc = torch.empty_like(h), False
        dq = torch.empty((B, H), dtype=torch.float32, device=h.device)
        dt = torch.empty((B, H), dtype=torch.float32, device=h.device)
        if B > 0:       # an empty batch makes no launch
            _lib.call("b2_dien_scores_bwd", _ptr(h), _ptr(t), t.stride(0), _ptr(W), _ptr(mask), _ptr(q), _ptr(_f32c(ds)),
                      B, L, H, _ptr(dh), int(acc), _ptr(dq), _ptr(dt), _stream())
        gW = None
        if W is not None and ctx.needs_input_grad[4]:
            gW = _grad_buffer(W, zero=False)
            if B > 0:
                gemm_f32(dq, t, gW, a_t=True)
            else:
                gW.zero_()
        return (dh if sink is None else None), dt, None, None, gW


def dien_scores(interest, target, mask, W_kernel=None, sink=None):
    """AttentionLayer's bilinear (W_kernel (H, H)) or dot (W_kernel None) scores on the interests (B, L, H) against
    the target (B, H), times mask (B, L) uint8: (B, L).  sink: interest is a shared_grad view."""
    _require_cuda(interest, target, mask, W_kernel)
    if interest.dim() != 3:
        raise ValueError("dien_scores: interest%s is not (B, L, H)" % (tuple(interest.shape),))
    B, L, H = interest.shape
    bound = dien_bound(H, L)
    if bound is not None:
        raise NotImplementedError("DIEN kernels: " + bound)
    _dien_mask(mask, B, L)
    if tuple(target.shape) != (B, H) or (W_kernel is not None and tuple(W_kernel.shape) != (H, H)):
        raise ValueError("dien_scores: target%s or W_kernel does not match H = %d" % (tuple(target.shape), H))
    return _DienScores.apply(_f32c(interest), target, mask, sink, W_kernel)


def dien_softmax(scores, mask):
    """softmax_L(s mask - 1e9 (1 - mask)), AttentionLayer's use_attention_softmax (b2_din_softmax_fwd / _bwd)."""
    return _DinSoftmax.apply(scores, mask)


class _DienDinInput(torch.autograd.Function):
    """[t, h, t - h, t h] ((B L), 4H) of din_attention (b2_din_input_fwd); backward adds dh into the sink's buffer."""

    @staticmethod
    def forward(ctx, target, hist, sink):
        target = _f32c(target)
        B, L, d = hist.shape
        out = torch.empty((B * L, 4 * d), dtype=torch.float32, device=hist.device)
        _lib.call("b2_din_input_fwd", _ptr(target), _ptr(hist), B, L, d, _ptr(out), _stream())
        ctx.sink = sink
        ctx.save_for_backward(target, hist)
        return out

    @staticmethod
    def backward(ctx, gin):
        target, hist = ctx.saved_tensors
        B, L, d = hist.shape
        gt = torch.empty_like(target)
        gh, acc = ctx.sink.target(hist)
        _lib.call("b2_din_input_bwd", _ptr(target), _ptr(hist), _ptr(_f32c(gin)), B, L, d, _ptr(gt), _ptr(gh),
                  int(acc), _stream())
        return gt, None, None


def dien_din_input(target, interest, sink):
    """din_attention's MLP input from the target (B, H) and the interests (B, L, H), a shared_grad view with its sink."""
    _require_cuda(target, interest)
    return _DienDinInput.apply(target, _f32c(interest), sink)


class _DienSumPool(torch.autograd.Function):
    """[sum_t x_t | t * sum_t x_t] (B, 2H) of DIEN's enable_sum_pooling (b2_dien_sum_pool_fwd / _bwd)."""

    @staticmethod
    def forward(ctx, x, target):
        x = x.float().contiguous()
        t = target if (target.dtype == torch.float32 and target.stride(1) == 1) else target.float().contiguous()
        B, L, H = x.shape
        out = torch.empty((B, 2 * H), dtype=torch.float32, device=x.device)
        if B > 0:       # an empty batch makes no launch
            _lib.call("b2_dien_sum_pool_fwd", _ptr(x), _ptr(t), t.stride(0), B, L, H, _ptr(out), 2 * H, _stream())
        ctx.save_for_backward(x, t)
        return out

    @staticmethod
    def backward(ctx, g):
        x, t = ctx.saved_tensors
        B, L, H = x.shape
        g = _f32c(g)
        dx = torch.empty_like(x)
        dt = torch.empty((B, H), dtype=torch.float32, device=x.device)
        if B > 0:       # an empty batch makes no launch
            _lib.call("b2_dien_sum_pool_bwd", _ptr(x), _ptr(t), t.stride(0), _ptr(g), g.stride(0), B, L, H, _ptr(dx),
                      _ptr(dt), 0, _stream())
        return dx, dt


def dien_sum_pool(sequence_emb, target):
    """(B, 2H): MaskedSumPooling of the zero-padded sequence (B, L, H) and its product with the target (B, H)."""
    _require_cuda(sequence_emb, target)
    B, L, H = sequence_emb.shape
    bound = dien_bound(H, L)
    if bound is not None:
        raise NotImplementedError("DIEN kernels: " + bound)
    if tuple(target.shape) != (B, H):
        raise ValueError("dien_sum_pool: target%s is not (%d, %d)" % (tuple(target.shape), B, H))
    return _DienSumPool.apply(sequence_emb, target)


# --------------------------------------------------------------------------------------
# FinalNet (include/fuxictr_b200.h "FinalNet")
# --------------------------------------------------------------------------------------
FINALNET_RESIDUAL = {"concat": _lib.B2_FINALNET_CONCAT, "sum": _lib.B2_FINALNET_SUM}


def finalnet_bound(widths=(), fields=None, embedding_dim=None):
    """None when the FinalNet kernels cover FinalBlock layers of output widths `widths` and, with `fields`, a
    FeatureGating over (fields, embedding_dim); else the bound it breaks."""
    for n in widths:
        if not 1 <= n <= _lib.B2_FINALNET_MAX_WIDTH:
            return "FinalBlock hidden units must lie in [1, %d], got %d" % (_lib.B2_FINALNET_MAX_WIDTH, n)
    if fields is not None:
        if not 1 <= fields <= _lib.B2_FINALNET_MAX_FIELDS:
            return "feature gating needs 1 to %d fields, got %d" % (_lib.B2_FINALNET_MAX_FIELDS, fields)
        if not 1 <= embedding_dim <= _lib.B2_FINALNET_MAX_DIM:
            return "feature gating needs embedding_dim in [1, %d], got %d" % (_lib.B2_FINALNET_MAX_DIM, embedding_dim)
        if fields * embedding_dim > _lib.B2_FINALNET_MAX_GATE_WIDTH:
            return "feature gating needs fields * embedding_dim <= %d, got %d" % (_lib.B2_FINALNET_MAX_GATE_WIDTH,
                                                                                  fields * embedding_dim)
    return None


class _FactorizedInteraction(torch.autograd.Function):
    """One FinalBlock layer (FinalNet.py, FinalBlock.forward with FactorizedInteraction) as one GEMM and the row
    kernels of include/fuxictr_b200.h "FinalNet": h = x W^T + b (bias in the epilogue), out = dropout(act(BN(z))) with
    z the product form of h (b2_finalnet_fi_fwd, which also writes out's operand copy for the next layer's GEMM when
    asked).  Backward: dh, the bias and the BatchNorm gradients (b2_finalnet_fi_bwd), dx = dh W (added into the
    EmbeddingGrad buffer when x is a shared_grad view), dW = dh^T x.  bn: None, or (training, eps, momentum,
    running_mean, running_var, num_batches_tracked) of the layer's nn.BatchNorm1d, whose buffers the kernels update."""

    @staticmethod
    def forward(ctx, x, sink, cfg, W, b, gamma, beta):
        residual, act, bn, drop, want_aux = cfg
        ctx.params, ctx.cfg, ctx.sink = (W, b, gamma, beta), cfg, sink
        B = x.shape[0]
        H = W.shape[0]
        half = H // 2
        n = 2 * half if residual == _lib.B2_FINALNET_CONCAT else half
        dev = x.device
        out = torch.empty((B, n), dtype=torch.float32, device=dev)
        if B == 0:          # no rows: no launch (an empty tensor has no device address)
            ctx.tc, ctx.x_aux, ctx.ws = False, None, None
            ctx.save_for_backward(x, None, None, None)
            return out
        tc = _tc_layer_ok(W) and x.data_ptr() % 16 == 0
        x_aux = (sink.emb_aux(x) if sink is not None else make_aux(x)) if tc else None
        h = torch.empty((B, H), dtype=torch.float32, device=dev)
        _linear_fwd(tc, x, x_aux, W, h, bias=b)
        out_aux = empty_aux(B, n, dev) if want_aux else None
        mean = rstd = ws = None
        training, eps, momentum, rm, rv, nbt = bn if bn is not None else (0, 0.0, 0.0, None, None, None)
        if bn is not None:
            mean = torch.empty(n, dtype=torch.float32, device=dev)
            rstd = torch.empty_like(mean)
            ws = torch.empty(4 * n, dtype=torch.float64, device=dev)
        _lib.call("b2_finalnet_fi_fwd", _ptr(h), B, half, residual, _ptr(gamma), _ptr(beta), eps, momentum,
                  int(training), _ptr(rm), _ptr(rv), _ptr(nbt), _ptr(ws), act, *_drop_args(drop), _ptr(out),
                  *_aux_args(out_aux), _ptr(mean), _ptr(rstd), _stream())
        if out_aux is not None:         # the next layer's make_aux finds it
            out._b2_aux = (_MATMUL["mode"], out_aux, out._version)
        ctx.save_for_backward(x, h, mean, rstd)
        ctx.tc, ctx.x_aux, ctx.ws = tc, x_aux, ws
        return out

    @staticmethod
    def backward(ctx, g):
        x, h, mean, rstd = ctx.saved_tensors
        W, b, gamma, beta = ctx.params
        residual, act, bn, drop, _ = ctx.cfg
        sink, tc = ctx.sink, ctx.tc
        B = x.shape[0]
        H = W.shape[0]
        half = H // 2
        n = 2 * half if residual == _lib.B2_FINALNET_CONCAT else half
        gW = _grad_buffer(W, zero=False)
        gb = _grad_buffer(b, zero=True) if b is not None else None
        gg = _grad_buffer(gamma, zero=False) if gamma is not None else None
        gbe = _grad_buffer(beta, zero=False) if beta is not None else None
        if B == 0:          # every gradient is zero; a shared buffer is left to its other writers
            for t in (gW, gg, gbe):
                if t is not None:
                    t.zero_()
            gx = torch.zeros_like(x) if sink is None and ctx.needs_input_grad[0] else None
            return gx, None, None, gW, gb, gg, gbe
        g = _f32c(g)
        dh = torch.empty((B, H), dtype=torch.float32, device=x.device)
        dh_aux = empty_aux(B, H, x.device) if tc else None
        training = bool(bn[0]) if bn is not None else False
        ws = ctx.ws[2 * n:] if bn is not None else None
        _lib.call("b2_finalnet_fi_bwd", _ptr(h), B, half, residual, _ptr(gamma), _ptr(beta), _ptr(mean), _ptr(rstd),
                  int(training), _ptr(ws), 0 if training else 1, act, *_drop_args(drop), _ptr(g), _ptr(dh),
                  *_aux_args(dh_aux), _ptr(gb), _ptr(gg), _ptr(gbe), _stream())
        if tc and dh_aux is None:
            dh_aux = make_aux(dh)
        gx = None
        if sink is not None:
            target, acc = sink.target(x)
            _linear_dgrad(tc, dh, dh_aux, W, target, accumulate=acc)
        elif ctx.needs_input_grad[0]:
            gx = torch.empty_like(x)
            _linear_dgrad(tc, dh, dh_aux, W, gx)
        _linear_wgrad(tc, dh, dh_aux, x, ctx.x_aux, gW)
        return gx, None, None, gW, gb, gg, gbe


def factorized_interaction(x, weight, bias=None, residual_type="sum", sink=None, batch_norm=None, act=B2_ACT_NONE,
                           dropout=None, want_aux=False):
    """One FinalBlock layer on x (B, K): FactorizedInteraction(x) with weight (2m, K) and bias (2m,), then the optional
    BatchNorm1d, activation and dropout.  batch_norm: (nn.BatchNorm1d, training) or None; act: B2_ACT_NONE,
    B2_ACT_RELU or B2_ACT_SIGMOID; dropout: (snapshot, layer, p) (dropout_snapshot) or None.  sink: x is a shared_grad
    view whose gradient is added into that EmbeddingGrad.  want_aux: also write the output's GEMM operand copy."""
    _require_cuda(x, weight)
    if residual_type not in FINALNET_RESIDUAL:
        raise ValueError("residual_type must be 'concat' or 'sum', got %r" % (residual_type,))
    if act not in (B2_ACT_NONE, B2_ACT_RELU, B2_ACT_SIGMOID):
        raise NotImplementedError("factorized_interaction: activation code %r" % (act,))
    H, K = weight.shape
    residual = FINALNET_RESIDUAL[residual_type]
    if x.dim() != 2 or x.shape[1] != K or H % 2 or (bias is not None and tuple(bias.shape) != (H,)):
        raise ValueError("factorized_interaction: shapes x%s weight%s do not match" % (tuple(x.shape),
                                                                                      tuple(weight.shape)))
    n = H if residual == _lib.B2_FINALNET_CONCAT else H // 2
    bound = finalnet_bound([n])
    if bound:
        raise NotImplementedError("FinalNet kernels: " + bound)
    bn = gamma = beta = None
    if batch_norm is not None:
        norm, training = batch_norm
        if norm.num_features != n or not norm.affine or not norm.track_running_stats or norm.momentum is None:
            raise NotImplementedError("FinalNet kernels: BatchNorm1d(%d) with affine, running statistics and a "
                                      "momentum, got %r" % (n, norm))
        if training and x.shape[0] == 1:
            raise ValueError("Expected more than 1 value per channel when training, got input size %s"
                             % ((1, n),))
        bn = (int(bool(training)), float(norm.eps), float(norm.momentum), norm.running_mean, norm.running_var,
              norm.num_batches_tracked)
        gamma, beta = norm.weight, norm.bias
    drop = None
    if dropout is not None:
        snap, layer, p = dropout
        drop = (snap, layer) + dropout_consts(p)
    return _FactorizedInteraction.apply(_f32c(x), sink, (residual, act, bn, drop, want_aux), weight, bias, gamma, beta)


class _FeatureGating(torch.autograd.Function):
    """FinalNet's FeatureGating with gate_residual "concat" (FinalNet.py, FeatureGating.forward) on e (B, F D), one
    row kernel each way: out = [e, e * (W e + b)] over the field axis, flattened (b2_finalnet_gate_fwd, with the
    operand copy block 1's first GEMM reads).  Backward: e's gradient added into the EmbeddingGrad buffer (or a fresh
    one without a sink), dW and db (b2_finalnet_gate_bwd)."""

    @staticmethod
    def forward(ctx, e, sink, want_aux, W, b):
        ctx.params, ctx.sink = (W, b), sink
        B, FD = e.shape
        F = W.shape[0]
        out = torch.empty((B, 2 * FD), dtype=torch.float32, device=e.device)
        ctx.save_for_backward(e)
        if B == 0:
            return out
        out_aux = empty_aux(B, 2 * FD, e.device) if want_aux else None
        _lib.call("b2_finalnet_gate_fwd", _ptr(e), B, F, FD // F, _ptr(_f32c(W)), _ptr(_f32c(b)), _ptr(out),
                  *_aux_args(out_aux), _stream())
        if out_aux is not None:
            out._b2_aux = (_MATMUL["mode"], out_aux, out._version)
        return out

    @staticmethod
    def backward(ctx, g):
        (e,) = ctx.saved_tensors
        W, b = ctx.params
        sink = ctx.sink
        B, FD = e.shape
        F = W.shape[0]
        gW, gb = _grad_buffer(W, zero=True), _grad_buffer(b, zero=True)
        if sink is not None:
            de, acc = sink.target(e) if B > 0 else (None, False)
        else:
            de, acc = torch.empty_like(e), False
        if B > 0:
            _lib.call("b2_finalnet_gate_bwd", _ptr(e), B, F, FD // F, _ptr(_f32c(W)), _ptr(_f32c(b)), _ptr(_f32c(g)),
                      _ptr(de), 1 if acc else 0, _ptr(gW), _ptr(gb), _stream())
        return (de if sink is None else None), None, None, gW, gb


def feature_gating(feature_emb, weight, bias, sink=None, want_aux=False):
    """[e, e * gates] flattened to (B, 2 F D), gates = Linear(F, F) over the field axis of feature_emb (B, F, D) or
    its flatten (B, F D) (a shared_grad view with its `sink`).  want_aux: also write the operand copy of the output."""
    _require_cuda(feature_emb, weight, bias)
    F = weight.shape[0]
    B = feature_emb.shape[0]
    e = feature_emb.reshape(B, -1) if feature_emb.dim() == 3 else feature_emb
    if tuple(weight.shape) != (F, F) or tuple(bias.shape) != (F,) or e.dim() != 2 or e.shape[1] % F:
        raise ValueError("feature_gating: shapes feature_emb%s weight%s bias%s do not match"
                         % (tuple(feature_emb.shape), tuple(weight.shape), tuple(bias.shape)))
    bound = finalnet_bound(fields=F, embedding_dim=e.shape[1] // F)
    if bound:
        raise NotImplementedError("FinalNet kernels: " + bound)
    return _FeatureGating.apply(e if sink is not None else _f32c(e), sink, want_aux, weight, bias)


class _FinalNetLoss(torch.autograd.Function):
    """FinalNet's two-block loss (FinalNet.py, add_loss with block_type "2B") from the logits y1, y2 in one launch
    (b2_finalnet_loss); also returns y_pred = sigmoid((y1 + y2) / 2) (not differentiable)."""

    @staticmethod
    def forward(ctx, label, y1, y2):
        ctx.shapes = (y1.shape, y2.shape)
        y1, y2 = _f32c(y1).view(-1), _f32c(y2).view(-1)
        B = y1.numel()
        dev = y1.device
        label = _f32c(label).view(-1)
        y_pred = torch.empty((B, 1), dtype=torch.float32, device=dev)
        loss = torch.empty((), dtype=torch.float32, device=dev)
        g1 = torch.empty((B,), dtype=torch.float32, device=dev)
        g2 = torch.empty_like(g1)
        _lib.call("b2_finalnet_loss", _ptr(y1), _ptr(y2), _ptr(label), B, _ptr(loss), _ptr(y_pred), _ptr(g1),
                  _ptr(g2), _stream())
        ctx.save_for_backward(g1, g2)
        ctx.mark_non_differentiable(y_pred)
        return loss, y_pred

    @staticmethod
    def backward(ctx, gloss, _gy):
        g1, g2 = ctx.saved_tensors
        return None, (g1 * gloss).view(ctx.shapes[0]), (g2 * gloss).view(ctx.shapes[1])


def finalnet_loss(label, y1, y2):
    """(loss, y_pred) of FinalNet's 2B loss, BCE(y_pred, y) + BCE(sigmoid(y1), p) + BCE(sigmoid(y2), p) with
    y_pred = p = sigmoid((y1 + y2) / 2) held constant in the last two terms; y1, y2 (B, 1) or (B,) logits."""
    _require_cuda(label, y1, y2)
    if y1.numel() != y2.numel() or y1.numel() != label.numel() or y1.numel() < 1:
        raise ValueError("finalnet_loss: y1, y2 and label must hold the same number (>= 1) of values")
    return _FinalNetLoss.apply(label, y1, y2)


# --------------------------------------------------------------------------------------
# WuKong (include/fuxictr_b200.h "WuKong")
# --------------------------------------------------------------------------------------
def wukong_bound(fields, out_fields, embedding_dim, rank_k):
    """None when the WuKong row kernels cover a layer of `fields` input and `out_fields` output fields, embedding_dim
    D and rank k, else the bound it breaks."""
    if rank_k is None:
        return "fmp_rank_k=None (the vanilla FM, F^2 wide) is not implemented; give a rank"
    for name, v, hi in (("the number of input fields", fields, _lib.B2_WUKONG_MAX_FIELDS),
                        ("lcb_features + fmb_features", out_fields, _lib.B2_WUKONG_MAX_FIELDS),
                        ("embedding_dim", embedding_dim, _lib.B2_WUKONG_MAX_DIM),
                        ("fmp_rank_k", rank_k, _lib.B2_WUKONG_MAX_RANK)):
        if not 1 <= v <= hi:
            return "%s must lie in [1, %d], got %d" % (name, hi, v)
    if fields * rank_k > _lib.B2_WUKONG_MAX_FM_WIDTH:
        return "input fields * fmp_rank_k must be at most %d, got %d" % (_lib.B2_WUKONG_MAX_FM_WIDTH, fields * rank_k)
    return None


def wukong_pitch(fields):
    """The field pitch of a WuKong layer's X' (B D, fp): fields rounded up to a multiple of 4."""
    return (fields + 3) // 4 * 4


def _wukong_tc_shape(n, k):
    """True when a field-axis GEMM with a stacked weight of (n, k) would take the tensor cores (_tc_layer_ok)."""
    return _MATMUL["mode"] != "fp32" and n >= 16 and k >= 16 and n % 4 == 0 and k % 4 == 0


class _WuKongFM(torch.autograd.Function):
    """The factorization-machine half of a WuKong layer (WuKong.py, FactorizationMachineBlock.optimized_fm and its
    LayerNorm), one launch each way (b2_wukong_fm_fwd / _bwd): fm = LN(flatten(x (x^T Y))).  Layout 0 reads the
    embedding (B, F, D) and also returns X'_0 (B D, fp), the layer's field-axis GEMM operand; layout 1 reads X' (a
    shared_grad view) and adds its gradient into the sink's buffer."""

    @staticmethod
    def forward(ctx, x, sink, cfg, Y, gamma, beta):
        layout, F, D, k, eps, fm_aux_on, xp_aux_on = cfg
        ctx.set_materialize_grads(False)
        ctx.params, ctx.sink, ctx.cfg = (Y, gamma, beta), sink, cfg
        B = x.shape[0] if layout == 0 else x.shape[0] // D
        dev = x.device
        fp = wukong_pitch(F)
        fm = torch.empty((B, F * k), dtype=torch.float32, device=dev)
        xp = torch.empty((B * D, fp), dtype=torch.float32, device=dev) if layout == 0 else None
        ctx.B = B
        if B == 0:
            ctx.save_for_backward(x, None, None)
            return (fm, xp) if layout == 0 else fm
        fm_aux = empty_aux(B, F * k, dev) if fm_aux_on else None
        xp_aux = empty_aux(B * D, fp, dev) if (xp_aux_on and xp is not None) else None
        mean = torch.empty(B, dtype=torch.float32, device=dev)
        rstd = torch.empty_like(mean)
        _lib.call("b2_wukong_fm_fwd", _ptr(x), layout, B, F, D, k, _ptr(_f32c(Y)), _ptr(gamma), _ptr(beta), eps,
                  _ptr(fm), *_aux_args(fm_aux), _ptr(xp), _ptr(xp_aux), xp_aux.stride(0) if xp_aux is not None else 0,
                  _ptr(mean), _ptr(rstd), _stream())
        for t, aux in ((fm, fm_aux), (xp, xp_aux)):
            if aux is not None:         # the consuming GEMM's make_aux finds it
                t._b2_aux = (_MATMUL["mode"], aux, t._version)
        ctx.save_for_backward(x, mean, rstd)
        return (fm, xp) if layout == 0 else fm

    @staticmethod
    def backward(ctx, g, gxp=None):
        layout, F, D, k, _, _, _ = ctx.cfg
        Y, gamma, beta = ctx.params
        x, mean, rstd = ctx.saved_tensors
        gY, dgamma, dbeta = (_grad_buffer(p, zero=True) for p in (Y, gamma, beta))
        if layout == 0:
            gx, acc = torch.zeros_like(x) if ctx.B == 0 else torch.empty_like(x), False
        else:
            gx, acc = ctx.sink.target(x)
        if ctx.B > 0:
            if g is None:
                g = torch.zeros((ctx.B, F * k), dtype=torch.float32, device=x.device)
            _lib.call("b2_wukong_fm_bwd", _ptr(x), layout, ctx.B, F, D, k, _ptr(_f32c(Y)), _ptr(gamma), _ptr(mean),
                      _ptr(rstd), _ptr(_f32c(g)), _ptr(_f32c(gxp) if gxp is not None else None), _ptr(gx),
                      1 if acc else 0, _ptr(gY), _ptr(dgamma), _ptr(dbeta), _stream())
        elif layout == 1 and not acc:
            gx.zero_()
        return (gx if layout == 0 else None, None, None, gY, dgamma, dbeta)


class _WuKongMix(torch.autograd.Function):
    """The rest of a WuKong layer (WuKong.py, WuKongLayer.forward after the FMB's MLP): one field-axis GEMM
    C = X' Ws^T + bs on Ws = [W_lcb; W_res] (packed by b2_wukong_pack with a projection residual or an X' pitch wider
    than F; W_lcb itself otherwise) and one row kernel (b2_wukong_out_fwd) that forms cat(FMB, LCB) + residual and the
    LayerNorm(D), writing the next layer's X' or, for the last layer, the (B, Fo D) flatten.  Backward: the row kernel
    (b2_wukong_out_bwd) writes the MLP output's gradient, dC and, for an identity residual, X''s gradient; the dgrad
    adds dC Ws into it, the wgrad forms dWs = dC^T X' (split by b2_wukong_unpack when packed).  X''s gradient goes into
    the sink's buffer (a shared_grad view), or is returned (layer 0, whose FM node takes it)."""

    @staticmethod
    def forward(ctx, xp, sink, mlp_out, cfg, W_lcb, W_res, b_res, gamma, beta):
        B, F, D, lcb, fmb, eps, last, want_aux = cfg
        ctx.set_materialize_grads(False)
        ctx.params, ctx.sink, ctx.cfg = (W_lcb, W_res, b_res, gamma, beta), sink, cfg
        Fo = lcb + fmb
        fpi, fpo = wukong_pitch(F), wukong_pitch(Fo)
        dev = xp.device
        proj = W_res is not None
        N = lcb + (Fo if proj else 0)
        out = torch.empty((B, Fo * D) if last else (B * D, fpo), dtype=torch.float32, device=dev)
        packed = proj or fpi != F
        ctx.shape = (N, fpi, packed)
        if B == 0:
            ctx.tc = False
            ctx.save_for_backward(xp, None, None, None, None, None)
            return out
        if packed:
            Ws = torch.empty((N, fpi), dtype=torch.float32, device=dev)
            bs = torch.empty(N, dtype=torch.float32, device=dev) if proj else None
            _lib.call("b2_wukong_pack", _ptr(_f32c(W_lcb)), _ptr(_f32c(W_res) if proj else None),
                      _ptr(_f32c(b_res) if proj else None), F, lcb, Fo, _ptr(Ws), _ptr(bs), _stream())
        else:
            Ws, bs = _f32c(W_lcb), None
        tc = _tc_layer_ok(Ws) and xp.data_ptr() % 16 == 0
        x_aux = make_aux(xp) if tc else None
        ws_aux = (make_aux(Ws) if packed else weight_aux(Ws)) if tc else None
        C = torch.empty((B * D, N), dtype=torch.float32, device=dev)
        _linear_fwd(tc, xp, x_aux, Ws, C, ws_aux, bias=bs)
        out_aux = (empty_aux(B, Fo * D, dev) if last else empty_aux(B * D, fpo, dev)) if want_aux else None
        ln = gamma is not None
        mean = torch.empty(B * Fo, dtype=torch.float32, device=dev) if ln else None
        rstd = torch.empty_like(mean) if ln else None
        _lib.call("b2_wukong_out_fwd", _ptr(mlp_out), _ptr(C), _ptr(xp), B, F, D, lcb, fmb, 2 if proj else 1,
                  _ptr(gamma), _ptr(beta), eps, 0 if last else 1, _ptr(out), *_aux_args(out_aux), _ptr(mean),
                  _ptr(rstd), _stream())
        if out_aux is not None:
            out._b2_aux = (_MATMUL["mode"], out_aux, out._version)
        ctx.save_for_backward(xp, mlp_out, C, Ws, mean, rstd)
        ctx.tc, ctx.aux = tc, (x_aux, ws_aux)
        return out

    @staticmethod
    def backward(ctx, g):
        B, F, D, lcb, fmb, _, last, _ = ctx.cfg
        W_lcb, W_res, b_res, gamma, beta = ctx.params
        xp, mlp_out, C, Ws, mean, rstd = ctx.saved_tensors
        N, fpi, packed = ctx.shape
        proj, ln = W_res is not None, gamma is not None
        sink = ctx.sink
        dev = xp.device
        if sink is not None:
            gx, acc = sink.target(xp)
        else:
            gx, acc = torch.empty_like(xp), False
        dgamma = _grad_buffer(gamma, zero=True) if ln else None
        dbeta = _grad_buffer(beta, zero=True) if ln else None
        dbias = _grad_buffer(b_res, zero=True) if proj else None
        gW_lcb = _grad_buffer(W_lcb, zero=False)
        gW_res = _grad_buffer(W_res, zero=False) if proj else None
        g_mlp = torch.zeros((B, fmb * D), dtype=torch.float32, device=dev) if B == 0 else \
            torch.empty((B, fmb * D), dtype=torch.float32, device=dev)
        if B == 0 or g is None:
            if not acc:
                gx.zero_()
            g_mlp.zero_()
            gW_lcb.zero_()
            if proj:
                gW_res.zero_()
            return (gx if sink is None else None, None, g_mlp, None, gW_lcb, gW_res, dbias, dgamma, dbeta)
        x_aux, ws_aux = ctx.aux
        tc = ctx.tc
        dC = torch.empty((B * D, N), dtype=torch.float32, device=dev)
        dc_aux = empty_aux(B * D, N, dev) if tc else None
        _lib.call("b2_wukong_out_bwd", _ptr(mlp_out), _ptr(C), _ptr(xp), B, F, D, lcb, fmb, 2 if proj else 1,
                  _ptr(gamma), _ptr(mean), _ptr(rstd), 0 if last else 1, _ptr(_f32c(g)), _ptr(g_mlp), _ptr(dC),
                  *_aux_args(dc_aux), _ptr(gx if not proj else None), 1 if acc else 0, _ptr(dbias), _ptr(dgamma),
                  _ptr(dbeta), _stream())
        _linear_dgrad(tc, dC, dc_aux, Ws, gx, ws_aux, accumulate=acc or not proj)               # dX' (+)= dC Ws
        if packed:
            dWs = torch.empty_like(Ws)
            _linear_wgrad(tc, dC, dc_aux, xp, x_aux, dWs)                                        # dWs = dC^T X'
            _lib.call("b2_wukong_unpack", _ptr(dWs), F, lcb, lcb + fmb, _ptr(gW_lcb), _ptr(gW_res), _stream())
        else:
            _linear_wgrad(tc, dC, dc_aux, xp, x_aux, gW_lcb)
        return (gx if sink is None else None, None, g_mlp, None, gW_lcb, gW_res, dbias, dgamma, dbeta)


def wukong_layer(x, proj_Y, fm_gamma, fm_beta, mlp, W_lcb, W_res=None, b_res=None, gamma=None, beta=None,
                 fm_eps=1e-5, eps=1e-5, embedding_dim=None, sink=None, last=True, fm_aux=False, want_aux=False):
    """One WuKong layer.  x: the embedding (B, F, D), or X' (B D, fp) as a shared_grad view with its sink and
    embedding_dim given (the previous layer's output with last=False).  proj_Y (F, k), fm_gamma, fm_beta (F k): the
    FMB's projection and LayerNorm; mlp: the FMB's MLP, a callable (B, F k) -> (B, fmb D); W_lcb (lcb, F): the LCB's
    weight; W_res (Fo, F), b_res (Fo): the residual projection (None: the identity, F == Fo); gamma, beta (D): the
    output LayerNorm (None: none).  Returns the (B, Fo D) flatten [b, f, d] when last, else X' (B D, fpo) for the
    next layer.  fm_aux: write the MLP input's GEMM operand copy; want_aux: the output's, for the GEMM that reads it."""
    _require_cuda(x, proj_Y, fm_gamma, fm_beta, W_lcb, W_res, b_res, gamma, beta)
    F, k = proj_Y.shape
    lcb = W_lcb.shape[0]
    if sink is None:
        if x.dim() != 3 or x.shape[1] != F:
            raise ValueError("wukong_layer: x%s is not (B, %d, D)" % (tuple(x.shape), F))
        B, _, D = x.shape
        layout = 0
    else:
        D = embedding_dim
        if D is None or x.dim() != 2 or x.shape[1] != wukong_pitch(F) or x.shape[0] % D:
            raise ValueError("wukong_layer: X'%s is not (B * %s, %d)" % (tuple(x.shape), D, wukong_pitch(F)))
        B = x.shape[0] // D
        layout = 1
    if W_res is not None:
        Fo = W_res.shape[0]
    else:
        Fo = F
    fmb = Fo - lcb
    bound = wukong_bound(F, Fo, D, k)
    if bound is not None:
        raise NotImplementedError("WuKong kernels: " + bound)
    if fmb < 1 or tuple(W_lcb.shape) != (lcb, F) or fm_gamma.numel() != F * k or fm_beta.numel() != F * k \
            or (W_res is not None and (tuple(W_res.shape) != (Fo, F) or b_res is None or b_res.numel() != Fo)):
        raise ValueError("wukong_layer: shapes x%s proj_Y%s W_lcb%s W_res%s do not match"
                         % (tuple(x.shape), tuple(proj_Y.shape), tuple(W_lcb.shape),
                            tuple(W_res.shape) if W_res is not None else None))
    if (gamma is None) != (beta is None) or (gamma is not None and (gamma.numel() != D or beta.numel() != D)):
        raise ValueError("wukong_layer: the output LayerNorm needs a weight and a bias of %d" % D)
    N = lcb + (Fo if W_res is not None else 0)
    x = _f32c(x)
    cfg = (layout, F, D, k, float(fm_eps), fm_aux, layout == 0 and _wukong_tc_shape(N, wukong_pitch(F)))
    if layout == 0:
        fm, xp = _WuKongFM.apply(x, None, cfg, proj_Y, fm_gamma, fm_beta)
    else:
        fm, xp = _WuKongFM.apply(x, sink, cfg, proj_Y, fm_gamma, fm_beta), x
    mlp_out = _f32c(mlp(fm)) if B > 0 else fm.new_zeros((0, fmb * D))     # an empty batch: nothing to multiply
    if tuple(mlp_out.shape) != (B, fmb * D):
        raise ValueError("wukong_layer: the FMB's MLP returned %s, not (%d, %d)" % (tuple(mlp_out.shape), B, fmb * D))
    cfg = (B, F, D, lcb, fmb, float(eps), bool(last), want_aux)
    return _WuKongMix.apply(xp, sink, mlp_out, cfg, W_lcb, W_res, b_res, gamma, beta)


class _FsGate(torch.autograd.Function):
    """FinalMLP's gating products f_s = e * (2 g_s), s = 1, 2 (FinalMLP.py, FeatureSelection.forward) in one launch
    (include/fuxictr_b200.h "FinalMLP"), which also writes f1's and f2's auxiliary operands for the towers' first
    GEMMs.  A gate of one row (1, d) is broadcast over the batch; its gradient is the column sum over the batch, so
    the gate MLP behind it runs its forward and backward on that one row.  Backward: one launch for de, dg1, dg2."""

    @staticmethod
    def forward(ctx, e, g1, g2):
        e, g1, g2 = _f32c(e), _f32c(g1), _f32c(g2)
        B, d = e.shape
        f1, f2 = torch.empty_like(e), torch.empty_like(e)
        a1, a2 = empty_aux(B, d, e.device), empty_aux(B, d, e.device)
        rows = (int(g1.shape[0] != 1), int(g2.shape[0] != 1))
        if B:                   # an empty batch has no rows to gate (and NULL data pointers)
            _lib.call("b2_fs_gate_fwd", _ptr(e), _ptr(g1), _ptr(g2), *rows, B, d, _ptr(f1), _ptr(f2), _ptr(a1),
                      _ptr(a2), *_aux_args(a1)[1:], _stream())
        for f, a in ((f1, a1), (f2, a2)):
            if a is not None:           # the tower's first layer (make_aux) finds it
                f._b2_aux = (_MATMUL["mode"], a, f._version)
        ctx.save_for_backward(e, g1, g2)
        ctx.rows = rows
        return f1, f2

    @staticmethod
    def backward(ctx, df1, df2):
        e, g1, g2 = ctx.saved_tensors
        df1, df2 = _f32c(df1), _f32c(df2)
        B, d = e.shape
        de = torch.empty_like(e)
        dg1 = torch.empty_like(g1) if ctx.rows[0] else torch.zeros_like(g1)
        dg2 = torch.empty_like(g2) if ctx.rows[1] else torch.zeros_like(g2)
        if B:
            _lib.call("b2_fs_gate_bwd", _ptr(e), _ptr(g1), _ptr(g2), *ctx.rows, _ptr(df1), _ptr(df2), B, d, _ptr(de),
                      _ptr(dg1), _ptr(dg2), _stream())
        return de, dg1, dg2


def fs_gate(flat_emb, g1, g2):
    """(flat_emb * (2 g1), flat_emb * (2 g2)): flat_emb (B, d); each gate (B, d), or (1, d) for every row."""
    _require_cuda(flat_emb, g1, g2)
    if flat_emb.dim() != 2:
        raise ValueError("fs_gate: flat_emb%s must be (B, d)" % (tuple(flat_emb.shape),))
    B, d = flat_emb.shape
    for g in (g1, g2):
        if g.dim() != 2 or g.shape[1] != d or g.shape[0] not in (1, B):
            raise ValueError("fs_gate: a gate%s must be (1, %d) or (%d, %d)" % (tuple(g.shape), d, B, d))
    return _FsGate.apply(flat_emb, g1, g2)


class _InteractionAggregation(torch.autograd.Function):
    """FinalMLP's InteractionAggregation at output_dim 1 (FinalMLP.py), out = w_x(x) + w_y(y) + sum_h x_h^T W_h y_h,
    as one GEMM between two row kernels (include/fuxictr_b200.h "FinalMLP"): W_aug = [block diagonal of the W_h^T;
    w_x; 0] and bias_aug = [w_y, 0] (b2_agg_pack), Q = x W_aug^T + bias_aug, out = y.Q[:, :dy] + Q[:, dy] + b_x + b_y
    (b2_agg_fwd).  Backward: dy, ys = [g y | g | 0] and the w_y, b_x, b_y gradients (b2_agg_bwd), dx = ys W_aug
    (one dgrad, which includes g w_x), dW_aug = ys^T x (one wgrad) and one b2_agg_unpack into the w_xy, w_x
    gradients.  W_aug changes every step, so its auxiliary operand is made here by make_aux and handed to gemm_ex as
    it is (None where the precision has none), never looked up in weight_aux's per-weight cache."""

    @staticmethod
    def forward(ctx, x, y, wx, bx, wy, by, wxy, heads):
        ctx.params = (wx, bx, wy, by, wxy)         # their gradients may live in an arena
        x, y = _f32c(x), _f32c(y)
        wx, bx, wy, by, wxy = _f32c(wx), _f32c(bx), _f32c(wy), _f32c(by), _f32c(wxy)
        B, dx = x.shape
        dy = y.shape[1]
        n = (dy + 4) // 4 * 4                      # B2_AGG_COLS
        dev = x.device
        W = torch.empty((n, dx), dtype=torch.float32, device=dev)
        bias = torch.empty((n,), dtype=torch.float32, device=dev)
        _lib.call("b2_agg_pack", _ptr(wxy), _ptr(wx), _ptr(wy), dx, dy, heads, _ptr(W), _ptr(bias), _stream())
        tc = _tc_layer_ok(W) and x.data_ptr() % 16 == 0 and B > 0
        x_aux = make_aux(x) if tc else None
        w_aux = make_aux(W) if tc else None
        Q = torch.empty((B, n), dtype=torch.float32, device=dev)
        out = torch.empty((B, 1), dtype=torch.float32, device=dev)
        if B:                   # an empty batch: nothing to multiply (and NULL data pointers)
            if tc:
                gemm_ex(x, W, Q, a_small=x_aux, b_small=w_aux, bias=bias)
            else:
                gemm_f32(x, W, Q, b_t=True, bias=bias)
            _lib.call("b2_agg_fwd", _ptr(Q), _ptr(y), _ptr(bx), _ptr(by), B, dy, _ptr(out), _stream())
        ctx.save_for_backward(x, y, Q, W)
        ctx.tc, ctx.aux, ctx.heads = tc, (x_aux, w_aux), heads
        return out

    @staticmethod
    def backward(ctx, g):
        x, y, Q, W = ctx.saved_tensors
        g = _f32c(g)
        x_aux, w_aux = ctx.aux
        tc = ctx.tc
        B, dx = x.shape
        dy = y.shape[1]
        dev = x.device
        wx, bx, wy, by, wxy = ctx.params
        need = ctx.needs_input_grad
        gy = torch.empty_like(y)
        ys = torch.empty((B, W.shape[0]), dtype=torch.float32, device=dev)
        ys_aux = empty_aux(B, W.shape[0], dev) if tc else None
        gwy = _grad_buffer(wy, zero=True) if need[4] else torch.zeros_like(wy)
        gbx = _grad_buffer(bx, zero=True) if need[3] else torch.zeros_like(bx)
        gby = _grad_buffer(by, zero=True) if need[5] else torch.zeros_like(by)
        gx = torch.empty_like(x)
        if B:
            _lib.call("b2_agg_bwd", _ptr(Q), _ptr(y), _ptr(g), B, dy, _ptr(gy), _ptr(ys), *_aux_args(ys_aux),
                      _ptr(gwy), _ptr(gbx), _ptr(gby), _stream())
            if tc:                                                                       # dx = ys W_aug
                gemm_ex(ys, W, gx, b_mn=True, a_small=ys_aux, b_small=w_aux)
            else:
                gemm_f32(ys, W, gx)
        gwx = gwxy = None
        if need[2] or need[6]:
            dW = torch.empty_like(W) if B else torch.zeros_like(W)
            if B:
                _linear_wgrad(tc, ys, ys_aux, x, x_aux, dW)                              # dW_aug = ys^T x
            gwx = _grad_buffer(wx, zero=False) if need[2] else torch.empty_like(wx)
            gwxy = _grad_buffer(wxy, zero=False) if need[6] else torch.empty_like(wxy)
            _lib.call("b2_agg_unpack", _ptr(dW), dx, dy, ctx.heads, _ptr(gwxy), _ptr(gwx), _stream())
        return (gx, gy, gwx if need[2] else None, gbx if need[3] else None, gwy if need[4] else None,
                gby if need[5] else None, gwxy if need[6] else None, None)


def interaction_aggregation(x, y, w_x, b_x, w_y, b_y, w_xy, num_heads):
    """InteractionAggregation.forward at output_dim 1, (B, 1): x (B, dx), y (B, dy); w_x (1, dx), b_x (1,), w_y (1, dy),
    b_y (1,) the w_x / w_y Linears' parameters; w_xy (num_heads * (dx / num_heads) * (dy / num_heads), 1)."""
    _require_cuda(x, y, w_x, b_x, w_y, b_y, w_xy)
    if x.dim() != 2 or y.dim() != 2 or x.shape[0] != y.shape[0]:
        raise ValueError("interaction_aggregation: x%s and y%s must be (B, dx) and (B, dy)"
                         % (tuple(x.shape), tuple(y.shape)))
    dx, dy = x.shape[1], y.shape[1]
    if num_heads < 1 or dx % num_heads or dy % num_heads:
        raise ValueError("interaction_aggregation: num_heads %d must divide dx %d and dy %d" % (num_heads, dx, dy))
    if w_x.numel() != dx or w_y.numel() != dy or b_x.numel() != 1 or b_y.numel() != 1 \
            or w_xy.numel() != dx * dy // num_heads:
        raise ValueError("interaction_aggregation: shapes w_x%s b_x%s w_y%s b_y%s w_xy%s do not match dx %d, dy %d"
                         % (tuple(w_x.shape), tuple(b_x.shape), tuple(w_y.shape), tuple(b_y.shape),
                            tuple(w_xy.shape), dx, dy))
    return _InteractionAggregation.apply(x, y, w_x, b_x, w_y, b_y, w_xy, num_heads)


# --------------------------------------------------------------------------------------
# MultiHeadTargetAttention
# --------------------------------------------------------------------------------------
def target_attention_bound(width, heads):
    """None when the MultiHeadTargetAttention kernels cover a row of `width` columns split into `heads` heads,
    else the bound it breaks.  width is the row of q' and p: heads * input_dim with the projections (use_qkvo),
    input_dim without."""
    if not 1 <= heads <= _lib.B2_MHTA_MAX_HEADS:
        return "num_heads must lie in [1, %d], got %d" % (_lib.B2_MHTA_MAX_HEADS, heads)
    if not 1 <= width <= _lib.B2_MHTA_MAX_WIDTH:
        return "the attention row width (num_heads * input_dim with use_qkvo, else input_dim) must lie in " \
               "[1, %d], got %d" % (_lib.B2_MHTA_MAX_WIDTH, width)
    return None


class _TargetAttention(torch.autograd.Function):
    """MultiHeadTargetAttention.forward (target_attention.py:150-172) on the kernels (include/fuxictr_b200.h
    "MultiHeadTargetAttention").  With the projections: W_M, W_N packed from W_q, W_k, W_v, W_o (b2_mhta_pack),
    q' = t W_M^T (GEMM1), the row kernel's masked online softmax and pooled p (b2_mhta_fwd), out = p W_N^T
    (GEMM2).  Backward: dp = g W_N, dW_N = g^T p, the row kernel back to dq' and dx (b2_mhta_bwd),
    dt = dq' W_M, dW_M = dq'^T t, and one unpack of dW_M, dW_N into the four weights.  Without them the row
    kernels alone, sliced by head: q = t, out = p.  The GEMMs follow the matmul precision (SIMT below 16 or
    off-by-4 shapes); the row kernels run in fp32."""

    @staticmethod
    def forward(ctx, t, x, mask_u8, heads, scale, Wq, Wk, Wv, Wo):
        t, x = _f32c(t), _f32c(x)
        B, L, d = x.shape
        H, dev = heads, x.device
        qkvo = Wq is not None
        tc, aux, packed = False, (None, None, None, None), (None, None)
        if qkvo:
            Wq, Wk, Wv, Wo = _f32c(Wq), _f32c(Wk), _f32c(Wv), _f32c(Wo)
            hd = Wq.shape[0] // H
            WM = torch.empty((H * d, d), dtype=torch.float32, device=dev)
            WN = torch.empty((d, H * d), dtype=torch.float32, device=dev)
            _lib.call("b2_mhta_pack", _ptr(Wq), _ptr(Wk), _ptr(Wv), _ptr(Wo), d, H, hd, scale, _ptr(WM), _ptr(WN),
                      _stream())
            tc = _tc_layer_ok(WM) and _tc_layer_ok(WN) and t.data_ptr() % 16 == 0
            if tc:
                aux = (make_aux(t), make_aux(WM), make_aux(WN), empty_aux(B, H * d, dev))
            q = torch.empty((B, H * d), dtype=torch.float32, device=dev)
            _linear_fwd(tc, t, aux[0], WM, q, aux[1])
            width, x_step, row_scale, packed = d, 0, 1.0, (WM, WN)
        else:
            q, width, x_step, row_scale = t, d // H, d // H, scale
        p = torch.empty((B, H * width), dtype=torch.float32, device=dev)
        stats = torch.empty((B, H, 2), dtype=torch.float32, device=dev)
        _lib.call("b2_mhta_fwd", _ptr(q), _ptr(x), _ptr(mask_u8), B, L, d, H, width, x_step, row_scale, _ptr(p),
                  _ptr(stats), *_aux_args(aux[3]), _stream())
        out = p
        if qkvo:
            out = torch.empty((B, d), dtype=torch.float32, device=dev)
            _linear_fwd(tc, p, aux[3], packed[1], out, aux[2])
        ctx.save_for_backward(t, x, q, p, stats, *packed, Wq, Wk, Wv, Wo)
        ctx.mask, ctx.tc, ctx.aux, ctx.geom = mask_u8, tc, aux, (H, width, x_step, row_scale, scale)
        return out

    @staticmethod
    def backward(ctx, g):
        t, x, q, p, stats, WM, WN, Wq, Wk, Wv, Wo = ctx.saved_tensors
        g = _f32c(g)
        t_aux, wm_aux, wn_aux, p_aux = ctx.aux
        H, width, x_step, row_scale, scale = ctx.geom
        tc, qkvo = ctx.tc, Wq is not None
        B, L, d = x.shape
        dev = x.device
        dp = g
        if qkvo:
            g_aux = make_aux(g) if tc else None
            dp = torch.empty((B, H * d), dtype=torch.float32, device=dev)
            dWN = torch.empty((d, H * d), dtype=torch.float32, device=dev)
            _linear_dgrad(tc, g, g_aux, WN, dp, wn_aux)                        # dp = g W_N
            _linear_wgrad(tc, g, g_aux, p, p_aux, dWN)                        # dW_N = g^T p
        dq = torch.empty((B, H * width), dtype=torch.float32, device=dev)
        dx = torch.empty_like(x)
        dq_aux = empty_aux(B, H * width, dev) if tc else None
        _lib.call("b2_mhta_bwd", _ptr(q), _ptr(x), _ptr(ctx.mask), _ptr(p), _ptr(stats), _ptr(dp), B, L, d, H, width,
                  x_step, row_scale, _ptr(dq), _ptr(dx), *_aux_args(dq_aux), _stream())
        if not qkvo:
            return dq, dx, None, None, None, None, None, None, None
        dt = torch.empty_like(t)
        dWM = torch.empty((H * d, d), dtype=torch.float32, device=dev)
        _linear_dgrad(tc, dq, dq_aux, WM, dt, wm_aux)                          # dt = dq' W_M
        _linear_wgrad(tc, dq, dq_aux, t, t_aux, dWM)                          # dW_M = dq'^T t
        gWq, gWk, gWv, gWo = (torch.empty_like(w) for w in (Wq, Wk, Wv, Wo))
        _lib.call("b2_mhta_unpack", _ptr(Wq), _ptr(Wk), _ptr(Wv), _ptr(Wo), _ptr(dWM), _ptr(dWN), d, H,
                  Wq.shape[0] // H, scale, _ptr(gWq), _ptr(gWk), _ptr(gWv), _ptr(gWo), _stream())
        return dt, dx, None, None, None, gWq, gWk, gWv, gWo


def target_attention(target_item, history_sequence, mask=None, num_heads=1, use_scale=True, W_q=None, W_k=None,
                     W_v=None, W_o=None):
    """MultiHeadTargetAttention with ScaledDotProductAttention (no attention dropout): target_item (B, d),
    history_sequence (B, L, d), mask any B*L elements (nonzero = valid) or None; W_q, W_k, W_v (A, d) and
    W_o (d, A), all four or none (use_qkvo False: A = d, heads slice the columns).  Returns (B, d)."""
    _require_cuda(target_item, history_sequence, mask, W_q, W_k, W_v, W_o)
    if history_sequence.dim() != 3 or target_item.dim() != 2:
        raise ValueError("target_attention: target%s history%s must be (B, d) and (B, L, d)"
                         % (tuple(target_item.shape), tuple(history_sequence.shape)))
    B, L, d = history_sequence.shape
    weights = (W_q, W_k, W_v, W_o)
    qkvo = W_q is not None
    if tuple(target_item.shape) != (B, d) or (mask is not None and mask.numel() != B * L) \
            or any((w is None) == qkvo for w in weights):
        raise ValueError("target_attention: target%s history%s mask%s or the weights do not match"
                         % (tuple(target_item.shape), tuple(history_sequence.shape),
                            None if mask is None else tuple(mask.shape)))
    A = W_q.shape[0] if qkvo else d
    if A % num_heads != 0 or (qkvo and (tuple(W_k.shape) != (A, d) or tuple(W_v.shape) != (A, d)
                                        or tuple(W_q.shape) != (A, d) or tuple(W_o.shape) != (d, A))):
        raise ValueError("target_attention: attention_dim %d, num_heads %d and the weights do not match"
                         % (A, num_heads))
    bound = target_attention_bound(num_heads * d if qkvo else d, num_heads)
    if bound is not None:
        raise NotImplementedError("MultiHeadTargetAttention kernels: " + bound)
    scale = 1.0 / (A // num_heads) ** 0.5 if use_scale else 1.0
    mask_u8 = None if mask is None else torch.ne(mask.reshape(B, L), 0).view(torch.uint8)
    return _TargetAttention.apply(target_item, history_sequence, mask_u8, num_heads, scale, *weights)


# --------------------------------------------------------------------------------------
# LongCTR interest blocks: ETA's SimHash top-k retrieval and SDIM's hash-collision pooling
# --------------------------------------------------------------------------------------
def _lsh_common_bound(batch, d, L):
    if not 1 <= d <= _lib.B2_LSH_MAX_DIM:
        return "the item width d (item_info_dim) must lie in [1, %d], got %d" % (_lib.B2_LSH_MAX_DIM, d)
    if not 1 <= L <= _lib.B2_LSH_MAX_LEN:
        return "the history length L must lie in [1, %d], got %d" % (_lib.B2_LSH_MAX_LEN, L)
    if batch * (L + 1) >= 2 ** 31:
        return "batch (L + 1) must stay below 2^31, got %d" % (batch * (L + 1))
    return None


def eta_bound(d, L, topk, hash_bits, batch=1):
    """None when the ETA kernels cover item width d, history length L, topk and hash_bits, else the bound it breaks."""
    msg = _lsh_common_bound(batch, d, L)
    if msg is not None:
        return msg
    if not 1 <= hash_bits <= _lib.B2_ETA_MAX_BITS:
        return "hash_bits must lie in [1, %d], got %d" % (_lib.B2_ETA_MAX_BITS, hash_bits)
    if not 1 <= topk <= _lib.B2_LSH_MAX_TOPK:
        return "topk must lie in [1, %d], got %d" % (_lib.B2_LSH_MAX_TOPK, topk)
    k = min(topk, L)
    if 4 * d * hash_bits + 4 * k + 4 * hash_bits + L + 16 > _lib.B2_LSH_MAX_SMEM:
        return "d hash_bits = %d needs more shared memory than a CTA has" % (d * hash_bits)
    return None


def sdim_bound(d, L, num_hashes, hash_bits, batch=1):
    """None when the SDIM kernels cover item width d, history length L, num_hashes and hash_bits, else the bound it
    breaks.  hash_bits stops at 24: above it the reference's float bucket code . powers_of_two is no longer exact, so
    its collisions cannot be reproduced."""
    msg = _lsh_common_bound(batch, d, L)
    if msg is not None:
        return msg
    if not 1 <= hash_bits <= _lib.B2_SDIM_MAX_BITS:
        return "hash_bits must lie in [1, %d] (a wider float bucket code is not exact), got %d" \
            % (_lib.B2_SDIM_MAX_BITS, hash_bits)
    if not 1 <= num_hashes <= _lib.B2_SDIM_MAX_HASHES:
        return "num_hashes must lie in [1, %d], got %d" % (_lib.B2_SDIM_MAX_HASHES, num_hashes)
    pool = 4 * d * num_hashes * hash_bits + 4 * (256 // d) * num_hashes * d + 4 * num_hashes + 4 * L
    if pool > _lib.B2_LSH_MAX_SMEM or 4 * num_hashes * d + 4 * L > _lib.B2_LSH_MAX_SMEM:
        return "d num_hashes hash_bits = %d needs more shared memory than a CTA has" % (d * num_hashes * hash_bits)
    return None


class _SavedCtx(object):
    """Stands in for an autograd ctx, so that an interest block's node can run _TargetAttention's forward and
    backward inside its own."""

    def save_for_backward(self, *tensors):
        self.saved_tensors = tensors


def _mhta_fwd(t, x, mask_u8, heads, scale, weights):
    ctx = _SavedCtx()
    out = _TargetAttention.forward(ctx, t, x, mask_u8, heads, scale, *(weights or (None,) * 4))
    return out, ctx


def _mhta_bwd(ctx, g):
    """(dt, dx, (dW_q, dW_k, dW_v, dW_o) or ())."""
    grads = _TargetAttention.backward(ctx, g)
    return grads[0], grads[1], tuple(w for w in grads[5:] if w is not None)


def _mhta_scale(weights, d, heads, use_scale):
    A = weights[0].shape[0] if weights else d
    return 1.0 / (A // heads) ** 0.5 if use_scale else 1.0


def _short_window(x, mask_u8, S):
    """The reference's item_feat_emb[:, -short_seq_len:-1] and mask[:, -short_seq_len:-1] with S = short_seq_len - 1:
    the embeddings of positions [L - S, L) and the mask of positions [L - S - 1, L - 1), one apart as in the reference."""
    L = mask_u8.shape[1]
    return x[:, L - S:L], mask_u8[:, L - S - 1:L - 1].contiguous()


class _EtaInterest(torch.autograd.Function):
    """ETA.forward's interest block (ETA.py:150-165) over item_feat_emb x (B, L + 1, d) as one node: the short target
    attention over the window, SimHash retrieval of the k = min(topk, L) nearest history rows (b2_eta_retrieve_fwd),
    the long target attention over them.  Returns (target, short interest, long interest), each (B, d).  The backward
    runs both attentions' backwards and one assembly launch (b2_eta_assemble_bwd) that writes dx once."""

    @staticmethod
    def forward(ctx, x, mask_u8, R, r_stride, S, k, heads, use_scale, *weights):
        x = _f32c(x)
        B, L1, d = x.shape
        L = L1 - 1
        ws, wl = weights[:4], weights[4:]
        target = x[:, L].contiguous()
        hs, ms = _short_window(x, mask_u8, S)
        short, sctx = _mhta_fwd(target, hs, ms, heads, _mhta_scale(ws, d, heads, use_scale), ws)
        bits = R.shape[-1]
        topk_emb = torch.empty((B, k, d), dtype=torch.float32, device=x.device)
        topk_mask = torch.empty((B, k), dtype=torch.uint8, device=x.device)
        pos = torch.empty((B, k), dtype=torch.int32, device=x.device)
        _lib.call("b2_eta_retrieve_fwd", _ptr(x), _ptr(mask_u8), _ptr(R), r_stride, B, L, d, bits, k, _ptr(topk_emb),
                  _ptr(topk_mask), _ptr(pos), _stream())
        long, lctx = _mhta_fwd(target, topk_emb, topk_mask, heads, _mhta_scale(wl, d, heads, use_scale), wl)
        ctx.parts = (sctx, lctx, S, k, pos, L)
        ctx.mark_non_differentiable(pos)
        return target, short, long, pos

    @staticmethod
    def backward(ctx, g_target, g_short, g_long, _):
        sctx, lctx, S, k, pos, L = ctx.parts
        dt_s, dx_s, dws = _mhta_bwd(sctx, _f32c(g_short))
        dt_l, dx_l, dwl = _mhta_bwd(lctx, _f32c(g_long))
        B, d = dt_s.shape
        g_target = _f32c(g_target)
        dx = torch.empty((B, L + 1, d), dtype=torch.float32, device=dt_s.device)
        _lib.call("b2_eta_assemble_bwd", _ptr(g_target), _ptr(dt_s), _ptr(dt_l), _ptr(dx_s), S, _ptr(dx_l),
                  _ptr(pos), B, L, d, k, _ptr(dx), _stream())
        return (dx, None, None, None, None, None, None, None) + dws + dwl


class _SdimInterest(torch.autograd.Function):
    """SDIM.forward's interest block (SDIM.py:155-167) over item_feat_emb x (B, L + 1, d) as one node: the short target
    attention over the window and the hash-collision pooling of the history (b2_sdim_pool_fwd).  Returns (target,
    short interest, long interest), each (B, d).  The backward runs the attention's backward and one assembly launch
    (b2_sdim_assemble_bwd) that writes dx once."""

    @staticmethod
    def forward(ctx, x, mask_u8, R, r_stride, S, l2_norm, heads, use_scale, *weights):
        x = _f32c(x)
        B, L1, d = x.shape
        L = L1 - 1
        target = x[:, L].contiguous()
        hs, ms = _short_window(x, mask_u8, S)
        short, sctx = _mhta_fwd(target, hs, ms, heads, _mhta_scale(weights, d, heads, use_scale), weights)
        nh, bits = R.shape[-2], R.shape[-1]
        long = torch.empty((B, d), dtype=torch.float32, device=x.device)
        sums = torch.empty((B, nh, d), dtype=torch.float32, device=x.device)
        collide = torch.empty((B, L), dtype=torch.int32, device=x.device)
        _lib.call("b2_sdim_pool_fwd", _ptr(x), _ptr(mask_u8), _ptr(R), r_stride, B, L, d, nh, bits, int(l2_norm),
                  _ptr(long), _ptr(sums), _ptr(collide), _stream())
        ctx.parts = (sctx, S, l2_norm, sums, collide, L)
        return target, short, long

    @staticmethod
    def backward(ctx, g_target, g_short, g_long):
        sctx, S, l2_norm, sums, collide, L = ctx.parts
        dt_s, dx_s, dws = _mhta_bwd(sctx, _f32c(g_short))
        B, d = dt_s.shape
        # both held until the launch: a temporary freed inside the argument list would hand its block to the next one
        g_target, g_long = _f32c(g_target), _f32c(g_long)
        zero = torch.zeros((B, d), dtype=torch.float32, device=dt_s.device)
        dx = torch.empty((B, L + 1, d), dtype=torch.float32, device=dt_s.device)
        _lib.call("b2_sdim_assemble_bwd", _ptr(g_target), _ptr(dt_s), _ptr(zero), _ptr(dx_s), S, _ptr(g_long),
                  _ptr(sums), _ptr(collide), B, L, d, sums.shape[1], int(l2_norm), _ptr(dx), _stream())
        return (dx, None, None, None, None, None, None, None) + dws


def _lsh_inputs(name, item_emb, mask, R, hash_dims, short_seq_len):
    _require_cuda(R)
    mask_u8, B, L, d = _longctr_inputs(name, item_emb, mask, short_seq_len)
    if R.dim() != 2 + hash_dims or R.shape[0] not in (1, B) or R.shape[1] != d:
        raise ValueError("%s: rotations%s must be (1 or B, d, ...) with d = %d" % (name, tuple(R.shape), d))
    R = _f32c(R)
    r_stride = 0 if R.shape[0] == 1 else R[0].numel()
    return mask_u8, R, r_stride, B, L, d


def _longctr_inputs(name, item_emb, mask, short_seq_len):
    """(mask bytes, B, L, d) of a LongCTR interest block's item_feat_emb (B, L + 1, d) and mask (B, L)."""
    _require_cuda(item_emb, mask)
    if item_emb.dim() != 3 or mask.dim() != 2 or mask.shape[0] != item_emb.shape[0] \
            or item_emb.shape[1] != mask.shape[1] + 1:
        raise ValueError("%s: item_feat_emb%s must be (B, L + 1, d) and mask%s (B, L)"
                         % (name, tuple(item_emb.shape), tuple(mask.shape)))
    B, L1, d = item_emb.shape
    L = L1 - 1
    if L == 0:
        raise ValueError("%s: the batch has an empty history axis (L = 0)" % name)
    if short_seq_len < 2:
        raise ValueError("%s: short_seq_len must be at least 2 (the window [-short_seq_len:-1] would be empty), got %d"
                         % (name, short_seq_len))
    if L < short_seq_len:
        raise ValueError("%s: the history length L = %d is below short_seq_len = %d, where the reference's "
                         "[-short_seq_len:-1] windows of the embeddings and of the mask differ in length"
                         % (name, L, short_seq_len))
    return torch.ne(mask, 0).view(torch.uint8), B, L, d


def eta_interest(item_emb, mask, rotations, short_seq_len, topk, num_heads, use_scale, short_weights, long_weights):
    """ETA's interest block: item_emb (B, L + 1, d) (the last position the target), mask (B, L) (non-zero = valid),
    rotations (1 or B, d, hash_bits), short_weights and long_weights the (W_q, W_k, W_v, W_o) of the two attentions.
    Returns (target, short interest, long interest, positions): three (B, d) and the chosen history positions (B, k)
    int32, k = min(topk, L), sorted by (Hamming distance, position).  Ties at equal distance go to the lower position."""
    mask_u8, R, r_stride, B, L, d = _lsh_inputs("ETA", item_emb, mask, rotations, 1, short_seq_len)
    bound = eta_bound(d, L, topk, R.shape[-1], B)
    if bound is not None:
        raise NotImplementedError("ETA kernels: " + bound)
    for w in tuple(short_weights) + tuple(long_weights):
        _require_cuda(w)
    return _EtaInterest.apply(item_emb, mask_u8, R, r_stride, short_seq_len - 1, min(topk, L), num_heads, use_scale,
                              *short_weights, *long_weights)


def sdim_interest(item_emb, mask, rotations, short_seq_len, l2_norm, num_heads, use_scale, short_weights):
    """SDIM's interest block: item_emb (B, L + 1, d) (the last position the target), mask (B, L) (non-zero = valid),
    rotations (1 or B, d, num_hashes, hash_bits), short_weights (W_q, W_k, W_v, W_o) of the short attention or () for
    use_qkvo=False.  Returns (target, short interest, long interest), each (B, d)."""
    mask_u8, R, r_stride, B, L, d = _lsh_inputs("SDIM", item_emb, mask, rotations, 2, short_seq_len)
    bound = sdim_bound(d, L, R.shape[-2], R.shape[-1], B)
    if bound is not None:
        raise NotImplementedError("SDIM kernels: " + bound)
    for w in short_weights:
        _require_cuda(w)
    return _SdimInterest.apply(item_emb, mask_u8, R, r_stride, short_seq_len - 1, bool(l2_norm), num_heads, use_scale,
                               *short_weights)


# --------------------------------------------------------------------------------------
# LongCTR interest block: MIRRN's three SimHash retrievals and FilterLayer2 blocks
# --------------------------------------------------------------------------------------
MIRRN_FILTER_DROPOUT = 0.1      # FilterLayer2's out_dropout, hard-coded in MIRRN.__init__
MIRRN_LN_EPS = 1e-12            # FilterLayer2's TF-style LayerNorm


def mirrn_bound(d, L, topk, hash_bits, batch=1):
    """None when the MIRRN kernels cover item width d, history length L, topk and hash_bits, else the bound it
    breaks."""
    msg = _lsh_common_bound(batch, d, L)
    if msg is not None:
        return msg
    if d % 4:
        return "the item width d (item_info_dim) must be a multiple of 4 (FilterLayer2's four blocks), got %d" % d
    if not 1 <= hash_bits <= _lib.B2_MIRRN_MAX_BITS:
        return "hash_bits must lie in [1, %d], got %d" % (_lib.B2_MIRRN_MAX_BITS, hash_bits)
    if not 1 <= topk <= _lib.B2_LSH_MAX_TOPK:
        return "topk must lie in [1, %d], got %d" % (_lib.B2_LSH_MAX_TOPK, topk)
    k = min(topk, L)
    G = 256 // d
    retrieve = 4 * 3 * d * hash_bits + 8 * G * d + 8 * d + 12 * (hash_bits + 2) + 24 + 3 * L
    if retrieve > _lib.B2_LSH_MAX_SMEM:
        return "d hash_bits = %d needs more shared memory than a CTA has" % (d * hash_bits)
    if 8 * k * d + 8 * k + 8 * G * d > _lib.B2_LSH_MAX_SMEM:
        return "k d = %d needs more shared memory than a CTA has" % (k * d)
    return None


def mirrn_filter_table(k):
    """First column h (k,) float64 of FilterLayer2's circulant at FFT length k: irfft(rfft(u) (a + i b), n=k, ortho)
    = a u + b (H u) with (H u)_t = sum_s h[(t - s) mod k] u_s and h[m] = -(2 / k) sum_{f=1}^{ceil(k/2)-1}
    sin(2 pi f m / k).  The DC and Nyquist bins drop out of the sum because irfft ignores their imaginary parts."""
    m = torch.arange(k, dtype=torch.float64)
    h = torch.zeros(k, dtype=torch.float64)
    for f in range(1, (k + 1) // 2):
        h -= torch.sin(2 * math.pi * f * m / k)
    return h * (2.0 / k)


_MIRRN_TABLES = {}


def _mirrn_table(k, dev):
    key = (k, str(dev))
    h = _MIRRN_TABLES.get(key)
    if h is None:
        h = _MIRRN_TABLES[key] = mirrn_filter_table(k).float().to(dev)
    return h


class _MirrnInterest(torch.autograd.Function):
    """MIRRN.forward's interest block (MIRRN.py:149-196) over item_feat_emb x (B, L + 1, d) as one node: the short
    target attention over the window; three SimHash retrievals (b2_mirrn_retrieve_fwd); per retrieval the gathered
    rows plus 0.02 pos[L - idx] through FilterLayer2 (b2_mirrn_filter_fwd, then b2_bst_addnorm_fwd with eps 1e-12 and
    the Philox dropout), their mean over the k slots (b2_mirrn_mean_fwd); the long target attention over the three
    interests, unmasked.  Returns (target, short interest, long interest, positions (B, 3, k)).  The backward runs the
    attentions', add-norms' and filters' backwards and one assembly launch (b2_mirrn_assemble_bwd) that writes dx
    once."""

    @staticmethod
    def forward(ctx, x, mask_u8, R, r_stride, cfg, pos_table, *params):
        S, k, heads, use_scale, drop = cfg
        x = _f32c(x)
        B, L1, d = x.shape
        L = L1 - 1
        dev = x.device
        ctx.empty = B == 0
        if B == 0:                  # nothing to launch; every gradient is empty or zero
            ctx.shape = (L, d)
            empty = torch.empty((0, d), dtype=torch.float32, device=dev)
            pos = torch.empty((0, 3, k), dtype=torch.int32, device=dev)
            ctx.mark_non_differentiable(pos)
            return empty, empty.clone(), empty.clone(), pos
        ws, wl = params[:4], params[4:8]
        cws, gammas, betas = params[8:11], params[11:14], params[14:17]
        target = x[:, L].contiguous()
        hs, ms = _short_window(x, mask_u8, S)
        short, sctx = _mhta_fwd(target, hs, ms, heads, _mhta_scale(ws, d, heads, use_scale), ws)
        pos = torch.empty((B, 3, k), dtype=torch.int32, device=dev)
        _lib.call("b2_mirrn_retrieve_fwd", _ptr(x), _ptr(mask_u8), _ptr(R), r_stride, B, L, d, R.shape[-1], k,
                  _ptr(pos), _stream())
        htab = _mirrn_table(k, dev)
        pos_table = _f32c(pos_table)
        cws = tuple(_f32c(w) for w in cws)
        u = torch.empty((3, B * k, d), dtype=torch.float32, device=dev)
        y = torch.empty_like(u)
        _lib.call("b2_mirrn_filter_fwd", _ptr(x), _ptr(pos), _ptr(pos_table), pos_table.shape[0], *map(_ptr, cws),
                  _ptr(htab), B, L, d, k, _ptr(u), _ptr(y), _stream())
        z = torch.empty_like(u)
        mean = torch.empty((3, B * k), dtype=torch.float32, device=dev)
        rstd = torch.empty_like(mean)
        for q in range(3):
            _lib.call("b2_bst_addnorm_fwd", _ptr(y[q]), _ptr(u[q]), B * k, d, _ptr(gammas[q]), _ptr(betas[q]),
                      MIRRN_LN_EPS, *_drop_args(drop[q]), _ptr(z[q]), *_aux_args(None), _ptr(mean[q]), _ptr(rstd[q]),
                      _stream())
        interests = torch.empty((B, 3, d), dtype=torch.float32, device=dev)
        _lib.call("b2_mirrn_mean_fwd", _ptr(z), B, d, k, _ptr(interests), _stream())
        long, lctx = _mhta_fwd(target, interests, None, heads, _mhta_scale(wl, d, heads, use_scale), wl)
        ctx.parts = (sctx, lctx, S, k, L, pos, u, y, mean, rstd, htab, drop, pos_table)
        ctx.params = (cws, gammas, betas)
        ctx.leaves = (params[8:11], pos_table)
        ctx.mark_non_differentiable(pos)
        return target, short, long, pos

    @staticmethod
    def backward(ctx, g_target, g_short, g_long, _):
        if ctx.empty:
            L, d = ctx.shape
            dx = torch.zeros((0, L + 1, d), dtype=torch.float32, device=g_target.device)
            return (dx,) + (None,) * 22
        sctx, lctx, S, k, L, pos, u, y, mean, rstd, htab, drop, pos_table = ctx.parts
        cws, gammas, betas = ctx.params
        dt_s, dx_s, dws = _mhta_bwd(sctx, _f32c(g_short))
        dt_l, dint, dwl = _mhta_bwd(lctx, _f32c(g_long))
        B, d = dt_s.shape
        dev = dt_s.device
        dz = torch.empty((3, B * k, d), dtype=torch.float32, device=dev)
        _lib.call("b2_mirrn_mean_bwd", _ptr(dint), B, d, k, _ptr(dz), _stream())
        dgam = [_grad_buffer(p, zero=True) for p in gammas]
        dbet = [_grad_buffer(p, zero=True) for p in betas]
        dy = torch.empty_like(dz)
        dropping = any(dq is not None for dq in drop)
        dres = torch.empty_like(dz) if dropping else dy     # without dropout the residual's gradient is dy itself
        for q in range(3):
            _lib.call("b2_bst_addnorm_bwd", _ptr(y[q]), _ptr(u[q]), _ptr(dz[q]), None, B * k, d, _ptr(gammas[q]),
                      _ptr(mean[q]), _ptr(rstd[q]), *_drop_args(drop[q]), _ptr(dy[q]), *_aux_args(None),
                      _ptr(dres[q] if dropping else None), _ptr(dgam[q]), _ptr(dbet[q]), _stream())
        dcw = [_grad_buffer(p, zero=True) for p in ctx.leaves[0]]
        dpos = _grad_buffer(ctx.leaves[1], zero=True)
        du = torch.empty_like(dz)
        _lib.call("b2_mirrn_filter_bwd", _ptr(dy), _ptr(dres), _ptr(u), _ptr(pos), pos_table.shape[0],
                  *map(_ptr, cws), _ptr(htab), B, L, d, k, _ptr(du), *map(_ptr, dcw), _ptr(dpos), _stream())
        g_target = _f32c(g_target)
        dx = torch.empty((B, L + 1, d), dtype=torch.float32, device=dev)
        _lib.call("b2_mirrn_assemble_bwd", _ptr(g_target), _ptr(dt_s), _ptr(dt_l), _ptr(dx_s), S, _ptr(du),
                  _ptr(pos), B, L, d, k, _ptr(dx), _stream())
        return (dx, None, None, None, None, dpos) + dws + dwl + tuple(dcw) + tuple(dgam) + tuple(dbet)


def mirrn_interest(item_emb, mask, rotations, short_seq_len, topk, num_heads, use_scale, short_weights, long_weights,
                   pos_table, complex_weights, ln_weights, ln_biases, dropout=0.0):
    """MIRRN's interest block: item_emb (B, L + 1, d) (the last position the target), mask (B, L) (non-zero = valid),
    rotations (d, hash_bits) shared by the three retrievals or (3, d, hash_bits) one set per retrieval (target, short,
    global); short_weights and long_weights the (W_q, W_k, W_v, W_o) of the two attentions; pos_table (max_len + 1, d)
    the position embedding; complex_weights, ln_weights, ln_biases the three FilterLayer2 blocks' complex_weight
    (4, d / 4, d / 4, 2) and LayerNorm weight and bias (d).  dropout: the blocks' out_dropout probability, one for
    all three or one per block (0: none), drawn from the Philox masks (block q at layer q of one snapshot).  Returns
    (target, short interest, long interest, positions): three (B, d) and the retrieved history positions (B, 3, k)
    int32, k = min(topk, L), each row in ascending position order.  Ties at equal distance go to the lower
    position."""
    _require_cuda(rotations, pos_table)
    mask_u8, B, L, d = _longctr_inputs("MIRRN", item_emb, mask, short_seq_len)
    R = rotations
    if R.dim() == 2:
        R3 = R.unsqueeze(0)
    elif R.dim() == 3 and R.shape[0] == 3:
        R3 = R
    else:
        R3 = None
    if R3 is None or R3.shape[1] != d:
        raise ValueError("MIRRN: rotations%s must be (d, hash_bits) or (3, d, hash_bits) with d = %d"
                         % (tuple(R.shape), d))
    R3 = _f32c(R3)
    r_stride = 0 if R.dim() == 2 else R3[0].numel()
    bound = mirrn_bound(d, L, topk, R3.shape[-1], B)
    if bound is not None:
        raise NotImplementedError("MIRRN kernels: " + bound)
    if pos_table.dim() != 2 or pos_table.shape[1] != d:
        raise ValueError("MIRRN: pos_table%s must be (max_len + 1, %d)" % (tuple(pos_table.shape), d))
    if L >= pos_table.shape[0]:
        raise ValueError("MIRRN: the history length L = %d exceeds max_len = %d (the position embedding has rows "
                         "0 .. max_len and the reference indexes row L - idx)" % (L, pos_table.shape[0] - 1))
    filt = tuple(complex_weights) + tuple(ln_weights) + tuple(ln_biases)
    if len(filt) != 9 or any(tuple(w.shape) != (4, d // 4, d // 4, 2) for w in complex_weights) \
            or any(w.numel() != d for w in tuple(ln_weights) + tuple(ln_biases)):
        raise ValueError("MIRRN: three complex_weight (4, d / 4, d / 4, 2) and three LayerNorm weights and biases (d) "
                         "are needed, d = %d" % d)
    for w in tuple(short_weights) + tuple(long_weights) + filt:
        _require_cuda(w)
    ps = [float(p) for p in dropout] if isinstance(dropout, (list, tuple)) else [float(dropout)] * 3
    if len(ps) != 3:
        raise ValueError("MIRRN: dropout must be one probability or one per filter block (3), got %d" % len(ps))
    drop = [None] * 3
    if any(p > 0 for p in ps):
        snap = dropout_snapshot(item_emb.device, 3)
        drop = [(snap, q) + dropout_consts(p) if p > 0 else None for q, p in enumerate(ps)]
    cfg = (short_seq_len - 1, min(topk, L), num_heads, use_scale, drop)
    return _MirrnInterest.apply(item_emb, mask_u8, R3, r_stride, cfg, pos_table, *short_weights, *long_weights, *filt)


# --------------------------------------------------------------------------------------
# LongCTR interest blocks: SIM's soft-search retrieval and TWIN's top-k attention
# --------------------------------------------------------------------------------------
def _topk_common_bound(batch, d, L, topk):
    if not 1 <= d <= _lib.B2_TOPK_MAX_DIM:
        return "the item width d (item_info_dim) must lie in [1, %d], got %d" % (_lib.B2_TOPK_MAX_DIM, d)
    if not 1 <= L <= _lib.B2_TOPK_MAX_LEN:
        return "the history length L must lie in [1, %d], got %d" % (_lib.B2_TOPK_MAX_LEN, L)
    if not 1 <= topk <= _lib.B2_TOPK_MAX_K:
        return "topk must lie in [1, %d], got %d" % (_lib.B2_TOPK_MAX_K, topk)
    if batch * (L + 1) >= 2 ** 31:
        return "batch (L + 1) must stay below 2^31, got %d" % (batch * (L + 1))
    return None


def _heads_bound(d, num_heads):
    if not 1 <= num_heads <= _lib.B2_MHTA_MAX_HEADS or num_heads * d > _lib.B2_MHTA_MAX_WIDTH:
        return "num_heads must lie in [1, %d] with num_heads d <= %d, got num_heads %d, d %d" \
            % (_lib.B2_MHTA_MAX_HEADS, _lib.B2_MHTA_MAX_WIDTH, num_heads, d)
    return None


def _part_bytes(d):
    return 4 * (256 // d) * d


def sim_bound(d, L, topk, num_heads, batch=1):
    """None when the SIM kernels cover item width d, history length L, topk and num_heads, else the bound it breaks."""
    msg = _topk_common_bound(batch, d, L, topk) or _heads_bound(d, num_heads)
    if msg is not None:
        return msg
    k = min(topk, L)
    if 8 * L + 4 * d + _part_bytes(d) + 4 * k > _lib.B2_TOPK_MAX_SMEM:
        return "L = %d needs more shared memory than a CTA has" % L
    return None


def twin_bound(d, L, topk, num_heads, batch=1):
    """None when the TWIN kernels cover item width d, history length L, topk and num_heads, else the bound it breaks."""
    msg = _topk_common_bound(batch, d, L, topk) or _heads_bound(d, num_heads)
    if msg is not None:
        return msg
    k, H = min(topk, L), num_heads
    fwd = 4 * L + 4 * d + 8 * k + _part_bytes(d)
    bwd = 4 * ((H * L + 1) // 2) + 12 * H * d + 12 * H * k + 4 * H
    if max(fwd, bwd) > _lib.B2_TOPK_MAX_SMEM:
        return "num_heads L = %d needs more shared memory than a CTA has" % (H * L)
    return None


class _SimInterest(torch.autograd.Function):
    """SIM.forward's interest block (SIM.py:128-153) over item_feat_emb x (B, L + 1, d) as one node: the short target
    attention over the window; the soft-search GSU, u = W_b^T W_a t on two fp32 GEMMs, then the scores
    qk_l = (u . x_l) mask_l, pooled = sum_l qk_l x_l and the k = min(topk, L) best rows (b2_sim_retrieve_fwd); the long
    target attention over them.  Returns (target, short, long, pooled, positions).  The backward runs both attentions'
    backwards, the GSU's (b2_sim_gsu_bwd, then the fp32 GEMMs back to dW_a, dW_b and dt) and one assembly launch
    (b2_sim_assemble_bwd) that writes dx once."""

    @staticmethod
    def forward(ctx, x, mask_u8, S, k, heads, use_scale, Wa, Wb, *weights):
        x = _f32c(x)
        B, L1, d = x.shape
        L, dev = L1 - 1, x.device
        ws, wl = weights[:4], weights[4:]
        target = x[:, L].contiguous()
        hs, ms = _short_window(x, mask_u8, S)
        short, sctx = _mhta_fwd(target, hs, ms, heads, _mhta_scale(ws, d, heads, use_scale), ws)
        # the scores decide the selection, so they are fp32 in every matmul mode
        Wa, Wb = _f32c(Wa), _f32c(Wb)
        a = gemm_f32(target, Wa, torch.empty((B, Wa.shape[0]), dtype=torch.float32, device=dev), b_t=True)
        u = gemm_f32(a, Wb, torch.empty((B, d), dtype=torch.float32, device=dev))
        qk = torch.empty((B, L), dtype=torch.float32, device=dev)
        pooled = torch.empty((B, d), dtype=torch.float32, device=dev)
        topk_emb = torch.empty((B, k, d), dtype=torch.float32, device=dev)
        topk_mask = torch.empty((B, k), dtype=torch.uint8, device=dev)
        pos = torch.empty((B, k), dtype=torch.int32, device=dev)
        _lib.call("b2_sim_retrieve_fwd", _ptr(x), _ptr(mask_u8), _ptr(u), B, L, d, k, _ptr(qk), _ptr(pooled),
                  _ptr(topk_emb), _ptr(topk_mask), _ptr(pos), _stream())
        long, lctx = _mhta_fwd(target, topk_emb, topk_mask, heads, _mhta_scale(wl, d, heads, use_scale), wl)
        ctx.parts = (sctx, lctx, S, k, L, x, mask_u8, target, a, u, qk, pos, Wa, Wb)
        ctx.mark_non_differentiable(pos)
        return target, short, long, pooled, pos

    @staticmethod
    def backward(ctx, g_target, g_short, g_long, g_pooled, _):
        sctx, lctx, S, k, L, x, mask_u8, target, a, u, qk, pos, Wa, Wb = ctx.parts
        dt_s, dx_s, dws = _mhta_bwd(sctx, _f32c(g_short))
        dt_l, dx_l, dwl = _mhta_bwd(lctx, _f32c(g_long))
        B, d = dt_s.shape
        dev = x.device
        g_target, g_pooled = _f32c(g_target), _f32c(g_pooled)
        dqk = torch.empty((B, L), dtype=torch.float32, device=dev)
        du = torch.empty((B, d), dtype=torch.float32, device=dev)
        _lib.call("b2_sim_gsu_bwd", _ptr(x), _ptr(mask_u8), _ptr(g_pooled), B, L, d, _ptr(dqk), _ptr(du), _stream())
        da = gemm_f32(du, Wb, torch.empty_like(a), b_t=True)                   # da = du W_b^T
        dWb = gemm_f32(a, du, torch.empty_like(Wb), a_t=True)                  # dW_b = a^T du
        dt_g = gemm_f32(da, Wa, torch.empty_like(target))                      # dt = da W_a
        dWa = gemm_f32(da, target, torch.empty_like(Wa), a_t=True)             # dW_a = da^T t
        dx = torch.empty((B, L + 1, d), dtype=torch.float32, device=dev)
        _lib.call("b2_sim_assemble_bwd", _ptr(g_target), _ptr(dt_s), _ptr(dt_l), _ptr(dt_g), _ptr(dx_s), S,
                  _ptr(dx_l), _ptr(pos), _ptr(qk), _ptr(dqk), _ptr(u), _ptr(g_pooled), B, L, d, k, _ptr(dx),
                  _stream())
        return (dx, None, None, None, None, None, dWa, dWb) + dws + dwl


class _TwinInterest(torch.autograd.Function):
    """TWIN.forward's interest block (TWIN.py:125-141 with MultiHeadTopKAttention, TWIN.py:243-293) over item_feat_emb
    x (B, L + 1, d) as one node: the short target attention over the window, then the top-k attention over the whole
    history.  W_q, W_h, W_v, W_o fold as MultiHeadTargetAttention's do (b2_mhta_pack, scale 1 / sqrt(head_dim)), so
    the history is never projected: q' = t W_M^T (fp32 in every matmul mode: the scores decide the selection), the row
    kernel's per-head selection, softmax and pooled p (b2_twin_topk_fwd), out = p W_N^T (the matmul mode's GEMM).
    Returns (target, short, long, positions (B, heads, k)).  The backward's row kernel (b2_twin_topk_bwd) writes dq'
    and all of dx, the target row's dq' W_M included."""

    @staticmethod
    def forward(ctx, x, mask_u8, S, k, heads, use_scale, *weights):
        x = _f32c(x)
        B, L1, d = x.shape
        L, H, dev = L1 - 1, heads, x.device
        ws = weights[:4]
        Wq, Wh, Wv, Wo = (_f32c(w) for w in weights[4:])
        target = x[:, L].contiguous()
        hs, ms = _short_window(x, mask_u8, S)
        short, sctx = _mhta_fwd(target, hs, ms, heads, _mhta_scale(ws, d, heads, use_scale), ws)
        hd = Wq.shape[0] // H
        scale = 1.0 / hd ** 0.5
        WM = torch.empty((H * d, d), dtype=torch.float32, device=dev)
        WN = torch.empty((d, H * d), dtype=torch.float32, device=dev)
        _lib.call("b2_mhta_pack", _ptr(Wq), _ptr(Wh), _ptr(Wv), _ptr(Wo), d, H, hd, scale, _ptr(WM), _ptr(WN),
                  _stream())
        q = gemm_f32(target, WM, torch.empty((B, H * d), dtype=torch.float32, device=dev), b_t=True)
        p = torch.empty((B, H * d), dtype=torch.float32, device=dev)
        stats = torch.empty((B, H, 2), dtype=torch.float32, device=dev)
        pos = torch.empty((B, H, k), dtype=torch.int32, device=dev)
        _lib.call("b2_twin_topk_fwd", _ptr(q), _ptr(x), _ptr(mask_u8), B, L, d, H, k, _ptr(p), _ptr(stats), _ptr(pos),
                  _stream())
        tc = _tc_layer_ok(WN)
        p_aux, wn_aux = (make_aux(p), make_aux(WN)) if tc else (None, None)
        long = _linear_fwd(tc, p, p_aux, WN, torch.empty((B, d), dtype=torch.float32, device=dev), wn_aux)
        ctx.parts = (sctx, S, k, H, hd, scale, x, mask_u8, target, q, p, stats, pos, WM, WN, tc, p_aux, wn_aux,
                     (Wq, Wh, Wv, Wo))
        ctx.mark_non_differentiable(pos)
        return target, short, long, pos

    @staticmethod
    def backward(ctx, g_target, g_short, g_long, _):
        (sctx, S, k, H, hd, scale, x, mask_u8, target, q, p, stats, pos, WM, WN, tc, p_aux, wn_aux,
         (Wq, Wh, Wv, Wo)) = ctx.parts
        dt_s, dx_s, dws = _mhta_bwd(sctx, _f32c(g_short))
        B, L1, d = x.shape
        dev = x.device
        g, g_target = _f32c(g_long), _f32c(g_target)
        g_aux = make_aux(g) if tc else None
        dp = torch.empty((B, H * d), dtype=torch.float32, device=dev)
        dWN = torch.empty((d, H * d), dtype=torch.float32, device=dev)
        _linear_dgrad(tc, g, g_aux, WN, dp, wn_aux)                           # dp = g W_N
        _linear_wgrad(tc, g, g_aux, p, p_aux, dWN)                           # dW_N = g^T p
        dq = torch.empty((B, H * d), dtype=torch.float32, device=dev)
        dx = torch.empty_like(x)
        _lib.call("b2_twin_topk_bwd", _ptr(q), _ptr(x), _ptr(mask_u8), _ptr(p), _ptr(stats), _ptr(pos), _ptr(dp),
                  _ptr(WM), _ptr(g_target), _ptr(dt_s), _ptr(dx_s), S, B, L1 - 1, d, H, k, _ptr(dq), _ptr(dx),
                  _stream())
        dWM = gemm_f32(dq, target, torch.empty_like(WM), a_t=True)             # dW_M = dq'^T t
        gWq, gWh, gWv, gWo = (torch.empty_like(w) for w in (Wq, Wh, Wv, Wo))
        _lib.call("b2_mhta_unpack", _ptr(Wq), _ptr(Wh), _ptr(Wv), _ptr(Wo), _ptr(dWM), _ptr(dWN), d, H, hd, scale,
                  _ptr(gWq), _ptr(gWh), _ptr(gWv), _ptr(gWo), _stream())
        return (dx, None, None, None, None, None) + dws + (gWq, gWh, gWv, gWo)


def _topk_weights(name, weights, d, heads):
    for w in weights:
        _require_cuda(w)
    A = weights[0].shape[0]
    if A % heads or any(tuple(w.shape) != (A, d) for w in weights[:-1]) or tuple(weights[-1].shape) != (d, A):
        raise ValueError("%s: attention_dim %d, num_heads %d and the weights do not match" % (name, A, heads))


def sim_interest(item_emb, mask, short_seq_len, topk, num_heads, W_a, W_b, short_weights, long_weights):
    """SIM's interest block: item_emb (B, L + 1, d) (the last position the target), mask (B, L) (non-zero = valid),
    W_a, W_b (A, d) the GSU's Linears, short_weights and long_weights the (W_q, W_k, W_v, W_o) of the two attentions
    (use_scale on, as SIM builds them).  Returns (target, short interest, long interest, pooled, positions): four
    (B, d) and the chosen history positions (B, k) int32, k = min(topk, L), sorted by (score desc, position asc).
    Masked positions score 0, as in the reference; ties go to the lower position, and -0.0 ties with +0.0."""
    mask_u8, B, L, d = _longctr_inputs("SIM", item_emb, mask, short_seq_len)
    bound = sim_bound(d, L, topk, num_heads, B)
    if bound is not None:
        raise NotImplementedError("SIM kernels: " + bound)
    _topk_weights("SIM", tuple(short_weights), d, num_heads)
    _topk_weights("SIM", tuple(long_weights), d, num_heads)
    _require_cuda(W_a, W_b)
    if W_a.dim() != 2 or tuple(W_b.shape) != tuple(W_a.shape) or W_a.shape[1] != d:
        raise ValueError("SIM: W_a%s and W_b%s must both be (attention_dim, d = %d)"
                         % (tuple(W_a.shape), tuple(W_b.shape), d))
    return _SimInterest.apply(item_emb, mask_u8, short_seq_len - 1, min(topk, L), num_heads, True, W_a, W_b,
                              *short_weights, *long_weights)


def twin_interest(item_emb, mask, short_seq_len, topk, num_heads, short_weights, topk_weights):
    """TWIN's interest block: item_emb (B, L + 1, d) (the last position the target), mask (B, L) (non-zero = valid),
    short_weights the (W_q, W_k, W_v, W_o) of the short attention, topk_weights the (W_q, W_h, W_v, W_o) of
    MultiHeadTopKAttention.  Returns (target, short interest, long interest, positions): three (B, d) and the chosen
    history positions (B, num_heads, k) int32, k = min(topk, L), per head sorted by (score desc, position asc).  A
    masked score is exactly -1e9, so masked rows tie and go to the lower positions."""
    mask_u8, B, L, d = _longctr_inputs("TWIN", item_emb, mask, short_seq_len)
    bound = twin_bound(d, L, topk, num_heads, B)
    if bound is not None:
        raise NotImplementedError("TWIN kernels: " + bound)
    _topk_weights("TWIN", tuple(short_weights), d, num_heads)
    _topk_weights("TWIN", tuple(topk_weights), d, num_heads)
    return _TwinInterest.apply(item_emb, mask_u8, short_seq_len - 1, min(topk, L), num_heads, True, *short_weights,
                               *topk_weights)


def mlp_chain_supported():
    return _MATMUL["mode"] != "fp32"


def mlp_chain(x, layers):
    """layers: list of (weight, bias or None, act code[, dropout p]).  Returns h_L with
    h_{i+1} = dropout_{p_i}(act_i(h_i W_i^T + b_i)), h_0 = x; p = 0 (or absent) is no dropout, else 0 < p < 1
    (training-mode nn.Dropout: a fresh mask every forward, see dropout_state)."""
    _require_cuda(x)
    acts = tuple(layer[2] for layer in layers)
    drops = tuple(float(layer[3]) if len(layer) > 3 and layer[3] else 0.0 for layer in layers)
    for p in drops:
        if p:
            dropout_consts(p)           # raises outside (0, 1)
    drops = drops if any(drops) else None
    flat = []
    for layer in layers:
        w, b = layer[0], layer[1]
        _require_cuda(w, b)
        flat += [w, b]
    if x.dim() != 2:
        lead = x.shape[:-1]
        return _MLPChain.apply(x.reshape(-1, x.shape[-1]), acts, drops, *flat).view(*lead, -1)
    return _MLPChain.apply(x, acts, drops, *flat)


def linear_act(x, weight, bias=None, act=B2_ACT_NONE):
    _require_cuda(x, weight, bias)
    if x.dim() != 2:
        lead = x.shape[:-1]
        return _LinearAct.apply(x.reshape(-1, x.shape[-1]), weight, bias, act).view(*lead, -1)
    return _LinearAct.apply(x, weight, bias, act)


# --------------------------------------------------------------------------------------
# Fused logit + sigmoid + BCE(mean)
# --------------------------------------------------------------------------------------
class _LogitBCE(torch.autograd.Function):
    """loss = BCE(sigmoid(sum(terms)), y).mean(); also returns y_pred (not differentiable)."""

    @staticmethod
    def forward(ctx, label, *terms):
        ctx.shapes = [t.shape for t in terms]
        terms = [_f32c(t).view(-1) for t in terms]
        B = terms[0].numel()
        dev = terms[0].device
        label = _f32c(label).view(-1)
        y_pred = torch.empty((B, 1), dtype=torch.float32, device=dev)
        loss = torch.empty((), dtype=torch.float32, device=dev)
        glogit = torch.empty((B,), dtype=torch.float32, device=dev)
        ptrs = [_ptr(t) for t in terms] + [ctypes.c_void_p(0)] * (4 - len(terms))
        _lib.call("b2_logit_bce_fwd", ptrs[0], ptrs[1], ptrs[2], ptrs[3], _ptr(label), B,
                  _ptr(y_pred), _ptr(loss), _ptr(glogit), _stream())
        ctx.save_for_backward(glogit)
        ctx.mark_non_differentiable(y_pred)
        return loss, y_pred

    @staticmethod
    def backward(ctx, gloss, _gy):
        (glogit,) = ctx.saved_tensors
        g = glogit * gloss
        return (None,) + tuple(g.view(shape) for shape in ctx.shapes)


def logit_bce(label, *terms):
    """terms: 1..4 tensors of (B,1)/(B,) logits that are summed. Returns (loss, y_pred)."""
    if not 1 <= len(terms) <= 4:
        raise ValueError("logit_bce takes 1..4 logit terms")
    _require_cuda(label, *terms)
    return _LogitBCE.apply(label, *terms)


# --------------------------------------------------------------------------------------
# Compositions whose dense contractions already run on the b2 GEMM; the remaining
# elementwise/outer-product pieces are stock torch ops until their fused kernels land
# (tracked in DESIGN.md "kernel status").
# --------------------------------------------------------------------------------------
class _CinLayer(torch.autograd.Function):
    """X_next (B,H',D) = Conv1x1(outer(X_0, X_i)) with the outer product kept in registers
    (compressed_interaction_net.py:70-73)."""

    @staticmethod
    def forward(ctx, x0, xk, weight, bias):
        x0, xk = _f32c(x0), _f32c(xk)
        B, F, D = x0.shape
        H = xk.shape[1]
        HO = weight.shape[0]
        out = torch.empty((B, HO, D), dtype=torch.float32, device=x0.device)
        _lib.call("b2_cin_fwd", _ptr(x0), _ptr(xk), _ptr(weight), _ptr(bias), B, F, H, HO, D, _ptr(out), _stream())
        ctx.save_for_backward(x0, xk, weight)
        ctx.w_param, ctx.b_param = weight, bias
        return out

    @staticmethod
    def backward(ctx, g):
        x0, xk, weight = ctx.saved_tensors
        g = _f32c(g)
        B, F, D = x0.shape
        H = xk.shape[1]
        HO = weight.shape[0]
        gx0 = torch.empty_like(x0)
        gxk = torch.empty_like(xk)
        gw = _grad_buffer(ctx.w_param, zero=False)
        _lib.call("b2_cin_bwd", _ptr(x0), _ptr(xk), _ptr(weight), _ptr(g), B, F, H, HO, D, _ptr(gx0), 0, _ptr(gxk),
                  _ptr(gw), _stream())
        gb = None
        if ctx.b_param is not None and ctx.b_param.requires_grad:
            gb = g.sum(dim=(0, 2))
        return gx0, gxk, gw, gb


def cin_supported(num_fields, hidden_units):
    hs = [num_fields] + list(hidden_units)
    return all(h <= 32 for h in hidden_units) and all(h <= 64 for h in hs[:-1])


def cin_forward(feature_emb, conv_layers, fc):
    """CompressedInteractionNet.forward (compressed_interaction_net.py:64-76)."""
    _require_cuda(feature_emb)
    X0 = feature_emb
    B, F, D = X0.shape
    Xi = X0
    pools = []
    fused = cin_supported(F, [c.out_channels for c in conv_layers])
    for conv in conv_layers:
        if fused:
            Xi = _CinLayer.apply(X0, Xi, conv.weight, conv.bias)       # weight (H', F*H, 1): contiguous (H', F*H)
        else:
            # shapes beyond the fused kernel's register budget: materialise like the reference does
            had = torch.einsum("bhd,bmd->bhmd", X0, Xi).reshape(B, -1, D)
            w = conv.weight.view(conv.out_channels, -1)
            rows = had.transpose(1, 2).reshape(B * D, -1)
            Xi = linear_act(rows, w, conv.bias, B2_ACT_NONE).view(B, D, -1).transpose(1, 2)
        pools.append(Xi.sum(dim=-1))
    return linear_act(torch.cat(pools, dim=-1), fc.weight, fc.bias, B2_ACT_NONE)


class _Dice(torch.autograd.Function):
    """Dice.forward (activations.py:49-50) on (M, C): column statistics + gate, one C-ABI call each way."""

    @staticmethod
    def forward(ctx, x, alpha, bn, training):
        x = _f32c(x)
        M, C = x.shape
        dev = x.device
        out = torch.empty_like(x)
        mean = torch.empty(C, dtype=torch.float32, device=dev)
        rstd = torch.empty(C, dtype=torch.float32, device=dev)
        ws = torch.empty(3 * C, dtype=torch.float64, device=dev)
        track = bn.track_running_stats and bn.running_mean is not None
        use_batch_stats = training or not track
        momentum = 0.0 if bn.momentum is None else float(bn.momentum)
        _lib.call("b2_dice_fwd", _ptr(x), _ptr(alpha), M, C, float(bn.eps), momentum, 1 if use_batch_stats else 0,
                  _ptr(bn.running_mean) if (track and training) or not use_batch_stats else None,
                  _ptr(bn.running_var) if (track and training) or not use_batch_stats else None,
                  _ptr(mean), _ptr(rstd), _ptr(ws), _ptr(out), _stream())
        if training and track and bn.num_batches_tracked is not None:
            bn.num_batches_tracked.add_(1)
        ctx.save_for_backward(x, alpha, mean, rstd)
        ctx.batch_stats = use_batch_stats
        ctx.alpha_param = alpha
        return out

    @staticmethod
    def backward(ctx, gout):
        x, alpha, mean, rstd = ctx.saved_tensors
        gout = _f32c(gout)
        M, C = x.shape
        gx = torch.empty_like(x)
        galpha = _grad_buffer(ctx.alpha_param, zero=False)
        ws = torch.empty(3 * C, dtype=torch.float64, device=x.device)
        _lib.call("b2_dice_bwd", _ptr(x), _ptr(gout), _ptr(alpha), _ptr(mean), _ptr(rstd), M, C,
                  1 if ctx.batch_stats else 0, _ptr(ws), _ptr(gx), _ptr(galpha), _stream())
        return gx, galpha, None, None


def dice_forward(X, bn, alpha, training):
    """Dice.forward (activations.py:49-50)."""
    _require_cuda(X, alpha)
    if X.dim() != 2:
        lead = X.shape[:-1]
        return _Dice.apply(X.reshape(-1, X.shape[-1]), alpha, bn, training).view(*lead, -1)
    return _Dice.apply(X, alpha, bn, training)


class _DinInput(torch.autograd.Function):
    """att_in ((B*L), 4d) = [t, h, t-h, t*h]  (target_attention.py:80-82) in one launch."""

    @staticmethod
    def forward(ctx, target, hist):
        target, hist = _f32c(target), _f32c(hist)
        B, L, d = hist.shape
        out = torch.empty((B * L, 4 * d), dtype=torch.float32, device=hist.device)
        _lib.call("b2_din_input_fwd", _ptr(target), _ptr(hist), B, L, d, _ptr(out), _stream())
        ctx.save_for_backward(target, hist)
        return out

    @staticmethod
    def backward(ctx, gin):
        target, hist = ctx.saved_tensors
        B, L, d = hist.shape
        gin = _f32c(gin)
        gt = torch.empty_like(target)
        gh = torch.empty_like(hist)
        _lib.call("b2_din_input_bwd", _ptr(target), _ptr(hist), _ptr(gin), B, L, d, _ptr(gt), _ptr(gh), 0, _stream())
        return gt, gh


class _DinWeightedSum(torch.autograd.Function):
    """out (B,d) = sum_l (w*mask)[b,l] * hist[b,l,:]  (target_attention.py:85-86,91)."""

    @staticmethod
    def forward(ctx, w, mask_u8, hist):
        w, hist = _f32c(w), _f32c(hist)
        B, L, d = hist.shape
        out = torch.empty((B, d), dtype=torch.float32, device=hist.device)
        _lib.call("b2_din_wsum_fwd", _ptr(w), _ptr(mask_u8), _ptr(hist), B, L, d, _ptr(out), _stream())
        ctx.save_for_backward(w, hist)
        ctx.mask = mask_u8
        return out

    @staticmethod
    def backward(ctx, gout):
        w, hist = ctx.saved_tensors
        B, L, d = hist.shape
        gout = _f32c(gout)
        gw = torch.empty_like(w)
        gh = torch.empty_like(hist)
        _lib.call("b2_din_wsum_bwd", _ptr(w), _ptr(ctx.mask), _ptr(hist), _ptr(gout), B, L, d, _ptr(gw), _ptr(gh),
                  _stream())
        return gw, None, gh


class _DinSoftmax(torch.autograd.Function):
    """p = softmax_L(w * mask + (-1e9)(1 - mask))  (target_attention.py:85-90), one launch each way."""

    @staticmethod
    def forward(ctx, w, mask_u8):
        w = _f32c(w)
        B, L = w.shape
        p = torch.empty_like(w)
        _lib.call("b2_din_softmax_fwd", _ptr(w), _ptr(mask_u8), B, L, _ptr(p), _stream())
        ctx.save_for_backward(p)
        ctx.mask = mask_u8
        return p

    @staticmethod
    def backward(ctx, g):
        (p,) = ctx.saved_tensors
        B, L = p.shape
        gw = torch.empty_like(p)
        _lib.call("b2_din_softmax_bwd", _ptr(p), _ptr(_f32c(g)), _ptr(ctx.mask), B, L, _ptr(gw), _stream())
        return gw, None


def din_attention(module, target_item, history_sequence, mask=None):
    """DIN_Attention.forward (target_attention.py:79-92): input construction, mask (+ softmax) and
    weighted sum are single launches; the attention MLP runs on the b2 GEMM + Dice kernels."""
    _require_cuda(target_item, history_sequence)
    B, L, d = history_sequence.shape
    att_in = _DinInput.apply(target_item, history_sequence)
    weight = module.attention_layer(att_in).view(B, L)
    mask_u8 = None
    if mask is not None:
        mask_u8 = mask.to(torch.uint8).contiguous() if mask.dtype != torch.uint8 else mask.contiguous()
    if module.use_softmax:      # softmax variant (:87-90): mask, additive -1e9 fill and softmax in one kernel
        weight = _DinSoftmax.apply(weight, mask_u8)
        mask_u8 = None
    return _DinWeightedSum.apply(weight, mask_u8, history_sequence)


# --------------------------------------------------------------------------------------
# Fused sparse front: embedding gather + FM product_sum + LogisticRegression in one launch
# --------------------------------------------------------------------------------------
class _Front(torch.autograd.Function):
    """(emb (B, F*D), logit (B,1)) = b2_front_fwd; backward = b2_front_bwd (one launch each).

    Reference: FeatureEmbedding.forward (feature_embedding.py:73-88) + FactorizationMachine.forward
    (factorization_machine.py:56-59) = InnerProductInteraction product_sum (inner_product.py:56-62)
    + LogisticRegression (logistic_regression.py:55-58)."""

    @staticmethod
    def forward(ctx, plan, lr_plan, idx_list, status, want_fm, bias, n_emb, *tables):
        emb_tables, lr_tables = tables[:n_emb], tables[n_emb:]
        batch = idx_list[0].shape[0]
        dev = emb_tables[0].device
        arena = torch.empty((batch, plan.width), dtype=torch.float32, device=dev)
        logit = torch.empty((batch, 1), dtype=torch.float32, device=dev)
        dim = plan.fields[0].dim
        sums = torch.empty((batch, dim), dtype=torch.float32, device=dev) if want_fm else None
        descs = plan.fill(emb_tables, idx_list, arena, batch)
        lr_descs = None
        if lr_plan is not None:
            lr_descs = lr_plan._descs
            for d, f, idx in zip(lr_descs, lr_plan.fields, idx_list):
                t = lr_tables[f.table_slot]
                d.table, d.vocab = t.data_ptr(), t.shape[0]
                d.idx, d.idx_stride = idx.data_ptr(), (idx.stride(0) if batch > 0 else 0)
                d.out, d.out_stride = 0, 0
        lazy = getattr(emb_tables[0], "_b2_lazy", None)       # set by arena.LazyTables on its parameters
        lz = lazy.ctx_for(plan, lr_plan, emb_tables, lr_tables) if lazy is not None else None
        # 3xTF32: the rows' small parts are written by the same kernel (no split pass over the arena);
        # the MLP finds them through the arena tensor (make_aux looks at `_b2_aux` of its input's base)
        small = torch.empty_like(arena) if (_x3_aux() and batch > 0) else None
        _lib.call("b2_front_fwd", descs, lr_descs, len(plan.fields), batch, ctx_code(idx_list),
                  1 if want_fm else 0, _ptr(bias), _ptr(logit), _ptr(sums), _ptr(status),
                  ctypes.byref(lz) if lz is not None else None, _ptr(small), _stream())
        if small is not None:
            arena._b2_aux = ("tf32x3", small, arena._version)
        ctx.lazy_ctx = lz
        ctx.plan, ctx.lr_plan, ctx.idx_list, ctx.want_fm = plan, lr_plan, idx_list, want_fm
        ctx.emb_tables, ctx.lr_tables, ctx.bias = emb_tables, lr_tables, bias
        ctx.save_for_backward(arena, sums)
        return arena, logit

    @staticmethod
    def backward(ctx, garena, glogit):
        arena, sums = ctx.saved_tensors
        plan, lr_plan, idx_list = ctx.plan, ctx.lr_plan, ctx.idx_list
        batch = idx_list[0].shape[0]
        garena = torch.zeros_like(arena) if garena is None else _f32c(garena)
        glogit = (torch.zeros((batch,), dtype=torch.float32, device=arena.device) if glogit is None
                  else _f32c(glogit).view(-1))
        egrads = [(_grad_buffer(t, zero=True, marks=True) if t.requires_grad else None) for t in ctx.emb_tables]
        lgrads = [(_grad_buffer(t, zero=True, marks=True) if t.requires_grad else None) for t in ctx.lr_tables]
        bias = ctx.bias
        gbias = _grad_buffer(bias, zero=True) if (bias is not None and bias.requires_grad) else None
        if batch > 0:
            descs = (b2_field * len(plan.fields))()
            base = garena.data_ptr()
            for d, f, idx in zip(descs, plan.fields, idx_list):
                g = egrads[f.table_slot]
                d.table = g.data_ptr() if g is not None else 0
                d.vocab = ctx.emb_tables[f.table_slot].shape[0]
                d.idx, d.idx_stride = idx.data_ptr(), idx.stride(0)
                d.out, d.out_stride = base + f.out_offset * 4, plan.width
                d.dim, d.seq_len, d.pool, d.padding_idx = f.dim, 1, 0, f.padding_idx
            lr_descs = None
            if lr_plan is not None:
                lr_descs = (b2_field * len(lr_plan.fields))()
                for d, f, idx in zip(lr_descs, lr_plan.fields, idx_list):
                    g = lgrads[f.table_slot]
                    d.table = g.data_ptr() if g is not None else 0
                    d.vocab = ctx.lr_tables[f.table_slot].shape[0]
                    d.idx, d.idx_stride = idx.data_ptr(), idx.stride(0)
                    d.dim, d.seq_len, d.pool, d.padding_idx = 1, 1, 0, f.padding_idx
            lz = ctx.lazy_ctx
            _lib.call("b2_front_bwd", descs, lr_descs, len(plan.fields), batch, ctx_code(idx_list),
                      1 if ctx.want_fm else 0, _ptr(arena), _ptr(garena), _ptr(sums), _ptr(glogit), _ptr(gbias),
                      ctypes.byref(lz) if lz is not None else None, _touch(egrads + lgrads), _stream())
        return (None, None, None, None, None, gbias, None) + tuple(egrads) + tuple(lgrads)


def front_supported(plan, lr_plan):
    """The fused front handles categorical-only fields of one common dim (% 4, <= 128)."""
    dims = set(f.dim for f in plan.fields)
    if len(dims) != 1 or any(f.seq_len != 1 for f in plan.fields):
        return False
    dim = plan.fields[0].dim
    if dim % 4 != 0 or dim > 128:
        return False
    if lr_plan is not None:
        if [f.name for f in lr_plan.fields] != [f.name for f in plan.fields]:
            return False
        if any(f.seq_len != 1 for f in lr_plan.fields):
            return False
    return True


def front(plan, lr_plan, idx_list, emb_tables, lr_tables, bias, want_fm, status=None):
    """Returns (emb arena (B, F*D), logit (B,1) = [FM product_sum] + [LR + bias])."""
    _require_cuda(*emb_tables)
    _require_cuda(*idx_list)
    idx_list, _ = _prep_indices(list(idx_list), plan.fields)
    return _Front.apply(plan, lr_plan, idx_list, status, bool(want_fm), bias, len(emb_tables),
                        *(tuple(emb_tables) + tuple(lr_tables)))


def table_mark(plan, lr_plan, idx_list, emb_tables, lr_tables, touch):
    """b2_table_mark on the current stream: flag (b2_touch `touch`, over the parameter arena) every granule of
    every table row the front (or gather) of `plan` reads for these ids.  Returns the index views the launch
    reads, which must stay alive until it has run."""
    _require_cuda(*idx_list)
    idx_list, code = _prep_indices(list(idx_list), plan.fields)
    batch = idx_list[0].shape[0]
    descs = (b2_field * len(plan.fields))()
    for d, f, idx in zip(descs, plan.fields, idx_list):
        t = emb_tables[f.table_slot]
        d.table, d.vocab, d.dim, d.seq_len = t.data_ptr(), t.shape[0], f.dim, 1
        d.idx, d.idx_stride = idx.data_ptr(), (idx.stride(0) if batch > 0 else 0)
    lr_descs = None
    if lr_plan is not None:
        lr_descs = (b2_field * len(lr_plan.fields))()
        for d, f, idx in zip(lr_descs, lr_plan.fields, idx_list):
            t = lr_tables[f.table_slot]
            d.table, d.vocab, d.dim, d.seq_len = t.data_ptr(), t.shape[0], 1, 1
            d.idx, d.idx_stride = idx.data_ptr(), (idx.stride(0) if batch > 0 else 0)
    _lib.call("b2_table_mark", descs, lr_descs, len(plan.fields), batch, code, ctypes.byref(touch), _stream())
    return idx_list

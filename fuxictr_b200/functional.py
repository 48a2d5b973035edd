"""torch.autograd bindings of the C-ABI kernels (device pointers in, device pointers out).

PyTorch is plumbing here: it owns device memory, the current stream and the autograd
tape; all arithmetic happens in libfuxictr_b200.so.  Every function requires CUDA
tensors and raises otherwise — there is no eager/CPU fallback on this path.
"""
import ctypes
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
def _grad_buffer(param, zero):
    slot = getattr(param, "_b2_slot", None)
    if slot is not None:
        arena = slot.arena
        if param.grad is None and slot.step_mark != arena.step_id:  # first hit this step
            slot.step_mark = arena.step_id
            view = arena.grad_view(slot)  # a fresh view object, so AccumulateGrad can steal it
            if zero and not arena.grads_are_zero:
                view.zero_()
            return view
    return torch.zeros_like(param) if zero else torch.empty_like(param)


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
        _lib.call("b2_embed_gather_hot_fwd", descs, len(plan.fields), batch, ctx_code(idx_list),
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
                grads[slot] = _grad_buffer(t, zero=True)
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
                      _ptr(count), _stream())
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
                grads[slot] = _grad_buffer(t, zero=True)
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
                          _ptr(gbias), _stream())
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


def transpose_f32(t, want_small):
    """(rows, cols) -> contiguous (cols, rows) [+ its 3xTF32 small part]."""
    rows, cols = t.shape
    out = torch.empty((cols, rows), dtype=torch.float32, device=t.device)
    small = torch.empty_like(out) if want_small else None
    _lib.call("b2_transpose_f32", _ptr(t), rows, cols, t.stride(0), _ptr(out), rows, _ptr(small), _stream())
    return out, small


def gemm_ex(a, b, out, a_mn=False, b_mn=False, a_small=None, b_small=None, bias=None, act=B2_ACT_NONE,
            mul=None, add=None, ybwd=None, act_bwd=B2_ACT_NONE, out_small=None, colsum=None, accumulate=False,
            out_pre=None, out_is_zero=False):
    """out (M,N) = epi(sum_k A(m,k) B(n,k)) on the wgmma kernel (b2_gemm_tc_ex).  a is (M,K), or (K,M) when
    a_mn (MN-major: the tensor is consumed as it lies, no transpose); b is (N,K), or (K,N) when b_mn.
    a_small / b_small: the operands' 3xTF32 small parts (both or neither).  Epilogue extras: ybwd/act_bwd
    (activation backward of the gradient's producer), out_small (3xTF32 small part of out), colsum (N)."""
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
    d.flags = (_lib.B2_GEMM_C_IS_ZERO if out_is_zero else 0) | (_lib.B2_GEMM_COLSUM_IS_ZERO if _is_zeroed(colsum) else 0)
    if a_small is None and not bf16 and _MATMUL["mode"] == "tf32x3" and _MATMUL["x3_inline"]:
        d.flags |= _lib.B2_GEMM_X3_INLINE
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
                 want_t_small=False, colsum=None):
    """One pass over x (R, C): [act-backward with y] -> out / out_small / out^T / out^T_small / column sums."""
    R, C = x.shape
    dev = x.device
    out = torch.empty((R, C), dtype=torch.float32, device=dev) if want_out else None
    small = torch.empty((R, C), dtype=torch.float32, device=dev) if want_small else None
    out_t = torch.empty((C, R), dtype=torch.float32, device=dev) if want_t else None
    t_small = torch.empty((C, R), dtype=torch.float32, device=dev) if want_t_small else None
    _lib.call("b2_prep_operand", _ptr(x), _ptr(y), act, R, C, _ptr(out), _ptr(small), _ptr(out_t), _ptr(t_small),
              _ptr(colsum), _stream())
    return out, small, out_t, t_small


def _tc_layer_ok(weight):
    """nn.Linear weight (N, K) usable by the tensor-core kernel in all three contractions
    (Y = X W^T, dX = dZ W, dW = dZ^T X): TMA needs 16-byte bases and leading dimensions % 4."""
    N, K = weight.shape
    return (_MATMUL["mode"] != "fp32" and N >= 16 and K >= 16 and N % 4 == 0 and K % 4 == 0
            and weight.is_contiguous() and weight.data_ptr() % 16 == 0)


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
        mode = _MATMUL["mode"]
        y = torch.empty((M, N), dtype=torch.float32, device=x.device)
        ctx.act, ctx.bias, ctx.has_bias = act, bias, bias is not None
        if N == 1 and weight.is_contiguous():
            ctx.kind = "head"
            _lib.call("b2_head_fwd", _ptr(x), _ptr(weight), _ptr(bias), M, K, act, _ptr(y), _stream())
            ctx.save_for_backward(x, weight, y if act != B2_ACT_NONE else None)
            return y
        if _tc_layer_ok(weight) and x.data_ptr() % 16 == 0:
            ctx.kind = "tc"
            x_small = make_aux(x)
            gemm_ex(x, weight, y, a_small=x_small, b_small=weight_aux(weight), bias=bias, act=act)
            ctx.x_small = x_small
            ctx.save_for_backward(x, weight, y if act != B2_ACT_NONE else None)
            return y
        ctx.kind = "simt"
        gemm_f32(x, weight, y, b_t=True, bias=bias, act=act)
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
        fused = act != B2_ACT_NONE
        if ctx.kind == "tc":
            x3 = _x3_aux()
            # dZ = act'(Y) * dY, its 3xTF32 small part and the bias gradient: one pass over dY
            gz, gz_small, _, _ = prep_operand(gy, y if fused else None, act, want_out=fused, want_small=x3, colsum=gb)
            if not fused:
                gz = gy
            if not x3:
                gz_small = make_aux(gz)          # bf16 mode: the bf16 operand of dZ (None for single-pass TF32)
            if need_x:
                gx = torch.empty((M, K), dtype=torch.float32, device=x.device)
                gemm_ex(gz, weight, gx, b_mn=True, a_small=gz_small, b_small=weight_aux(weight))   # dX = dZ W
            if need_w:
                gw = _grad_buffer(weight, zero=False)
                gemm_ex(gz, x, gw, a_mn=True, b_mn=True, a_small=gz_small, b_small=ctx.x_small,
                        out_is_zero=_is_zeroed(gw))                                                # dW = dZ^T X
            return gx, gw, gb, None
        # fp32 SIMT path
        gz = gy
        if fused or gb is not None:
            out, _, _, _ = prep_operand(gy, y if fused else None, act, want_out=fused, colsum=gb)
            if fused:
                gz = out
        if need_x:
            gx = torch.empty((M, K), dtype=torch.float32, device=x.device)
            gemm_f32(gz, weight, gx)
        if need_w:
            gw = _grad_buffer(weight, zero=False)
            gemm_f32(gz, x, gw, a_t=True)
        return gx, gw, gb, None


class _MLPChain(torch.autograd.Function):
    """A whole Linear(+ReLU/Sigmoid) chain of MLP_Block (mlp_block.py:64-85) as ONE autograd node, so that
    work can move across layer boundaries: the forward epilogue of layer i writes the 3xTF32 small part
    layer i+1 consumes; the dgrad GEMM of layer i+1 applies layer i's activation backward in its
    epilogue and emits dZ_i, its small part and layer i's bias gradient directly (the N = 1 head does
    the same in its fused backward).  Launches per 3-hidden-layer MLP step: 15 (was 26)."""

    @staticmethod
    def forward(ctx, x, acts, *params):
        x = _f32c(x)
        M = x.shape[0]
        L = len(acts)
        Ws, bs = params[0::2], params[1::2]
        x3 = _x3_aux()
        kinds = []
        for W in Ws:
            if W.shape[0] == 1 and W.is_contiguous():
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
                gemm_ex(h, W, y, a_small=smalls[-1], b_small=weight_aux(W), bias=b, act=act, out_small=y_small)
            else:
                kinds[i] = "simt"
                gemm_f32(h, W, y, b_t=True, bias=b, act=act)
            if want_small and y_small is None:
                y_small = make_aux(y)
            hs.append(y)
            smalls.append(y_small)
        ctx.acts, ctx.kinds, ctx.smalls, ctx.params = acts, kinds, smalls, params
        ctx.save_for_backward(*hs)
        return hs[-1]

    @staticmethod
    def backward(ctx, gy):
        hs = ctx.saved_tensors
        acts, kinds, smalls, params = ctx.acts, ctx.kinds, ctx.smalls, ctx.params
        Ws, bs = params[0::2], params[1::2]
        L = len(acts)
        M = hs[0].shape[0]
        dev = hs[0].device
        x3 = _x3_aux()
        grads = [None] * len(params)

        def bias_buf(i):
            b = bs[i]
            return _grad_buffer(b, zero=False) if (b is not None and b.requires_grad) else None

        g, g_small, g_is_dz = _f32c(gy), None, False     # g: gradient w.r.t. y_i; g_is_dz: already dZ_i (+ db_i done)
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
                gw = _grad_buffer(W, zero=False)
                gb = None if g_is_dz else bias_buf(i)          # g already dZ_i: activation backward and db_i are done
                gb_prev = bias_buf(i - 1) if fuse_prev else None
                fp32_small = gx_small if (gx_small is not None and gx_small.dtype == torch.float32) else None
                _lib.call("b2_head_bwd_ex", _ptr(h), _ptr(W), None if g_is_dz else _ptr(y), _ptr(g), M, K,
                          B2_ACT_NONE if g_is_dz else act, _ptr(gx), _ptr(gw), _ptr(gb),
                          acts[i - 1] if fuse_prev else B2_ACT_NONE, _ptr(fp32_small), _ptr(gb_prev),
                          1 if (_is_zeroed(gw) and (gb is None or _is_zeroed(gb))
                                and (gb_prev is None or _is_zeroed(gb_prev))) else 0, _stream())
                if gx_small is not None and fp32_small is None:     # bf16 mode: the head kernel emits fp32 only
                    gx_small = make_aux(gx)
                grads[2 * i] = gw
                if not g_is_dz:
                    grads[2 * i + 1] = gb
                if fuse_prev:
                    grads[2 * (i - 1) + 1] = gb_prev
                g, g_small, g_is_dz = gx, gx_small, fuse_prev
                continue
            if not g_is_dz:     # top of the chain (or below a non-fusing layer): one explicit pass over dY
                gb = bias_buf(i)
                fused = act != B2_ACT_NONE
                out, sm, _, _ = prep_operand(g, y if fused else None, act, want_out=fused,
                                             want_small=x3 and kinds[i] == "tc", colsum=gb)
                gz, gz_small = (out if fused else g), sm
                if gz_small is None and kinds[i] == "tc":
                    gz_small = make_aux(gz)          # bf16 mode (None for single-pass TF32)
                grads[2 * i + 1] = gb
            else:
                gz, gz_small = g, g_small
            if kinds[i] == "tc":
                if gx is not None:
                    prev_act = acts[i - 1] if fuse_prev else B2_ACT_NONE
                    gb_prev = bias_buf(i - 1) if fuse_prev else None
                    gemm_ex(gz, W, gx, b_mn=True, a_small=gz_small, b_small=weight_aux(W),
                            ybwd=hs[i] if (fuse_prev and prev_act != B2_ACT_NONE) else None, act_bwd=prev_act,
                            out_small=gx_small, colsum=gb_prev)                                   # dX (= dZ_{i-1})
                if W.requires_grad:
                    gw = _grad_buffer(W, zero=False)
                    gemm_ex(gz, h, gw, a_mn=True, b_mn=True, a_small=gz_small, b_small=smalls[i],
                            out_is_zero=_is_zeroed(gw))                                              # dW = dZ^T X
                    grads[2 * i] = gw
                g, g_small, g_is_dz = gx, gx_small, fuse_prev
            else:               # fp32 SIMT layer inside a chain (odd shapes)
                if gx is not None:
                    gemm_f32(gz, W, gx)
                if W.requires_grad:
                    gw = _grad_buffer(W, zero=False)
                    gemm_f32(gz, h, gw, a_t=True)
                    grads[2 * i] = gw
                g, g_small, g_is_dz = gx, None, False    # layer i-1 takes the explicit pass (its own db)
                continue
            if fuse_prev:
                grads[2 * (i - 1) + 1] = gb_prev
        return (g if ctx.needs_input_grad[0] else None, None) + tuple(grads)


class _CrossV2Layer(torch.autograd.Function):
    """One CrossNetV2 layer, x_next = x_i + x_0 * (x_i W^T + b) (cross_net.py:126-129): the GEMM epilogue
    applies `add + mul * (acc + bias)` and keeps lin = acc + bias for the backward — no elementwise pass.
    Backward: dlin = g * x_0 (one pass: value, 3xTF32 small part, bias gradient), dW = dlin^T x_i,
    dx_i = g + dlin W (epilogue add), dx_0 = g * lin."""

    @staticmethod
    def forward(ctx, x0, xi, weight, bias):
        x0, xi = _f32c(x0), _f32c(xi)
        M, d = xi.shape
        out = torch.empty_like(xi)
        lin = torch.empty_like(xi)
        ctx.tc = (_tc_layer_ok(weight) and weight.shape[0] == weight.shape[1] == d
                  and xi.data_ptr() % 16 == 0 and x0.data_ptr() % 16 == 0)
        ctx.xi_small = None
        if ctx.tc:
            ctx.xi_small = make_aux(xi)
            gemm_ex(xi, weight, out, a_small=ctx.xi_small, b_small=weight_aux(weight), bias=bias,
                    mul=x0, add=xi, out_pre=lin)
        else:
            gemm_f32(xi, weight, lin, b_t=True, bias=bias)
            torch.addcmul(xi, x0, lin, out=out)
        ctx.save_for_backward(x0, xi, lin, weight)
        ctx.bias = bias
        return out

    @staticmethod
    def backward(ctx, g):
        x0, xi, lin, weight = ctx.saved_tensors
        g = _f32c(g)
        bias = ctx.bias
        gb = _grad_buffer(bias, zero=False) if (bias is not None and bias.requires_grad) else None
        x3 = _x3_aux()
        dlin, dlin_small, _, _ = prep_operand(g, x0, B2_PREP_MUL, want_out=True, want_small=x3 and ctx.tc, colsum=gb)
        if ctx.tc and dlin_small is None:
            dlin_small = make_aux(dlin)          # bf16 mode (None for single-pass TF32)
        gxi = torch.empty_like(xi)
        gw = _grad_buffer(weight, zero=False) if weight.requires_grad else None
        if ctx.tc:
            gemm_ex(dlin, weight, gxi, b_mn=True, a_small=dlin_small, b_small=weight_aux(weight),
                    add=g)                                                                   # dx_i = g + dlin W
            if gw is not None:
                gemm_ex(dlin, xi, gw, a_mn=True, b_mn=True, a_small=dlin_small, b_small=ctx.xi_small, out_is_zero=_is_zeroed(gw))
        else:
            gemm_f32(dlin, weight, gxi, add=g)
            if gw is not None:
                gemm_f32(dlin, xi, gw, a_t=True)
        gx0 = g * lin if ctx.needs_input_grad[0] else None
        return gx0, gxi, gw, gb


def cross_v2_layer(x0, xi, weight, bias):
    _require_cuda(x0, xi, weight, bias)
    return _CrossV2Layer.apply(x0, xi, weight, bias)


def mlp_chain_supported():
    return _MATMUL["mode"] != "fp32"


def mlp_chain(x, layers):
    """layers: list of (weight, bias or None, act code).  Returns act_L(...act_0(x W_0^T + b_0)...)."""
    _require_cuda(x)
    acts = tuple(a for _, _, a in layers)
    flat = []
    for w, b, _ in layers:
        _require_cuda(w, b)
        flat += [w, b]
    if x.dim() != 2:
        lead = x.shape[:-1]
        return _MLPChain.apply(x.reshape(-1, x.shape[-1]), acts, *flat).view(*lead, -1)
    return _MLPChain.apply(x, acts, *flat)


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
        egrads = [(_grad_buffer(t, zero=True) if t.requires_grad else None) for t in ctx.emb_tables]
        lgrads = [(_grad_buffer(t, zero=True) if t.requires_grad else None) for t in ctx.lr_tables]
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
                      1 if ctx.want_fm else 0, _ptr(arena), _ptr(garena), _ptr(sums), _ptr(glogit),
                      _ptr(gbias), ctypes.byref(lz) if lz is not None else None, _stream())
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

"""Row-sharded embedding tables over the GPUs of one NVSwitch box (SURVEY.md 8e).

Row r of every table (embedding AND LogisticRegression) lives on rank ``r % world`` at local row
``r // world``; the dense part (FM reduce, MLPs) is data parallel.  The lookup + exchange is one
kernel per direction over NVLink peer memory (csrc/shard.cu): owners PUSH the looked-up rows into
the requesting rank's buffer, and PULL the gradient rows back; no NCCL all-to-all, no
variable-size splits, CUDA-graph capturable.  The only NCCL traffic left is the all-reduce of the
dense-parameter slice of the gradient arena and one scalar for the global gradient norm.

A ``PeerGroup`` supplies peer-mapped buffers and the cross-rank barrier:
  * ``SymmPeerGroup``    torch symmetric memory (one process per GPU, torchrun)
  * ``VirtualPeerGroup`` N "virtual ranks" inside ONE process / ONE GPU — the kernels cannot tell a
    local pointer from a peer pointer, so the whole algorithm is testable on a single GPU
    (tests/test_gpu_sharded.py drives the phases of all virtual ranks in lock step).
"""
import ctypes

import torch

from . import _lib
from . import functional as F2
from ._lib import b2_field


# --------------------------------------------------------------------------------------------
# shard / unshard a (vocab, dim) table:  rank r keeps rows r, r+world, r+2*world, ...
# --------------------------------------------------------------------------------------------
def shard_rows(weight, rank, world):
    return weight[rank::world].contiguous()


def local_rows(vocab, rank, world):
    return (vocab - rank + world - 1) // world if vocab > rank else 0


def unshard_rows(shards, vocab):
    """Inverse of shard_rows given the list of all ranks' shards."""
    world = len(shards)
    full = shards[0].new_empty((vocab,) + tuple(shards[0].shape[1:]))
    for r, s in enumerate(shards):
        full[r::world] = s
    return full


# --------------------------------------------------------------------------------------------
# Peer groups
# --------------------------------------------------------------------------------------------
class PeerGroup(object):
    world = 1
    rank = 0

    def alloc(self, name, shape, dtype):
        """Returns (local tensor, [device pointer of that buffer on every rank], peer_view) where
        peer_view(r) is a tensor aliasing rank r's copy of the buffer."""
        raise NotImplementedError

    def barrier(self):
        raise NotImplementedError

    def all_reduce_sum(self, buf):
        """buf <- sum over the ranks of buf (in place, on the current stream)."""
        raise NotImplementedError

    def gather(self, tensors):
        """Every rank's 1-D CUDA tensors, in rank order: [[rank 0's tensors[i], rank 1's, ...] for each i].  The
        tensors of one rank are equally long; the length may differ between ranks (a rank may have none)."""
        raise NotImplementedError


class SymmPeerGroup(PeerGroup):
    """One process per GPU; buffers come from torch.distributed symmetric memory (NVLink P2P)."""

    def __init__(self, group=None):
        import torch.distributed as dist
        import torch.distributed._symmetric_memory as symm_mem
        self._dist, self._symm = dist, symm_mem
        self.group = group if group is not None else dist.group.WORLD
        self.world, self.rank = dist.get_world_size(self.group), dist.get_rank(self.group)
        self._handles = []

    def alloc(self, name, shape, dtype):
        t = self._symm.empty(tuple(shape), dtype=dtype, device=torch.device("cuda", torch.cuda.current_device()))
        hdl = self._symm.rendezvous(t, self.group.group_name)
        self._handles.append(hdl)
        t.zero_()
        shape = tuple(shape)
        return t, [int(p) for p in hdl.buffer_ptrs], (lambda r: hdl.get_buffer(r, shape, dtype))

    def barrier(self):
        self._handles[0].barrier()      # device-side signal-pad barrier on the current stream

    def all_reduce_sum(self, buf):
        self._dist.all_reduce(buf, op=self._dist.ReduceOp.SUM, group=self.group)

    def gather(self, tensors):
        """NCCL: the lengths first, then one all_gather per tensor of buffers padded to the longest."""
        dist = self._dist
        dev = tensors[0].device
        counts = torch.empty(self.world, dtype=torch.int64, device=dev)
        dist.all_gather_into_tensor(counts, torch.tensor([tensors[0].numel()], dtype=torch.int64, device=dev),
                                    group=self.group)
        counts = [int(c) for c in counts.cpu()]
        width = max(counts)
        out = []
        for t in tensors:
            if width == 0:
                out.append([t.new_empty(0) for _ in range(self.world)])
                continue
            mine = t.new_zeros(width)
            mine[:t.numel()] = t
            every = t.new_empty(self.world * width)
            dist.all_gather_into_tensor(every, mine, group=self.group)
            out.append([every[r * width:r * width + counts[r]] for r in range(self.world)])
        return out


class VirtualPeerGroup(PeerGroup):
    """`world` virtual ranks in one process: buffers are ordinary tensors shared through a dict;
    barriers are no-ops because the test harness runs each phase for all virtual ranks in order."""

    def __init__(self, rank, world, registry):
        self.rank, self.world, self._reg = rank, world, registry

    def alloc(self, name, shape, dtype):
        bufs = self._reg.setdefault(name, {})
        bufs[self.rank] = torch.zeros(tuple(shape), dtype=dtype, device="cuda")
        return bufs[self.rank], _LazyPtrs(bufs, self.world), (lambda r: bufs[r])

    def barrier(self):
        pass

    def all_reduce_sum(self, buf):
        """A sum over virtual ranks needs every rank's buffer at once: lockstep_steps() does it between the
        phases of all ranks' optimizer steps.  One virtual rank is its own sum."""
        if self.world != 1:
            raise RuntimeError("virtual ranks sum over ranks in lock step: drive their optimizer steps with "
                               "fuxictr_b200.sharded.lockstep_steps")

    def gather(self, tensors):
        """One virtual rank is its own gather; more need every rank's tensors at once: lockstep_evaluate does it."""
        if self.world != 1:
            raise RuntimeError("virtual ranks evaluate in lock step: use fuxictr_b200.sharded.lockstep_evaluate / "
                               "lockstep_predict")
        return [[t] for t in tensors]


def lockstep_steps(optimizers, combine=None):
    """One FusedAdam step of every virtual rank, in lock step: each rank runs up to the point where its step
    sums a buffer over the ranks (FusedAdam.step_phases), the buffers are summed in rank order and the
    sum is written back to every rank, then every rank finishes.  `combine(bufs)` may replace that sum."""
    phases = [opt.step_phases() for opt in optimizers]
    while True:
        bufs = [next(ph, None) for ph in phases]
        if all(b is None for b in bufs):
            return
        if any(b is None for b in bufs):
            raise RuntimeError("virtual ranks disagree on the number of cross-rank sums in a step")
        if combine is not None:
            combine(bufs)
            continue
        total = bufs[0].clone()
        for b in bufs[1:]:
            total.add_(b)
        for b in bufs:
            b.copy_(total)


class _LazyPtrs(object):
    """Pointer list that resolves once all virtual ranks have allocated."""

    def __init__(self, bufs, world):
        self._bufs, self._world = bufs, world

    def __iter__(self):
        return iter([self._bufs[r].data_ptr() for r in range(self._world)])

    def __getitem__(self, r):
        return self._bufs[r].data_ptr()


def _ptr_array(ptrs):
    ptrs = list(ptrs)
    return (ctypes.c_void_p * len(ptrs))(*ptrs)


def slot_layout(seq_lens):
    """(slot_start, S): a one-slot field is one slot, an unpooled sequence of length L is L consecutive slots;
    slot s of sample b lands at b*S*D + s*D of the requester's (B, S*D) buffer."""
    starts, s = [], 0
    for n in seq_lens:
        starts.append(s)
        s += int(n)
    return starts + [s], s


def owned_capacity(world, batch_local, seq_lens):
    """Entries of the owned-row list: every (requester, sample, slot) candidate of the global batch, so the
    list can never overflow.  Entries and slot offsets are int32: refused (ValueError) past 2^31 - 1."""
    _, S = slot_layout(seq_lens)
    if batch_local * S >= 2 ** 31 or world * batch_local * S >= 2 ** 31:
        raise ValueError("sharded front: world * batch_local * slots = %d * %d * %d does not fit int32"
                         % (world, batch_local, S))
    return world * batch_local * S


def _distinct(tables):
    """(distinct tables in first-seen order, index of each entry in that list): a table shared by several
    fields (share_embedding) is one autograd input with one gradient buffer."""
    out, where = [], []
    for t in tables:
        for i, u in enumerate(out):
            if u is t:
                where.append(i)
                break
        else:
            where.append(len(out))
            out.append(t)
    return out, where


# --------------------------------------------------------------------------------------------
# The sharded front: FeatureEmbedding (+ FM product_sum) (+ LogisticRegression) over row shards
# --------------------------------------------------------------------------------------------
class ShardedFront(object):
    """Holds the peer buffers and launches the phases.

    emb_tables / lr_tables: lists of this rank's SHARD parameters (one per field, fp32 CUDA; a shared table
    appears once per field that reads it); vocabs: global vocabulary sizes; columns: column of each field
    in the batch matrix (its first column for a sequence); seq_lens: slots of each field (1, or the length
    of an unpooled sequence)."""

    def __init__(self, group, names, emb_tables, lr_tables, vocabs, columns, padding, dim, batch_local,
                 matrix_width, idx_dtype, bias=None, want_fm=True, seq_lens=None):
        self.group, self.names = group, list(names)
        self.emb_tables, self.lr_tables = list(emb_tables), (list(lr_tables) if lr_tables else None)
        self.vocabs, self.columns, self.padding = list(vocabs), list(columns), list(padding)
        self.dim, self.B, self.W = dim, batch_local, matrix_width
        self.F = len(self.names)
        self.seq_lens = [int(n) for n in seq_lens] if seq_lens is not None else [1] * self.F
        self.slot_start, self.S = slot_layout(self.seq_lens)
        self.bias, self.want_fm = bias, want_fm
        self.idx_dtype = idx_dtype
        self.idx_code = F2._IDX_CODE[idx_dtype]
        if max(self.vocabs) >= 2 ** 31:
            raise NotImplementedError("the id exchange narrows row numbers to int32 (vocabulary >= 2^31)")
        if self.S != self.F and (self.lr_tables or want_fm):
            raise NotImplementedError("sharded front: LR tables and the FM term need one slot per field "
                                      "(no sequences)")
        self.owned_cap = owned_capacity(group.world, batch_local, self.seq_lens)
        self._emb_distinct, self._emb_where = _distinct(self.emb_tables)
        self._lr_distinct, self._lr_where = _distinct(self.lr_tables or [])
        g = group
        # ids_all[p] = batch matrix of rank p: every rank BROADCASTS its ids into slot `rank` of all
        # peers (one launch of P2P stores), so the push kernel walks local memory only.
        # the slots hold int32 row numbers: the exchange narrows the collator's float64 on the fly.  The exchange
        # stores 16-byte vectors, so each slot starts 16-byte aligned: its pitch is rounded up to 4 ids.
        slot_ids = -(-batch_local * matrix_width // 4) * 4
        self.ids_all, self._ids_all_ptrs, self._ids_peer = g.alloc("ids_all", (g.world, slot_ids), torch.int32)
        esz = self.ids_all.element_size()
        self.src_code = self.idx_code          # dtype of the batch matrix handed to phase_ids
        self.idx_code = F2._IDX_CODE[torch.int32]
        self._slot_bytes = slot_ids * esz
        self.ids_ptrs = [self.ids_all.data_ptr() + p * self._slot_bytes for p in range(g.world)]
        self._ids_src = torch.empty((batch_local, matrix_width), dtype=idx_dtype, device="cuda")
        # rows this rank served in the forward (filled by the push, walked by the pull): int32[4] entries
        self.owned = torch.empty((self.owned_cap, 4), dtype=torch.int32, device="cuda")
        self.owned_count = torch.zeros(1, dtype=torch.int32, device="cuda")
        self.emb, self.emb_ptrs, _ = g.alloc("emb", (batch_local, self.S * dim), torch.float32)
        self.lrw, self.lrw_ptrs, _ = g.alloc("lrw", (batch_local, self.F), torch.float32)
        self.gemb, self.gemb_ptrs, _ = g.alloc("gemb", (batch_local, self.S * dim), torch.float32)
        # the padding row of every field (then its LR weight), published by its owner with the ids: each rank
        # fills its own padding slots from here, so no rank serves the others' (half of a DIN history)
        self.pad_rows, self.pad_ptrs, _ = g.alloc("pad_rows", (self.F * dim + self.F,), torch.float32)
        self.glogit, self.glogit_ptrs, _ = g.alloc("glogit", (batch_local,), torch.float32)
        # the evaluation round's row counts: word p = rows of rank p's batch, stored by p's publish (eval_phase_ids)
        self.rows_all, self.rows_ptrs, _ = g.alloc("rows_all", (g.world,), torch.int32)
        self._eval_rows = 0
        self._landed = None                  # (emb, logit) of an evaluation round, taken by the next sharded_front
        self.status = torch.zeros(1, dtype=torch.int32, device="cuda")
        # mean over the GLOBAL batch (rank_model.py:130): either the pull scales every gradient row by
        # 1/world (default), or the caller seeds backward() with 1/world and sets pull_scale = 1
        self.pull_scale = 1.0 / g.world
        self.on_dense_grads_ready = None     # set by RankModel.use_fused_optimizer (overlapped dense all-reduce)
        self._lazy_ctx = None                # b2_lazy_ctx when the shard tables are lazily evaluated (lazy_ctx())
        self._lazy_owner = None
        self._desc_cache = {}

    # -- descriptors --------------------------------------------------------------------------
    def _descs(self, tables, dim):
        """The b2_field array of `tables` (one per field), built once per set of table addresses: every launch of
        a step passes one (the ids launch, the push and the pull each take the tables or their gradients)."""
        key = (dim,) + tuple(t.data_ptr() if t is not None else 0 for t in tables)
        descs = self._desc_cache.get(key)
        if descs is not None:
            return descs
        if len(self._desc_cache) >= 16:
            self._desc_cache.clear()
        descs = self._desc_cache[key] = (b2_field * self.F)()
        for d, t, v, c, pad, n in zip(descs, tables, self.vocabs, self.columns, self.padding, self.seq_lens):
            d.table = t.data_ptr() if t is not None else 0
            d.vocab, d.idx_stride, d.dim, d.seq_len, d.pool = v, c, dim, n, 0
            d.padding_idx = -1 if pad is None else int(pad)
            d.idx, d.out, d.out_stride = 0, 0, 0
        return descs

    # -- forward phases -------------------------------------------------------------------------
    def phase_ids(self, batch_matrix):
        if tuple(batch_matrix.shape) != (self.B, self.W):
            raise ValueError("sharded front: a training batch matrix must be (batch_local, matrix_width) = (%d, %d), "
                             "got %s" % (self.B, self.W, tuple(batch_matrix.shape)))
        g = self.group
        src = batch_matrix
        if (not src.is_contiguous()) or src.data_ptr() % 16 != 0:
            self._ids_src.copy_(batch_matrix)
            src = self._ids_src
        dst = [int(base) + g.rank * self._slot_bytes for base in self._ids_all_ptrs]     # my slot on every rank
        lr = self._descs(self.lr_tables, 1) if self.lr_tables else None
        # the padding rows this rank owns travel in the same launch (the push reads them after the barrier)
        _lib.call("b2_shard_publish_ids", F2._ptr(src), self.src_code, self.B * self.W, _ptr_array(dst),
                  self._descs(self.emb_tables, self.dim), lr, self.F, g.world, g.rank, _ptr_array(self.pad_ptrs),
                  F2._stream())

    def lazy_ctx(self):
        """The b2_lazy_ctx of the shard tables when an optimizer evaluates them lazily (arena.LazyTables over
        this rank's shard parameters), else None.  Built once per LazyTables."""
        lazy = getattr(self.emb_tables[0], "_b2_lazy", None)
        if lazy is None:
            return None
        if self._lazy_owner is not lazy:
            self._lazy_ctx, self._lazy_owner = lazy.shard_ctx(self.emb_tables, self.lr_tables), lazy
        return self._lazy_ctx

    def phase_push(self):
        g = self.group
        lr = self._descs(self.lr_tables, 1) if self.lr_tables else None
        lz = self.lazy_ctx()
        _lib.call("b2_shard_push", self._descs(self.emb_tables, self.dim), lr, self.F, self.B, g.world, g.rank,
                  _ptr_array(self.ids_ptrs), self.idx_code, self.W, _ptr_array(self.emb_ptrs),
                  _ptr_array(self.lrw_ptrs) if lr is not None else None, F2._ptr(self.status),
                  F2._ptr(self.owned), F2._ptr(self.owned_count), self.owned_cap,
                  ctypes.byref(lz) if lz is not None else None, F2._ptr(self.pad_rows), F2._stream())

    def phase_reduce(self):
        """Local: logit (B,1) and field sums from the landed rows (one slot per field whenever there is a logit
        to reduce).  Returns (emb, logit, sums)."""
        # The landed rows are consumed in place: the next overwrite of this peer buffer is the NEXT
        # step's push, which is ordered after this step's backward (and its closing barrier).
        emb = self.emb
        if not self.lr_tables and not self.want_fm:     # embeddings only (DLRM): nothing to reduce
            return emb, torch.zeros((self.B, 1), dtype=torch.float32, device="cuda"), None
        logit = torch.empty((self.B, 1), dtype=torch.float32, device="cuda")
        sums = torch.empty((self.B, self.dim), dtype=torch.float32, device="cuda") if self.want_fm else None
        _lib.call("b2_front_reduce", F2._ptr(emb), F2._ptr(self.lrw) if self.lr_tables else None,
                  F2._ptr(self.bias), self.B, self.F, self.dim, 1 if self.want_fm else 0, F2._ptr(logit),
                  F2._ptr(sums), F2._stream())
        return emb, logit, sums

    # -- evaluation round (forward only, ragged) --------------------------------------------------
    # publish ids, rows and padding rows -> barrier -> lookup -> barrier -> reduce over `rows`.  The lookup keeps
    # no owned list (nothing is pulled) and takes no lazy context (evaluate() materialises lazy tables first), so
    # neither the owned list nor the lazy bookkeeping of the next training step is touched.  Every buffer the
    # round writes (ids_all, pad_rows, emb, lrw) is rewritten in full by the next training step's own publish
    # and push, inside a captured TrainPipeline graph too.
    def eval_rows(self, batch_matrix):
        """Rows of an evaluation batch matrix; refuses (ValueError) a batch the round cannot serve."""
        shape = tuple(batch_matrix.shape)
        if len(shape) != 2 or shape[1] != self.W:
            raise ValueError("sharded evaluation: the batch matrix is %s, the front was built for %d columns "
                             "(matrix_width)" % (shape, self.W))
        if shape[0] > self.B:
            raise ValueError("sharded evaluation: a batch of %d rows is more than batch_local = %d; build the "
                             "validation loader with batch_size <= batch_local" % (shape[0], self.B))
        return shape[0]

    def eval_phase_ids(self, batch_matrix):
        """Before the first barrier: this rank's ids, its row count and the padding rows it owns, to every rank.
        Returns the row count."""
        rows = self.eval_rows(batch_matrix)
        g = self.group
        src = batch_matrix if rows else None
        if rows and (src.dtype != self._ids_src.dtype or not src.is_contiguous() or src.data_ptr() % 16 != 0):
            src = self._ids_src[:rows]
            src.copy_(batch_matrix)
        dst = [int(base) + g.rank * self._slot_bytes for base in self._ids_all_ptrs]
        lr = self._descs(self.lr_tables, 1) if self.lr_tables else None
        _lib.call("b2_shard_publish_rows", F2._ptr(src), self.src_code, rows, self.W, self.B, _ptr_array(dst),
                  self._descs(self.emb_tables, self.dim), lr, self.F, g.world, g.rank, _ptr_array(self.pad_ptrs),
                  _ptr_array(self.rows_ptrs), F2._stream())
        self._eval_rows = rows
        self._landed = None
        return rows

    def eval_phase_lookup(self):
        """Between the barriers: the rows this rank owns, to every rank's first rows_all[p] samples."""
        g = self.group
        lr = self._descs(self.lr_tables, 1) if self.lr_tables else None
        _lib.call("b2_shard_lookup", self._descs(self.emb_tables, self.dim), lr, self.F, self.B, g.world, g.rank,
                  _ptr_array(self.ids_ptrs), self.W, _ptr_array(self.emb_ptrs),
                  _ptr_array(self.lrw_ptrs) if lr is not None else None, F2._ptr(self.rows_all), F2._ptr(self.status),
                  F2._ptr(self.pad_rows), F2._stream())

    def eval_phase_reduce(self):
        """After the second barrier: the logit of this rank's rows; leaves (emb (rows, S, D), logit (rows, 1)),
        views of the landed rows, for the model's forward (sharded_front takes them).  Nothing for 0 rows."""
        n = self._eval_rows
        if n == 0:
            self._landed = None
            return None
        emb = self.emb[:n]
        if not self.lr_tables and not self.want_fm:
            logit = torch.zeros((n, 1), dtype=torch.float32, device="cuda")
        else:
            logit = torch.empty((n, 1), dtype=torch.float32, device="cuda")
            sums = torch.empty((n, self.dim), dtype=torch.float32, device="cuda") if self.want_fm else None
            _lib.call("b2_front_reduce", F2._ptr(emb), F2._ptr(self.lrw) if self.lr_tables else None,
                      F2._ptr(self.bias), n, self.F, self.dim, 1 if self.want_fm else 0, F2._ptr(logit),
                      F2._ptr(sums), F2._stream())
        self._landed = (emb.view(n, self.S, self.dim), logit)
        return self._landed

    def take_landed(self):
        landed, self._landed = self._landed, None
        return landed

    # -- backward phases ------------------------------------------------------------------------
    def phase_gprep(self, gx, emb, sums, glogit, gbias=None):
        _lib.call("b2_front_gprep", F2._ptr(gx), F2._ptr(emb), F2._ptr(sums), F2._ptr(glogit), self.B, self.S,
                  self.dim, 1 if self.want_fm else 0, F2._ptr(self.gemb),
                  F2._ptr(self.glogit) if glogit is not None else None, F2._ptr(gbias),
                  1 if (gbias is not None and F2._is_zeroed(gbias)) else 0, F2._stream())

    def phase_pull(self, emb_grads, lr_grads):
        """emb_grads / lr_grads: the gradient buffer of each FIELD's table (one buffer, repeated, for a shared
        table: the pull adds both fields' rows into it)."""
        g = self.group
        lr = self._descs(lr_grads, 1) if lr_grads else None
        lz = self.lazy_ctx()        # lazy tables: the pull enqueues every row it scatters a gradient into
        _lib.call("b2_shard_pull", self._descs(emb_grads, self.dim), lr, self.F, self.B, g.world, g.rank,
                  _ptr_array(self.gemb_ptrs), _ptr_array(self.glogit_ptrs) if lr is not None else None,
                  self.pull_scale, F2._ptr(self.owned), F2._ptr(self.owned_count), self.owned_cap,
                  ctypes.byref(lz) if lz is not None else None, F2._touch(list(emb_grads) + list(lr_grads or ())),
                  F2._stream())

    def distinct_tables(self):
        """Every table once (embedding tables, then LR tables): the autograd inputs of sharded_front."""
        return tuple(self._emb_distinct) + tuple(self._lr_distinct)

    def field_views(self, emb):
        """(B, S, D) landed rows -> name -> (B, D) for a one-slot field, (B, L, D) for a sequence (views)."""
        out = {}
        for name, s0, n in zip(self.names, self.slot_start, self.seq_lens):
            out[name] = emb[:, s0] if n == 1 else emb[:, s0:s0 + n]
        return out


class _ShardedFrontFn(torch.autograd.Function):
    """(emb (B,S,D), logit (B,1)) with sharded tables; 2 barriers forward, 1 backward.  `tables` are the
    distinct tables (ShardedFront.distinct_tables): a shared table gets one gradient, the sum over its fields.

    No closing barrier: a peer buffer of this step is next written only behind the NEXT step's first
    barrier (ids visible), which no rank passes before every rank has finished this step's backward
    on its stream — and the pull walks the local owned-row list, not the peers' id matrices, so the
    early overwrite of `ids_all` by the next step's broadcast cannot race with it."""

    @staticmethod
    def forward(ctx, front, batch_matrix, bias, *tables):
        g = front.group
        front.phase_ids(batch_matrix)
        g.barrier()                      # every rank's ids are visible
        front.phase_push()
        g.barrier()                      # every owner's rows have landed here
        emb, logit, sums = front.phase_reduce()
        ctx.front, ctx.tables, ctx.bias = front, tables, bias
        ctx.save_for_backward(emb, sums)
        return emb.view(front.B, front.S, front.dim), logit

    @staticmethod
    def backward(ctx, gemb, glogit):
        front, tables, bias = ctx.front, ctx.tables, ctx.bias
        emb, sums = ctx.saved_tensors
        g = front.group
        gx = None if gemb is None else F2._f32c(gemb).view(front.B, -1)
        needs_logit = bool(front.lr_tables) or front.want_fm
        gl = None
        if needs_logit:
            gl = (torch.zeros(front.B, device="cuda") if glogit is None else F2._f32c(glogit).view(-1))
        gbias = None
        if bias is not None and bias.requires_grad:
            gbias = F2._grad_buffer(bias, zero=False)
        front.phase_gprep(gx, emb, sums, gl, gbias)      # also: LR bias gradient = sum_b glogit[b]
        if front.on_dense_grads_ready is not None:      # every dense gradient now exists: start their all-reduce
            front.on_dense_grads_ready()
        g.barrier()                      # every rank's gradient rows are ready to be pulled
        n = len(front._emb_distinct)
        egrads = [(F2._grad_buffer(t, zero=True, marks=True) if t.requires_grad else None) for t in tables[:n]]
        lgrads = [(F2._grad_buffer(t, zero=True, marks=True) if t.requires_grad else None) for t in tables[n:]]
        front.phase_pull([egrads[i] for i in front._emb_where],
                         [lgrads[i] for i in front._lr_where] if front.lr_tables else None)
        return (None, None, gbias) + tuple(egrads) + tuple(lgrads)


def sharded_front(front, batch_matrix):
    """(emb (B, S, D), logit (B, 1)) of this rank's samples, read from the row-sharded tables.  Inside an
    evaluation round the rows have already landed (ShardedFront.eval_phase_reduce): they are taken instead."""
    landed = front.take_landed()
    if landed is not None:
        if landed[0].shape[0] != batch_matrix.shape[0]:
            raise RuntimeError("sharded evaluation: %d landed rows for a batch of %d"
                               % (landed[0].shape[0], batch_matrix.shape[0]))
        return landed
    return _ShardedFrontFn.apply(front, batch_matrix, front.bias, *front.distinct_tables())


# --------------------------------------------------------------------------------------------
# Evaluation over row shards: every rank feeds its own shard of the split, the metrics cover all of them
# --------------------------------------------------------------------------------------------
def _loader_plan(generator):
    """(len(), batch_size) of an evaluation generator; None for what it does not tell."""
    try:
        n = len(generator)
    except TypeError:
        n = None
    bs = getattr(generator, "batch_size", None)
    return n, (int(bs) if isinstance(bs, int) else None)


def check_rounds(plans, names, batch_local):
    """Refuses (ValueError, alike on every rank) what would leave the ranks out of step.  Every rank must run the
    same number of evaluation rounds, each of them two barriers on every rank, so the lengths must agree.
    Batches must fit batch_local: a loader that declares a larger batch_size is refused up front, since a
    refusal inside a round would leave the other ranks at its barrier.  plans[r]: (len() or None, batch_size
    or None) of rank r's generator; names[r] describes that loader."""
    missing = [r for r, (n, _) in enumerate(plans) if n is None]
    if missing:
        raise ValueError("sharded evaluation needs generators with len() (every rank runs the same number of "
                         "rounds); %s has none" % ", ".join("rank %d's %s" % (r, names[r]) for r in missing))
    lengths = [n for n, _ in plans]
    if len(set(lengths)) != 1:
        raise ValueError("sharded evaluation: the ranks' generators have different lengths %s; every rank must run "
                         "the same number of rounds (MatrixDataLoader(shard=(rank, world), drop_last=False) does)"
                         % lengths)
    wide = [r for r, (_, bs) in enumerate(plans) if bs is not None and bs > batch_local]
    if wide:
        raise ValueError("sharded evaluation: rank %d's %s has batch_size %d, more than batch_local = %d; build the "
                         "validation loader with batch_size <= batch_local"
                         % (wide[0], names[wide[0]], plans[wide[0]][1], batch_local))


def _check_rounds_collective(group, generator, batch_local):
    """check_rounds over real ranks: one small gather of every rank's (len(), batch_size) (-1: none)."""
    n, bs = _loader_plan(generator)
    mine = torch.tensor([-1 if n is None else n, -1 if bs is None else bs], dtype=torch.int64, device="cuda")
    plans = [tuple(None if int(v) < 0 else int(v) for v in t.cpu()) for t in group.gather([mine])[0]]
    names = ["loader" if r != group.rank else type(generator).__name__ for r in range(group.world)]
    check_rounds(plans, names, batch_local)


def eval_rank_rounds(model, generator, acc, with_labels=True):
    """One rank's evaluation, as phases: yields at each of the two cross-rank barriers of a round, which the
    caller runs (real ranks) or fills with the same phase of every other virtual rank (lockstep_evaluate).
    Each round: publish this rank's ids and row count, lookup, reduce over its rows, then the model's own
    forward on the landed rows (a rank with 0 rows serves its peers and skips it); the predictions (and
    labels) are appended to `acc` (metrics.DeviceMetrics), in HBM.  Run under torch.no_grad() in eval()."""
    front = model._sharded_front
    try:
        for batch in generator:
            rows = front.eval_phase_ids(model._batch_matrix(batch))
            yield
            front.eval_phase_lookup()
            yield
            front.eval_phase_reduce()
            if rows:
                acc.append(model.forward(batch)["y_pred"], model.get_labels(batch) if with_labels else None)
    finally:
        front._landed = None


def _run_rounds(group, phases):
    for _ in phases:
        group.barrier()


def _lockstep_rounds(phase_lists):
    """Every virtual rank's phases in lock step: each rank runs up to its next barrier, in rank order."""
    end = object()
    try:
        while True:
            done = [next(ph, end) is end for ph in phase_lists]
            if all(done):
                return
            if any(done):
                raise RuntimeError("virtual ranks disagree on the number of evaluation rounds")
    finally:
        for ph in phase_lists:
            ph.close()


def _rank_check(models):
    for r, m in enumerate(models):
        front = getattr(m, "_sharded_front", None)
        if front is None:
            raise ValueError("model %d is not sharded (enable_sharding)" % r)
        if front.group.rank != r or front.group.world != len(models):
            raise ValueError("models must be virtual ranks 0..%d in rank order" % (len(models) - 1))


def _union_metrics(preds, labels, metrics):
    """The metric words (metrics.metric_words) of every rank's predictions, concatenated in rank order."""
    from .metrics import metric_words
    return metric_words(torch.cat(list(labels)), torch.cat(list(preds)), metrics)


def evaluate_sharded(model, generator, metrics):
    """RankModel.evaluate of a row-sharded model: a collective call.  Each rank feeds its own shard of the split
    (same len() on every rank, checked first); logloss / AUC cover the union of all ranks' rows, computed on
    rank 0 over the rank-ordered union and handed to every rank, so every rank returns the same dict, bit for bit."""
    from .metrics import DeviceMetrics, check_metrics, metrics_from_words
    check_metrics(metrics)
    group = model._sharded_front.group
    if isinstance(group, VirtualPeerGroup) and group.world != 1:
        raise RuntimeError("virtual ranks evaluate in lock step: use fuxictr_b200.sharded.lockstep_evaluate")
    _check_rounds_collective(group, generator, model._sharded_front.B)
    acc = DeviceMetrics(model.device)
    model.eval()
    with torch.no_grad():
        _run_rounds(group, eval_rank_rounds(model, generator, acc))
        preds, labels = group.gather([acc.predictions(), acc.labels()])
        n = sum(p.numel() for p in preds)
        if n == 0 and "AUC" in metrics:                # every rank knows n: they all raise
            raise ValueError("AUC of an empty prediction set is undefined")
        if group.rank == 0:
            words = _union_metrics(preds, labels, metrics)
        else:
            words = torch.zeros(6, dtype=torch.int64, device=model.device)
        words = group.gather([words])[0][0]           # rank 0's words, on every rank
    return metrics_from_words(words.cpu(), n, metrics)


def predict_sharded(model, generator):
    """RankModel.predict of a row-sharded model: a collective call (every rank runs the same rounds) that returns
    THIS rank's predictions, in its generator's order, as a float64 numpy array — the data-parallel meaning."""
    from .metrics import DeviceMetrics
    group = model._sharded_front.group
    if isinstance(group, VirtualPeerGroup) and group.world != 1:
        raise RuntimeError("virtual ranks predict in lock step: use fuxictr_b200.sharded.lockstep_predict")
    _check_rounds_collective(group, generator, model._sharded_front.B)
    acc = DeviceMetrics(model.device)
    model.eval()
    with torch.no_grad():
        _run_rounds(group, eval_rank_rounds(model, generator, acc, with_labels=False))
    return acc.predictions().cpu().numpy().astype("float64")


def _lockstep_accumulate(models, generators, with_labels):
    from .metrics import DeviceMetrics
    _rank_check(models)
    if len(generators) != len(models):
        raise ValueError("one generator per virtual rank (%d models, %d generators)" % (len(models), len(generators)))
    check_rounds([_loader_plan(g) for g in generators], [type(g).__name__ for g in generators],
                 models[0]._sharded_front.B)
    accs = [DeviceMetrics(m.device) for m in models]
    for m in models:
        m.materialize_tables()
        m.eval()
    with torch.no_grad():
        _lockstep_rounds([eval_rank_rounds(m, g, a, with_labels) for m, g, a in zip(models, generators, accs)])
    return accs


def lockstep_evaluate(models, generators, metrics=None):
    """evaluate() of every virtual rank (models[r] is rank r, generators[r] its shard of the split), each round's
    phases driven for all ranks in order; the same per-rank code as evaluate_sharded.  Returns one dict per
    rank — the same metrics over the rank-ordered union of every rank's rows."""
    from .metrics import check_metrics, metrics_from_words
    names = metrics if metrics is not None else ["logloss", "AUC"]
    check_metrics(names)
    accs = _lockstep_accumulate(models, generators, True)
    with torch.no_grad():
        words = _union_metrics([a.predictions() for a in accs], [a.labels() for a in accs], names)
    result = metrics_from_words(words.cpu(), sum(a.n for a in accs), names)
    return [result.copy() for _ in models]


def lockstep_predict(models, generators):
    """predict() of every virtual rank in lock step: each rank's own predictions (float64 numpy), in rank order."""
    return [a.predictions().cpu().numpy().astype("float64") for a in _lockstep_accumulate(models, generators, False)]

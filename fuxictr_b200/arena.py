"""Flat HBM arenas for parameters, gradients and Adam state + the fused dense optimizer.

H100-first memory layout: every trainable tensor of a model is a 16-byte-aligned slice
of ONE fp32 arena `P`; its gradient is the same slice of arena `G`; Adam's moments are
the same slices of `M` and `V`.  The Parameter *objects* are kept (the reference builds
its optimizer and state_dict around them, rank_model.py:92, 417-433) — only their
`.data` is re-pointed.  Backward kernels write gradients straight into `G`
(functional._grad_buffer), so `clip_grad_norm_ + Adam` (rank_model.py:321-322) becomes
two streaming kernels over the arena instead of ~6 launches per parameter.
"""
import ctypes

import numpy as np
import torch

from . import _lib
from . import functional as F2


class _Slot(object):
    __slots__ = ("arena", "offset", "numel", "shape", "step_mark")

    def __init__(self, arena, offset, numel, shape):
        self.arena, self.offset, self.numel, self.shape = arena, offset, numel, shape
        self.step_mark = -1


class ParamArena(object):
    """Re-homes the trainable fp32 CUDA parameters of `module` into one flat buffer."""

    ALIGN = 4  # floats (16 bytes): every slice is float4-addressable
    GRANULE = 16  # floats (64 bytes) per byte of `touched`

    def __init__(self, module, first=()):
        """`first`: parameters to place at the front of the arena (e.g. the row-sharded tables of a
        multi-GPU run, so that the replicated dense parameters form one contiguous tail slice)."""
        params = list(first) + [p for p in module.parameters() if p.requires_grad]
        seen, uniq = set(), []
        for p in params:
            if id(p) not in seen:
                seen.add(id(p))
                uniq.append(p)
        n_first = len(set(id(p) for p in first))
        if not uniq:
            raise ValueError("module has no trainable parameters")
        dev = uniq[0].device
        if dev.type != "cuda":
            raise RuntimeError("ParamArena needs CUDA parameters (model_to_device() first)")
        for p in uniq:
            if p.dtype != torch.float32 or p.device != dev:
                raise RuntimeError("ParamArena supports float32 parameters on one device")
        off = 0
        slots = []
        self.tail_offset = 0           # first element of the non-`first` (dense, replicated) slice
        for i, p in enumerate(uniq):
            if i == n_first:
                self.tail_offset = off
            if i < n_first:
                # tables start on a 64-byte granule of `touched`: a touched 16-float row then flags one granule, not two
                off = (off + self.GRANULE - 1) // self.GRANULE * self.GRANULE
            slots.append((p, off))
            off += (p.numel() + self.ALIGN - 1) // self.ALIGN * self.ALIGN
        if n_first >= len(uniq):
            self.tail_offset = off
        self.numel = off
        self.P = torch.zeros(off, dtype=torch.float32, device=dev)
        # 4 spare floats behind the gradient arena: the sharded optimizer parks the local sum of
        # squares there so that ONE all-reduce carries the dense gradients and the norm term
        self._G_ext = torch.zeros(off + 4, dtype=torch.float32, device=dev)
        self.G = self._G_ext[:off]
        self._G_ext._b2_arena = self          # lets a kernel wrapper recognise a slice of this (zeroed) arena
        self.params = uniq
        self.tail_params = uniq[n_first:]      # the dense (non-`first`) parameters, contiguous from tail_offset
        self.step_id = 0
        self.grads_are_zero = True
        # Weight gradients still being written on a side stream (functional._WgradFork): (event, operands kept
        # alive) pairs.  A backward leaves them here, instead of joining them itself, only while defer_join is set:
        # fused_train_step sets it around the backward of its fused-logit path (no regulariser: the MLP chain is the
        # one reader of its weights), and FusedAdam joins where it first reads the dense tail.
        self.defer_join = False
        self.pending = []
        # Touched-granule flags of the table prefix G[:tail_offset] (b2_touch): one byte per 16 floats.  The
        # backward kernels set the byte of every granule they add a table gradient into; FusedAdam's clip
        # and Adam passes read G only there and clear the bytes again.  Invariant: every nonzero float of
        # G[:tail_offset] lies in a flagged granule.  None: no table prefix, or lazy tables (own worklist).
        self.touched, self.touch = None, None
        # Set while FusedAdam's untouched-granule pass may run (between start_early_tables and the step): a
        # granule flagged now may already have had its g = 0 update, so only the front kernels, whose every
        # granule was flagged from the ids before that pass, may still write table gradients.
        self.flags_frozen = False
        if self.tail_offset > 0:
            self.touched = torch.zeros((self.tail_offset + self.GRANULE - 1) // self.GRANULE, dtype=torch.uint8,
                                       device=dev)
            self.touch = _lib.b2_touch(self.touched.data_ptr(), self.G.data_ptr(), self.tail_offset)
        with torch.no_grad():
            for p, o in slots:
                dst = self.P[o:o + p.numel()].view(p.shape)
                dst.copy_(p.data)
                p.data = dst
                p._b2_slot = _Slot(self, o, p.numel(), tuple(p.shape))
                p.grad = None

    def grad_view(self, slot):
        return self.G[slot.offset:slot.offset + slot.numel].view(slot.shape)

    def mark_slot(self, slot):
        """Flag every granule of `slot` (its gradient is written by something that sets no flags)."""
        if self.touched is not None and slot.offset < self.tail_offset:
            if self.flags_frozen:
                raise RuntimeError("a table gradient is written outside the fused front while the untouched table "
                                   "rows are being updated early; call fuxictr_b200.arena.set_early_table_adam(False)")
            end = min(slot.offset + slot.numel, self.tail_offset)
            self.touched[slot.offset // 16:(end + 15) // 16].fill_(1)

    def join_grads(self):
        """The current stream waits until every pending side-stream gradient is written."""
        cur = torch.cuda.current_stream() if self.pending else None
        for ev, _ in self.pending:
            cur.wait_event(ev)
        self.pending = []

    def begin_step(self, grads_zeroed):
        """Call once per training step before backward. `grads_zeroed`: G is already all-zero
        (e.g. the previous fused Adam step cleared it); otherwise sparse-written grads
        (embedding tables) are zero-filled lazily by the kernels' wrappers."""
        self.join_grads()
        self.step_id += 1
        self.grads_are_zero = bool(grads_zeroed)
        for p in self.params:
            p.grad = None

    def zero_grads(self):
        self.G.zero_()


def adam_consts(betas):
    """(fl32(1 - beta1), fl32(beta2), fl32(1 - beta2)): adam_const() in csrc/dense.cu and make_const() in
    csrc/lazy_adam.cu.  1 - beta is taken in double and rounded once, as torch.optim.Adam passes the Python float
    1 - beta2 to addcmul_; rounding beta to fp32 first would leave V 1e-5 (relative) off torch's."""
    b1, b2 = float(betas[0]), float(betas[1])
    return float(np.float32(1.0 - b1)), float(np.float32(b2)), float(np.float32(1.0 - b2))


class LazyTables(object):
    """Bookkeeping of the lazily evaluated tables (see b2_lazy_ctx in include/fuxictr_b200.h):
    per-row `last_step`, the per-step worklist, the schedule table shared with the dense pass."""

    SCHED_LEN = 1 << 20   # optimizer steps the schedule table can hold

    def __init__(self, arena, tables):
        self.arena = arena
        self.tables = list(tables)
        rows = sum(int(p.shape[0]) for p in self.tables)
        if rows > 2 ** 31 - 1:
            # worklist entries and the row numbers the kernels compute are int32
            raise ValueError("lazy tables: %d rows on this device; at most 2^31 - 1 are supported (row-shard the "
                             "tables over more GPUs)" % rows)
        dev = arena.P.device
        base = 0
        descs = (_lib.b2_lazy_table * len(self.tables))()
        for d, p in zip(descs, self.tables):
            if p.dim() != 2 or getattr(p, "_b2_slot", None) is None:
                raise ValueError("lazy tables must be 2-D parameters living in the arena")
            p._b2_lazy, p._b2_grow_base = self, base
            d.param, d.rows, d.grow_base, d.dim = p.data_ptr(), p.shape[0], base, p.shape[1]
            base += p.shape[0]
        self.total_rows = base
        raw = bytes(descs)
        self.tables_dev = torch.frombuffer(bytearray(raw), dtype=torch.uint8).to(dev)
        self.last_step = torch.zeros(base, dtype=torch.int32, device=dev)
        self.mark = torch.zeros(base, dtype=torch.int32, device=dev)
        self.capacity = base
        self.worklist = torch.zeros(base, dtype=torch.int32, device=dev)
        self.counter = torch.zeros(1, dtype=torch.int32, device=dev)
        self.sched = None      # FusedAdam.enable_lazy shares its schedule table
        self.opt = None
        self._ctx_cache = {}

    def _new_ctx(self, emb_tables, lr_tables):
        """b2_lazy_ctx with field i of the launch reading emb_tables[i] (and lr_tables[i])."""
        opt, a = self.opt, self.arena
        ctx = _lib.b2_lazy_ctx()
        ctx.last_step, ctx.sched = self.last_step.data_ptr(), self.sched.data_ptr()
        ctx.step_dev, ctx.mark = opt.step_dev.data_ptr(), self.mark.data_ptr()
        ctx.worklist, ctx.counter = self.worklist.data_ptr(), self.counter.data_ptr()
        ctx.delta_m = (opt.M.data_ptr() - a.P.data_ptr()) // 4
        ctx.delta_v = (opt.V.data_ptr() - a.P.data_ptr()) // 4
        ctx.w1, ctx.beta2, ctx.w2 = adam_consts(opt.betas)
        ctx.eps = opt.eps
        ctx.worklist_capacity = self.capacity
        for i, t in enumerate(emb_tables):
            ctx.grow_emb[i] = t._b2_grow_base
        for i, t in enumerate(lr_tables or ()):
            ctx.grow_lr[i] = t._b2_grow_base
        return ctx

    def ctx_for(self, plan, lr_plan, emb_tables, lr_tables):
        key = (id(plan), id(lr_plan))
        ctx = self._ctx_cache.get(key)
        if ctx is None:
            ctx = self._new_ctx([emb_tables[f.table_slot] for f in plan.fields],
                                [lr_tables[f.table_slot] for f in lr_plan.fields] if lr_plan is not None else None)
            self._ctx_cache[key] = ctx
        return ctx

    def shard_ctx(self, emb_tables, lr_tables):
        """The context of a sharded front (one shard table per field): rows are this rank's local rows."""
        return self._new_ctx(emb_tables, lr_tables)

    def materialize(self):
        """Bring every row up to date (before reading the tables outside the kernels)."""
        opt, a = self.opt, self.arena
        st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
        _lib.call("b2_lazy_materialize", ctypes.c_void_p(self.tables_dev.data_ptr()), len(self.tables),
                  self.total_rows, (opt.M.data_ptr() - a.P.data_ptr()) // 4,
                  (opt.V.data_ptr() - a.P.data_ptr()) // 4, ctypes.c_void_p(self.last_step.data_ptr()),
                  ctypes.c_void_p(self.sched.data_ptr()), ctypes.c_void_p(opt.step_dev.data_ptr()),
                  opt.betas[0], opt.betas[1], opt.eps, st)


_EARLY = {"on": True, "side": {}}     # the untouched-table-granule side stream of each device


def set_early_table_adam(on):
    """on (default): where FusedAdam.early_tables_ok() holds, a step updates the table granules its batch does not
    touch on a side stream while its forward and backward run (FusedAdam.start_early_tables); off: the whole
    table pass after the norm, one launch (the serial order the split is tested against)."""
    _EARLY["on"] = bool(on)


class FusedAdam(object):
    """clip_grad_norm_(max_norm) + Adam over a ParamArena, two kernels per step.

    Semantics: nn.utils.clip_grad_norm_(params, max_norm) followed by torch.optim.Adam with
    its defaults (rank_model.py:321-322, torch_utils.py:58-79).  The step counter lives on
    the device so the whole step can be captured in a CUDA graph.
    """

    def __init__(self, arena, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, max_norm=10.0,
                 zero_grad_in_step=True):
        self.arena = arena
        self.lr, self.betas, self.eps, self.max_norm = float(lr), betas, float(eps), max_norm
        dev = arena.P.device
        self.M = torch.zeros_like(arena.P)
        self.V = torch.zeros_like(arena.P)
        self.step_dev = torch.zeros((), dtype=torch.int64, device=dev)
        self.sumsq = torch.zeros((), dtype=torch.float32, device=dev)
        self.zero_grad_in_step = zero_grad_in_step
        self.lazy = None             # LazyTables: tables in G[:tail_offset] are updated row-wise, exactly
        self.sched = None            # per-step scalar table: only the lazy replay needs one (enable_lazy)
        self.host_steps = 0          # optimizer steps issued (eager calls + graph replays), see count_step()
        self.grad_allreduce = False  # data-parallel replicas: average G across ranks before the step
        self.sharded = False         # row-sharded tables in G[:tail_offset], replicated dense params after
        self.dense_prescaled = False # sharded: gradients were born divided by the world size (no mul_ after the all-reduce)
        self._side = None            # overlap: side stream + its own communicator for the dense-gradient all-reduce
        self._side_group = None
        self._early_pending = False
        self._early = None           # (done event, operands kept alive) of this step's untouched-granule pass

    # CTAs (= SMs, one 1024-thread CTA each) of the untouched-granule pass; tools/table_adam_overlap_times.py
    EARLY_CTAS = 32

    def early_tables_ok(self):
        """The step's table flags are final once its ids are known: one process, flags cleared by every step,
        dense (not lazy) tables.  The caller adds what only the model knows: every table gradient comes from the
        front kernels marked by start_early_tables."""
        a = self.arena
        return (_EARLY["on"] and not self.sharded and not self.grad_allreduce and self.zero_grad_in_step
                and self.lazy is None and a.touched is not None)

    def start_early_tables(self, plan, lr_plan, idx_list, emb_tables, lr_tables):
        """Fork: on a side stream, flag every table granule this step's front reads (b2_table_mark over the
        parameter arena, from the ids alone), then give every other table granule its g = 0 update of the coming
        step (b2_adam_untouched).  step_phases joins before it counts the step and then updates only the flagged
        granules (b2_adam_touched).  Hazards: the front reads P only in flagged granules and the side pass writes
        only unflagged ones; the previous step's touched pass cleared every flag before this fork; flags are
        cleared only after the join; until the join nothing but the front kernels may write a table gradient
        (ParamArena.flags_frozen)."""
        a = self.arena
        dev = a.P.device
        side = _EARLY["side"].get(dev)
        if side is None:
            side = _EARLY["side"][dev] = torch.cuda.Stream(device=dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        vp = ctypes.c_void_p
        touch = _lib.b2_touch(a.touched.data_ptr(), a.P.data_ptr(), a.tail_offset)
        with torch.cuda.stream(side):
            keep = F2.table_mark(plan, lr_plan, idx_list, emb_tables, lr_tables, touch)
            _lib.call("b2_adam_untouched", vp(a.P.data_ptr()), vp(self.M.data_ptr()), vp(self.V.data_ptr()),
                      a.tail_offset, vp(a.touched.data_ptr()), self.lr, self.betas[0], self.betas[1], self.eps,
                      vp(self.step_dev.data_ptr()), self.EARLY_CTAS, vp(side.cuda_stream))
            done = torch.cuda.Event()
            done.record(side)
        self._early = (done, keep)
        a.flags_frozen = True

    def enable_lazy(self, tables):
        """Evaluate the dense Adam semantics of `tables` (the arena's leading parameters) lazily."""
        self.sched = torch.zeros((LazyTables.SCHED_LEN, 2), dtype=torch.float32, device=self.arena.P.device)
        self.lazy = LazyTables(self.arena, tables)
        self.lazy.opt = self
        self.lazy.sched = self.sched          # one schedule table for the dense and the lazy kernels
        self.arena.touched, self.arena.touch = None, None    # the worklist says which rows carry a gradient
        return self.lazy

    def count_step(self, n=1):
        """Host-side count of optimizer steps (TrainPipeline calls it once per graph replay, step()
        once per eager call).  The lazy replay reads sched[t] for every step t it catches up on, and
        the table holds SCHED_LEN entries: refuse to run past it instead of reading out of bounds
        (the dense pass computes its two scalars in-kernel and has no such limit)."""
        self.host_steps += n
        if self.lazy is not None and self.host_steps >= LazyTables.SCHED_LEN - 1:
            raise RuntimeError("lazy Adam: the per-step schedule table holds %d steps; materialize_tables() and "
                               "rebuild the optimizer (or use the dense pass) before step %d"
                               % (LazyTables.SCHED_LEN, self.host_steps))

    def enable_dense_overlap(self):
        """Sharded runs: all-reduce the dense-gradient tail on a side stream (own NCCL communicator) as soon
        as the last dense gradient exists — the sharded front calls start_dense_allreduce() right after its
        gradient-prep kernel — so it overlaps the barrier + pull of the row gradients; step() then only
        exchanges the one norm scalar on the main stream.  Collective: call on every rank."""
        import torch.distributed as dist
        self._side = torch.cuda.Stream(device=self.arena.P.device)
        self._side_group = dist.new_group()

    def start_dense_allreduce(self):
        a = self.arena
        if self._side is None or not self.sharded or a.numel <= a.tail_offset:
            return
        import torch.distributed as dist
        self._side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(self._side):
            dist.all_reduce(a.G[a.tail_offset:a.numel], op=dist.ReduceOp.SUM, group=self._side_group)
        self._early_pending = True

    def zero_grad(self, set_to_none=True):
        self.arena.begin_step(grads_zeroed=self.zero_grad_in_step and self._stepped)
        if self.lazy is not None:
            self.lazy.counter.zero_()

    _stepped = False
    group = None                 # sharded: the PeerGroup (fuxictr_b200.sharded) that sums a buffer over the ranks

    def step(self):
        """clip + Adam.  A row-sharded step sums one buffer over the ranks midway (the norm term of the
        shards, and the dense gradients unless they are already being summed on the side stream)."""
        for buf in self.step_phases():
            self._sum_over_ranks(buf)

    def _sum_over_ranks(self, buf):
        if self.group is not None:
            self.group.all_reduce_sum(buf)
        else:
            import torch.distributed as dist
            dist.all_reduce(buf, op=dist.ReduceOp.SUM)

    def step_phases(self):
        """The step as a generator: it yields each buffer that has to be summed over the ranks (row-sharded
        runs: once) and finishes the step when resumed.  step() sums through the group; a driver of several
        virtual ranks in one process (sharded.lockstep_steps) sums across them in lock step instead."""
        a = self.arena
        st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
        if not torch.cuda.is_current_stream_capturing():
            self.count_step()
        F2.bump_weight_epoch()        # parameters change through raw pointers: cached 3xTF32 weight splits are stale
        early = self._early
        if early is not None:         # the untouched-granule pass reads step_dev as the step before this one
            torch.cuda.current_stream().wait_event(early[0])
            self._early = None
        self.step_dev.add_(1)
        # Gradients produced by stock autograd ops (parameters our kernels do not own, e.g. Dice's
        # alpha or a Conv1d weight reached through a view) live in p.grad, not in the arena: bring
        # them in.  Kernel-written gradients already alias their arena slot and are skipped.
        if self.grad_allreduce or self.sharded:
            a.join_grads()
        g_base = a.G.data_ptr()
        for p in a.params:
            g = p.grad
            if g is not None and g.data_ptr() != g_base + p._b2_slot.offset * 4:
                a.grad_view(p._b2_slot).copy_(g)
                a.mark_slot(p._b2_slot)
        a.flags_frozen = False
        if self.grad_allreduce:
            import torch.distributed as dist
            dist.all_reduce(a.G, op=dist.ReduceOp.SUM)   # one NCCL collective over the whole arena
            a.G.mul_(1.0 / dist.get_world_size())          # mean over the global batch (rank_model.py:130)
            if a.touched is not None:                      # a granule any rank wrote may now be nonzero here
                dist.all_reduce(a.touched, op=dist.ReduceOp.MAX)
        # The table passes read G only in flagged granules and clear the flags with the gradients: only when
        # the step zeroes G (otherwise the flags just accumulate, and the passes read everything).
        flags = a.touched if (self.zero_grad_in_step and self.lazy is None) else None
        sumsq_ptr = ctypes.c_void_p(0)
        if self.sharded:
            if self.group is not None:
                world = self.group.world
            else:
                import torch.distributed as dist
                world = dist.get_world_size()
            slot = a._G_ext[a.numel:a.numel + 1]               # rides behind the dense slice
            slot.zero_()
            if self.max_norm is not None and a.tail_offset > 0:
                if self.lazy is not None:   # only the enqueued rows carry a gradient: no pass over the shards
                    lz = self.lazy
                    _lib.call("b2_lazy_sumsq", ctypes.c_void_p(lz.tables_dev.data_ptr()), len(lz.tables),
                              ctypes.c_void_p(lz.worklist.data_ptr()), ctypes.c_void_p(lz.counter.data_ptr()),
                              lz.capacity, (a.G.data_ptr() - a.P.data_ptr()) // 4, ctypes.c_void_p(slot.data_ptr()),
                              st)
                elif flags is not None:     # this rank's shard part of ||g||^2
                    _lib.call("b2_sumsq_ex", ctypes.c_void_p(a.G.data_ptr()), a.tail_offset,
                              ctypes.c_void_p(slot.data_ptr()), ctypes.c_void_p(flags.data_ptr()), a.tail_offset, st)
                else:
                    _lib.call("b2_sumsq", ctypes.c_void_p(a.G.data_ptr()), a.tail_offset,
                              ctypes.c_void_p(slot.data_ptr()), st)
            if self._early_pending:
                # the dense gradients are already being summed on the side stream: only the norm scalar here
                yield slot
                torch.cuda.current_stream().wait_stream(self._side)
                self._early_pending = False
            else:
                # ONE sum: dense gradients (to be averaged) + the shard norm term (to be summed)
                yield a._G_ext[a.tail_offset:a.numel + 1]
            dense = a.G[a.tail_offset:]
            if dense.numel() > 0 and not self.dense_prescaled:
                dense.mul_(1.0 / world)                          # mean over the global batch
            if self.max_norm is not None:
                # global norm^2 = sum over ranks of the shard parts + the (replicated) dense part once
                self.sumsq.copy_(slot.view(()))
                if dense.numel() > 0:
                    _lib.call("b2_sumsq", ctypes.c_void_p(dense.data_ptr()), dense.numel(),
                              ctypes.c_void_p(self.sumsq.data_ptr()), st)
                sumsq_ptr = ctypes.c_void_p(self.sumsq.data_ptr())
        elif self.max_norm is not None:
            self.sumsq.zero_()
            if self.lazy is not None:
                lz = self.lazy
                dg = (a.G.data_ptr() - a.P.data_ptr()) // 4
                _lib.call("b2_lazy_sumsq", ctypes.c_void_p(lz.tables_dev.data_ptr()), len(lz.tables),
                          ctypes.c_void_p(lz.worklist.data_ptr()), ctypes.c_void_p(lz.counter.data_ptr()),
                          lz.capacity, dg, ctypes.c_void_p(self.sumsq.data_ptr()), st)
                a.join_grads()
                if a.numel > a.tail_offset:
                    _lib.call("b2_sumsq", ctypes.c_void_p(a.G.data_ptr() + 4 * a.tail_offset),
                              a.numel - a.tail_offset, ctypes.c_void_p(self.sumsq.data_ptr()), st)
            elif flags is not None and a.pending:
                # the table prefix depends only on the front's backward: summed while the MLP's weight-gradient
                # GEMMs still run on their side stream, the dense tail after the join
                _lib.call("b2_sumsq_ex", ctypes.c_void_p(a.G.data_ptr()), a.tail_offset,
                          ctypes.c_void_p(self.sumsq.data_ptr()), ctypes.c_void_p(flags.data_ptr()), a.tail_offset, st)
                a.join_grads()
                _lib.call("b2_sumsq", ctypes.c_void_p(a.G.data_ptr() + 4 * a.tail_offset), a.numel - a.tail_offset,
                          ctypes.c_void_p(self.sumsq.data_ptr()), st)
            elif flags is not None:
                _lib.call("b2_sumsq_ex", ctypes.c_void_p(a.G.data_ptr()), a.numel,
                          ctypes.c_void_p(self.sumsq.data_ptr()), ctypes.c_void_p(flags.data_ptr()), a.tail_offset, st)
            else:
                a.join_grads()
                _lib.call("b2_sumsq", ctypes.c_void_p(a.G.data_ptr()), a.numel,
                          ctypes.c_void_p(self.sumsq.data_ptr()), st)
            sumsq_ptr = ctypes.c_void_p(self.sumsq.data_ptr())
        a.join_grads()
        vp = ctypes.c_void_p
        lo = 0
        if flags is not None and early is not None:
            # tables: the unflagged granules were updated by the side pass; the flagged ones now
            _lib.call("b2_adam_touched", vp(a.P.data_ptr()), vp(a.G.data_ptr()), vp(self.M.data_ptr()),
                      vp(self.V.data_ptr()), a.tail_offset, sumsq_ptr, float(self.max_norm or 0.0), self.lr,
                      self.betas[0], self.betas[1], self.eps, vp(self.step_dev.data_ptr()), vp(flags.data_ptr()), st)
            lo = a.tail_offset
        elif flags is not None:
            # tables: G loaded (and zeroed, and its flag cleared) only in the granules a backward wrote
            _lib.call("b2_adam_step_ex", vp(a.P.data_ptr()), vp(a.G.data_ptr()), vp(self.M.data_ptr()),
                      vp(self.V.data_ptr()), a.tail_offset, sumsq_ptr, float(self.max_norm or 0.0), self.lr,
                      self.betas[0], self.betas[1], self.eps, vp(self.step_dev.data_ptr()), 1,
                      vp(flags.data_ptr()), a.tail_offset, st)
            lo = a.tail_offset
        if self.lazy is not None:
            _lib.call("b2_adam_sched", vp(self.step_dev.data_ptr()), self.lr, self.betas[0], self.betas[1],
                      vp(self.sched.data_ptr()), self.sched.shape[0], st)
            # tables: only the rows this step touched (missed zero-gradient steps are replayed)
            lz = self.lazy
            lo = a.tail_offset
            dg = (a.G.data_ptr() - a.P.data_ptr()) // 4
            dm = (self.M.data_ptr() - a.P.data_ptr()) // 4
            dv = (self.V.data_ptr() - a.P.data_ptr()) // 4
            _lib.call("b2_lazy_adam_step", vp(lz.tables_dev.data_ptr()), len(lz.tables), vp(lz.worklist.data_ptr()),
                      vp(lz.counter.data_ptr()), lz.capacity, dg, dm, dv, vp(lz.last_step.data_ptr()),
                      vp(self.sched.data_ptr()), vp(self.step_dev.data_ptr()), sumsq_ptr,
                      float(self.max_norm or 0.0), self.betas[0], self.betas[1], self.eps, st)
        n = a.numel - lo
        if n > 0 and self.lazy is not None:     # same scalars as the lazy replay: read them from the table
            _lib.call("b2_adam_step_sched", vp(a.P.data_ptr() + 4 * lo), vp(a.G.data_ptr() + 4 * lo),
                      vp(self.M.data_ptr() + 4 * lo), vp(self.V.data_ptr() + 4 * lo), n, sumsq_ptr,
                      float(self.max_norm or 0.0), self.betas[0], self.betas[1], self.eps,
                      vp(self.step_dev.data_ptr()), vp(self.sched.data_ptr()),
                      1 if self.zero_grad_in_step else 0, st)
        elif n > 0:                             # dense pass: the two per-step scalars are computed in-kernel
            _lib.call("b2_adam_step", vp(a.P.data_ptr() + 4 * lo), vp(a.G.data_ptr() + 4 * lo),
                      vp(self.M.data_ptr() + 4 * lo), vp(self.V.data_ptr() + 4 * lo), n, sumsq_ptr, float(self.max_norm or 0.0), self.lr,
                      self.betas[0], self.betas[1], self.eps, vp(self.step_dev.data_ptr()),
                      1 if self.zero_grad_in_step else 0, st)
        self._stepped = True

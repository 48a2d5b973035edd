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
        with torch.no_grad():
            for p, o in slots:
                dst = self.P[o:o + p.numel()].view(p.shape)
                dst.copy_(p.data)
                p.data = dst
                p._b2_slot = _Slot(self, o, p.numel(), tuple(p.shape))
                p.grad = None

    def grad_view(self, slot):
        return self.G[slot.offset:slot.offset + slot.numel].view(slot.shape)

    def begin_step(self, grads_zeroed):
        """Call once per training step before backward. `grads_zeroed`: G is already all-zero
        (e.g. the previous fused Adam step cleared it); otherwise sparse-written grads
        (embedding tables) are zero-filled lazily by the kernels' wrappers."""
        self.step_id += 1
        self.grads_are_zero = bool(grads_zeroed)
        for p in self.params:
            p.grad = None

    def zero_grads(self):
        self.G.zero_()


class LazyTables(object):
    """Bookkeeping of the lazily evaluated tables (see b2_lazy_ctx in include/fuxictr_b200.h):
    per-row `last_step`, the per-step worklist, the schedule table shared with the dense pass."""

    SCHED_LEN = 1 << 20   # optimizer steps the schedule table can hold

    def __init__(self, arena, tables):
        self.arena = arena
        self.tables = list(tables)
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

    def ctx_for(self, plan, lr_plan, emb_tables, lr_tables):
        key = (id(plan), id(lr_plan))
        ctx = self._ctx_cache.get(key)
        if ctx is None:
            opt, a = self.opt, self.arena
            ctx = _lib.b2_lazy_ctx()
            ctx.last_step, ctx.sched = self.last_step.data_ptr(), self.sched.data_ptr()
            ctx.step_dev, ctx.mark = opt.step_dev.data_ptr(), self.mark.data_ptr()
            ctx.worklist, ctx.counter = self.worklist.data_ptr(), self.counter.data_ptr()
            ctx.delta_m = (opt.M.data_ptr() - a.P.data_ptr()) // 4
            ctx.delta_v = (opt.V.data_ptr() - a.P.data_ptr()) // 4
            # the same float32 roundings as make_const() in csrc/lazy_adam.cu / adam_kernel in dense.cu:
            # beta is rounded to fp32 FIRST, then 1 - beta is taken in double and rounded again
            b1, b2 = float(np.float32(opt.betas[0])), float(np.float32(opt.betas[1]))
            ctx.w1, ctx.beta2 = float(np.float32(1.0 - b1)), b2
            ctx.w2, ctx.eps = float(np.float32(1.0 - b2)), opt.eps
            ctx.worklist_capacity = self.capacity
            for i, f in enumerate(plan.fields):
                ctx.grow_emb[i] = emb_tables[f.table_slot]._b2_grow_base
            if lr_plan is not None:
                for i, f in enumerate(lr_plan.fields):
                    ctx.grow_lr[i] = lr_tables[f.table_slot]._b2_grow_base
            self._ctx_cache[key] = ctx
        return ctx

    def materialize(self):
        """Bring every row up to date (before reading the tables outside the kernels)."""
        opt, a = self.opt, self.arena
        st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
        _lib.call("b2_lazy_materialize", ctypes.c_void_p(self.tables_dev.data_ptr()), len(self.tables),
                  self.total_rows, (opt.M.data_ptr() - a.P.data_ptr()) // 4,
                  (opt.V.data_ptr() - a.P.data_ptr()) // 4, ctypes.c_void_p(self.last_step.data_ptr()),
                  ctypes.c_void_p(self.sched.data_ptr()), ctypes.c_void_p(opt.step_dev.data_ptr()),
                  opt.betas[0], opt.betas[1], opt.eps, st)


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

    def enable_lazy(self, tables):
        """Evaluate the dense Adam semantics of `tables` (the arena's leading parameters) lazily."""
        self.sched = torch.zeros((LazyTables.SCHED_LEN, 2), dtype=torch.float32, device=self.arena.P.device)
        self.lazy = LazyTables(self.arena, tables)
        self.lazy.opt = self
        self.lazy.sched = self.sched          # one schedule table for the dense and the lazy kernels
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

    def step(self):
        a = self.arena
        st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
        if not torch.cuda.is_current_stream_capturing():
            self.count_step()
        F2.bump_weight_epoch()        # parameters change through raw pointers: cached 3xTF32 weight splits are stale
        self.step_dev.add_(1)
        # Gradients produced by stock autograd ops (parameters our kernels do not own, e.g. Dice's
        # alpha or a Conv1d weight reached through a view) live in p.grad, not in the arena: bring
        # them in.  Kernel-written gradients already alias their arena slot and are skipped.
        g_base = a.G.data_ptr()
        for p in a.params:
            g = p.grad
            if g is not None and g.data_ptr() != g_base + p._b2_slot.offset * 4:
                a.grad_view(p._b2_slot).copy_(g)
        if self.grad_allreduce:
            import torch.distributed as dist
            dist.all_reduce(a.G, op=dist.ReduceOp.SUM)   # one NCCL collective over the whole arena
            a.G.mul_(1.0 / dist.get_world_size())          # mean over the global batch (rank_model.py:130)
        sumsq_ptr = ctypes.c_void_p(0)
        if self.sharded:
            import torch.distributed as dist
            world = dist.get_world_size()
            slot = a._G_ext[a.numel:a.numel + 1]               # rides behind the dense slice
            slot.zero_()
            if self.max_norm is not None and a.tail_offset > 0:
                _lib.call("b2_sumsq", ctypes.c_void_p(a.G.data_ptr()), a.tail_offset,
                          ctypes.c_void_p(slot.data_ptr()), st)   # this rank's shard part of ||g||^2
            if self._early_pending:
                # the dense gradients are already being summed on the side stream: only the norm scalar here
                dist.all_reduce(slot, op=dist.ReduceOp.SUM)
                torch.cuda.current_stream().wait_stream(self._side)
                self._early_pending = False
            else:
                # ONE collective: dense gradients (to be averaged) + the shard norm term (to be summed)
                dist.all_reduce(a._G_ext[a.tail_offset:a.numel + 1], op=dist.ReduceOp.SUM)
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
                if a.numel > a.tail_offset:
                    _lib.call("b2_sumsq", ctypes.c_void_p(a.G.data_ptr() + 4 * a.tail_offset),
                              a.numel - a.tail_offset, ctypes.c_void_p(self.sumsq.data_ptr()), st)
            else:
                _lib.call("b2_sumsq", ctypes.c_void_p(a.G.data_ptr()), a.numel,
                          ctypes.c_void_p(self.sumsq.data_ptr()), st)
            sumsq_ptr = ctypes.c_void_p(self.sumsq.data_ptr())
        vp = ctypes.c_void_p
        lo = 0
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
            _lib.call("b2_adam_step", vp(a.P.data_ptr()), vp(a.G.data_ptr()), vp(self.M.data_ptr()),
                      vp(self.V.data_ptr()), n, sumsq_ptr, float(self.max_norm or 0.0), self.lr,
                      self.betas[0], self.betas[1], self.eps, vp(self.step_dev.data_ptr()),
                      1 if self.zero_grad_in_step else 0, st)
        self._stepped = True

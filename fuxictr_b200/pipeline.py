"""Host -> HBM input path and the captured training step (SURVEY.md 8f row 1).

The reference moves a batch to the GPU feature by feature: `BaseModel.get_inputs`
(fuxictr/pytorch/models/rank_model.py:169-189) calls `.to(device)` on every column view that
`BatchCollator.__call__` (fuxictr/pytorch/dataloaders/npz_dataloader.py:111-125) cut out of ONE
(B, input_length + n_labels) matrix, i.e. F small strided H2D copies plus F casts per step.
Here the matrix travels once:

    pinned host matrix --(copy stream, async)--> staging[k % depth] in HBM
                       --(compute stream, 8*B*W-byte D2D)--> the graph's static input
                       --> captured fused_train_step (fused front reads ids straight from it)
                       --> 4-byte loss D2H into pinned memory

The H2D of step k+1 overlaps the replay of step k (the front kernels read the ids again near the
end of backward, so the static input itself cannot be overwritten early: hence the staging ring).
Nothing here computes: it is stream/event plumbing around the C-ABI kernels.
"""
import torch

from . import functional as F2


class TrainPipeline(object):
    """model: a fuxictr_b200.zoo.RankModel after use_fused_optimizer().
    batch_rows / matrix_width / dtype: the collator's matrix, e.g. (4096, 40) float64 for
    Criteo-shape DeepFM.  graph=True captures the whole step (forward, backward, clip, Adam) into
    one CUDA graph; graph=False runs it eagerly (debugging, models with host-side control flow)."""

    def __init__(self, model, batch_rows, matrix_width, dtype=torch.float64, graph=True, depth=2,
                 capture_warmup=3):
        if not torch.cuda.is_available():
            raise RuntimeError("TrainPipeline needs a CUDA device (there is no CPU path)")
        if getattr(model, "_fused_optimizer", None) is None:
            raise RuntimeError("call model.use_fused_optimizer() before building a TrainPipeline")
        self.model = model
        dev = model.device
        self.shape = (int(batch_rows), int(matrix_width))
        self.dtype = dtype
        self.static_in = torch.zeros(self.shape, dtype=dtype, device=dev)
        self._views = self._input_views()
        self._stage = [torch.empty_like(self.static_in) for _ in range(depth)]
        self._pinned = [None] * depth           # lazily allocated: only for callers with pageable matrices
        self._h2d_done = [torch.cuda.Event() for _ in range(depth)]
        self._consumed = [torch.cuda.Event() for _ in range(depth)]
        self._copy_stream = torch.cuda.Stream(device=dev)
        self._k = 0
        self.loss_host = torch.zeros((), dtype=torch.float32).pin_memory()
        self._loss_ready = torch.cuda.Event()
        self.graph, self.loss_dev = None, None
        self.h2d_bytes_per_step = self.static_in.numel() * self.static_in.element_size()
        self.d2h_bytes_per_step = 4
        if graph:
            self._capture(capture_warmup)

    def _input_views(self):
        """The batch dict the captured step reads: every entry aliases static_in."""
        return self.model.feature_map.batch_views(self.static_in)

    # -- capture ---------------------------------------------------------------------------------
    def _eager(self):
        return self.model.fused_train_step(self._views)

    def capture(self, warmup=3):
        """Capture the step into a CUDA graph now (what graph=True does in the constructor)."""
        self._capture(warmup)

    def _capture(self, warmup):
        """Warm-up steps run on a side stream (they are REAL optimizer steps on whatever static_in
        holds: load a valid batch with `prime()` first if the trajectory matters)."""
        self.loss_dev = None            # a live loss of an earlier eager step pins its autograd graph (and the
        side = torch.cuda.Stream()      # AccumulateGrad nodes' stream) and would invalidate the capture
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(warmup):
                self._eager()
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph):
            self.loss_dev = self._eager().detach()

    def prime(self, matrix):
        """Put a valid batch into the static input (before capture warm-up / first replay)."""
        self.static_in.copy_(matrix)

    # -- one step --------------------------------------------------------------------------------
    def _run(self):
        if self.graph is not None:
            self.model._fused_optimizer.count_step()      # a replay is one optimizer step (host-side bound check)
            F2.bump_weight_epoch()                        # ... that moved the weights behind torch's back
            self.graph.replay()
            return self.loss_dev
        self.loss_dev = self._eager().detach()
        return self.loss_dev

    def step_device(self, dev_matrix):
        """Batch already resident in HBM: D2D into the static input, one replay.  Returns the loss
        as a device tensor (valid until the next step)."""
        self.static_in.copy_(dev_matrix, non_blocking=True)
        return self._run()

    def step(self, host_matrix):
        """Batch in host memory, laid out as the collator yields it.  Fully asynchronous: returns
        after enqueueing the H2D (copy stream), the replay and the loss D2H; read the loss with
        `loss()`.  A pinned `host_matrix` is copied from directly and must stay untouched until
        this step's H2D finished — guaranteed once `depth` further step() calls were entered, or after
        `wait_inputs()`; a pageable one is staged through the pipeline's own pinned ring first."""
        if tuple(host_matrix.shape) != self.shape or host_matrix.dtype != self.dtype:
            raise ValueError("batch matrix %s %s does not match the pipeline's %s %s"
                             % (tuple(host_matrix.shape), host_matrix.dtype, self.shape, self.dtype))
        self._load(host_matrix)
        return self._emit(self._run())

    def _load(self, host_matrix):
        """H2D of the first rows of static_in through the staging ring on the copy stream."""
        rows = host_matrix.shape[0]
        d = self._k % len(self._stage)
        self._k += 1
        # Host throttle: at most `depth` H2D copies are ever outstanding, so a caller that feeds pinned
        # ring buffers (dataloader.py) knows the copy of batch k-depth has left its source when step(k)
        # is entered.  The event is normally long complete; this costs a microsecond.
        self._h2d_done[d].synchronize()
        if not host_matrix.is_pinned():
            if self._pinned[d] is None:
                self._pinned[d] = torch.empty(self.shape, dtype=self.dtype).pin_memory()
            self._pinned[d][:rows].copy_(host_matrix)
            host_matrix = self._pinned[d][:rows]
        compute = torch.cuda.current_stream()
        cs = self._copy_stream
        cs.wait_event(self._consumed[d])         # staging[d] was drained by the step that used it last
        with torch.cuda.stream(cs):
            self._stage[d][:rows].copy_(host_matrix, non_blocking=True)
            self._h2d_done[d].record(cs)
        compute.wait_event(self._h2d_done[d])
        self.static_in[:rows].copy_(self._stage[d][:rows], non_blocking=True)
        self._consumed[d].record(compute)

    def _emit(self, loss):
        """Queue the 4-byte loss D2H into pinned memory behind the step."""
        self.loss_host.copy_(loss.detach(), non_blocking=True)
        self._loss_ready.record(torch.cuda.current_stream())
        return self.loss_host

    def wait_inputs(self):
        """Block the host until every H2D issued so far has left its pinned source."""
        for ev in self._h2d_done:
            ev.synchronize()

    def loss(self):
        """The most recent step()'s loss as a Python float (waits for that step)."""
        self._loss_ready.synchronize()
        return float(self.loss_host)


class LongCTRPipeline(TrainPipeline):
    """The LongCTR training step (ETA, SDIM, SIM, TWIN, MIRRN) fed by a longctr_data.LongCTRDataLoader:

        pinned batch matrix --(copy stream)--> staging ring --> static_in
                            --> b2_longctr_collate into the triple (batch_dict, item_dict, mask)
                            --> fused_train_step --> 4-byte loss D2H

    Only the batch matrix travels; the histories and item columns stay in the loader's store in HBM.  Feed it
    `step(matrix, L)` with what `loader.matrices()` yields.  With graph=True the full-batch shape at L = max_len, the
    shape of nearly every batch of real data, is captured after the first two steps of that shape have run eagerly
    (they are steps of the trajectory: capture adds no optimizer step), and replayed from then on.  Every other shape
    (the last, partial batch; batches whose longest history is shorter than max_len) runs eagerly into freshly
    allocated triples: one graph per L would each hold its own long-sequence activations.  Eager steps run on a side
    stream, as capture warm-up must."""

    def __init__(self, model, loader, graph=True, depth=2):
        self.loader = loader
        self.max_len = loader.max_len
        host = loader.matrix
        super(LongCTRPipeline, self).__init__(model, loader.batch_size, host.shape[1], dtype=host.dtype, graph=False,
                                              depth=depth)
        self._want_graph = bool(graph)
        self._full_eager = 0
        self.last_loss = None
        self._side = torch.cuda.Stream(device=model.device)
        B, C = self.shape[0], len(loader.item_columns)
        self._mask = torch.zeros((B, self.max_len), dtype=torch.float32, device=model.device)
        self._items = torch.zeros((C, B * (self.max_len + 1)), dtype=torch.int64, device=model.device)

    def _input_views(self):
        return None             # the triple is built per step, for that step's shape

    def _triple(self, rows, L):
        """Collate static_in's first rows into a triple (the static buffers at the captured shape)."""
        full = rows == self.shape[0] and L == self.max_len
        return self.loader.collate(self.static_in[:rows], L, *((self._mask, self._items) if full else ()))

    def _eager(self, rows=None, L=None):
        rows = self.shape[0] if rows is None else rows
        return self.model.fused_train_step(self._triple(rows, self.max_len if L is None else L))

    def _eager_side(self, rows, L):
        compute = torch.cuda.current_stream()
        self._side.wait_stream(compute)
        with torch.cuda.stream(self._side):
            loss = self._eager(rows, L).detach()
        compute.wait_stream(self._side)
        return loss

    def _capture_full(self):
        torch.cuda.synchronize()
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph):
            self.loss_dev = self._eager().detach()

    def step(self, host_matrix, L):
        """One training step on a batch of `host_matrix.shape[0] <= batch_size` rows whose histories are padded to
        L <= max_len.  Asynchronous like TrainPipeline.step; read the loss with `loss()`."""
        rows = host_matrix.shape[0]
        if host_matrix.dim() != 2 or host_matrix.shape[1] != self.shape[1] or host_matrix.dtype != self.dtype or \
                not 1 <= rows <= self.shape[0]:
            raise ValueError("batch matrix %s %s does not fit the pipeline's %s %s"
                             % (tuple(host_matrix.shape), host_matrix.dtype, self.shape, self.dtype))
        if not 0 <= int(L) <= self.max_len:
            raise ValueError("L = %s outside [0, max_len = %d]" % (L, self.max_len))
        self._load(host_matrix)
        full = rows == self.shape[0] and L == self.max_len
        if full and self.graph is None and self._want_graph and self._full_eager >= 2:
            self._capture_full()
        if full and self.graph is not None:
            loss = self._run()                  # loss_dev: the graph's output
        else:
            loss = self._eager_side(rows, int(L))
            self._full_eager += int(full)
        self.last_loss = loss                   # the device loss of this step, valid until the next
        return self._emit(loss)

    def epoch(self):
        """One pass over the loader; returns the step losses as floats, read with one synchronise at the end."""
        losses = torch.empty(len(self.loader), dtype=torch.float32, device=self.model.device)
        for k, (mat, L) in enumerate(self.loader.matrices()):
            self.step(mat, L)
            losses[k].copy_(self.last_loss)
        return losses.tolist()

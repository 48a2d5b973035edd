"""Matrix-first twins of fuxictr.pytorch.dataloaders (SURVEY.md 8f row 4, host side of the input path).

The reference's loaders hold a split as ONE (N, input_length + n_labels) numpy matrix
(`np.column_stack` over features + labels: npz_dataloader.py:63-66, parquet_dataloader.py:65-74),
hand single ROWS to torch's DataLoader, re-stack them with `default_collate`, and slice the batch
into per-feature column views (`BatchCollator`, npz_dataloader.py:111-125).  The H100 input path
(pipeline.TrainPipeline) wants exactly that (B, W) matrix, pinned, before it is sliced — so these
loaders skip the row-by-row round trip:

  * the split lives in one pinned host tensor; an unshuffled batch is a zero-copy row slice;
  * a shuffled batch is one `index_select` into a pinned ring slot, prefetched by a thread; the
    permutation is the one `DataLoader(shuffle=True)` would draw from the global torch RNG
    (base seed, then sampler seed, then `randperm`), so a seeded reference run sees identical batches;
  * block ("streaming") loaders read one part file at a time in the prefetch thread and emit batches
    that run across block boundaries, like the reference's chained datapipe with one worker.

Iterating a loader yields the reference's batch dict (name -> column views of the batch matrix;
`RankModel._batch_matrix` recovers the matrix from any view); `.matrices()` yields the matrices
themselves for `TrainPipeline.step`.  Same constructor arguments, `num_samples`, `num_blocks`,
`num_batches` and `len()` as the reference classes.  Pure host code: numpy / pandas / torch CPU.
"""
import glob
import logging
import os
import queue
import threading

import numpy as np
import torch


# ----------------------------------------------------------------------------------------------
# file -> (N, W) matrix
# ----------------------------------------------------------------------------------------------
def _all_columns(feature_map):
    return list(feature_map.features.keys()) + list(feature_map.labels)


def load_npz_matrix(feature_map, data_path):
    """NpzDataset.load_data (npz_dataloader.py:53-66)."""
    blob = np.load(data_path)
    return np.column_stack([blob[col] for col in _all_columns(feature_map)])


def load_parquet_matrix(feature_map, data_path):
    """ParquetDataset.load_data (parquet_dataloader.py:56-74): list-valued (sequence) columns
    become (N, L) blocks of the matrix."""
    import pandas as pd
    df = pd.read_parquet(data_path)
    arrays = []
    for col in _all_columns(feature_map):
        series = df[col]
        arrays.append(np.array(series.to_list()) if series.dtype == "object" else series.to_numpy())
    return np.column_stack(arrays)


def _to_host_tensor(darray, pin):
    t = torch.from_numpy(np.ascontiguousarray(darray))
    if pin == "auto":
        pin = torch.cuda.is_available()
    return t.pin_memory() if pin else t


def torch_loader_permutation(n):
    """The order `DataLoader(dataset, shuffle=True)` visits n rows in, drawn from the global torch
    RNG exactly as torch does: `_BaseDataLoaderIter.__init__` takes one int64 for the workers' base
    seed, then `RandomSampler.__iter__` takes one for its own generator and calls `randperm`."""
    torch.empty((), dtype=torch.int64).random_()
    seed = int(torch.empty((), dtype=torch.int64).random_().item())
    gen = torch.Generator()
    gen.manual_seed(seed)
    return torch.randperm(n, generator=gen)


class _Prefetcher(object):
    """Runs `producer()` (a generator) in a thread, `depth` items ahead."""
    _END = object()

    def __init__(self, producer, depth):
        self._q = queue.Queue(maxsize=depth)
        self._err = None
        self._stop = threading.Event()
        self._t = threading.Thread(target=self._run, args=(producer,), daemon=True)
        self._t.start()

    def _run(self, producer):
        try:
            for item in producer():
                while not self._stop.is_set():
                    try:
                        self._q.put(item, timeout=0.1)
                        break
                    except queue.Full:
                        continue
                if self._stop.is_set():
                    return
        except BaseException as exc:     # surfaced in the consumer thread
            self._err = exc
        finally:
            while not self._stop.is_set():
                try:
                    self._q.put(self._END, timeout=0.1)
                    break
                except queue.Full:
                    continue

    def __iter__(self):
        try:
            while True:
                item = self._q.get()
                if item is self._END:
                    if self._err is not None:
                        raise self._err
                    return
                yield item
        finally:
            self._stop.set()


class _MatrixLoaderBase(object):
    """Shared iteration protocol.  Ring sizing: a ring slot handed out for batch k is refilled for
    batch k + ring; TrainPipeline.step keeps at most `depth` (2) H2D copies outstanding, the
    prefetcher runs at most `prefetch` batches ahead, so ring >= prefetch + depth + 2 guarantees a
    slot's H2D has finished before the slot is overwritten."""
    prefetch = 2
    ring = 6
    _ring_backed = True

    def __init__(self, feature_map, batch_size, pin):
        self.feature_map = feature_map
        self.batch_size = int(batch_size)
        self._pin = pin

    def __len__(self):
        return self.num_batches

    def __iter__(self):
        """The reference protocol: one batch dict per step.  Ring-backed batches (shuffled or block
        loaders) are cloned so a consumer may keep them, as it may with the reference's loaders;
        `matrices()` hands out the pinned ring slots themselves and is what TrainPipeline wants."""
        for mat in self.matrices():
            yield self.feature_map.batch_dict(mat.clone() if self._ring_backed else mat)

    def _ring_slots(self, width, dtype):
        return [_to_host_tensor(np.empty((self.batch_size, width), dtype=dtype), self._pin)
                for _ in range(self.ring)]


# ----------------------------------------------------------------------------------------------
# In-memory splits (NpzDataLoader / ParquetDataLoader)
# ----------------------------------------------------------------------------------------------
class MatrixDataLoader(_MatrixLoaderBase):
    """One file, whole split resident in (pinned) host memory.

    shard=(rank, world) is the data-parallel view for one-process-per-GPU runs (SURVEY.md 8e; the
    reference is single-device): a GLOBAL batch is `batch_size * world` rows, taken in exactly the
    order the unsharded loader with that batch size would take them, and this rank gets rows
    [rank*batch_size, (rank+1)*batch_size) of it.  Every rank must seed the torch RNG identically so
    all draw the same permutation.  An incomplete last global batch is dropped (drop_last=True, the
    default when sharded: the captured step has a fixed shape) or split as evenly as its rows allow."""

    def __init__(self, feature_map, darray, batch_size=32, shuffle=False, pin="auto", shard=None,
                 drop_last=None):
        super(MatrixDataLoader, self).__init__(feature_map, batch_size, pin)
        # shuffled batches leave through the pinned ring slots (index_select into them), so page-locking
        # the whole split buys nothing there; unshuffled batches are zero-copy slices and want it pinned
        self.matrix = _to_host_tensor(darray, False if (shuffle and pin == "auto") else pin)
        self.shuffle = shuffle
        self.rank, self.world = (0, 1) if shard is None else (int(shard[0]), int(shard[1]))
        if not 0 <= self.rank < self.world:
            raise ValueError("shard=(rank, world) needs 0 <= rank < world, got %s" % (shard,))
        self.drop_last = (self.world > 1) if drop_last is None else bool(drop_last)
        self.num_samples = self.matrix.shape[0]
        self.num_blocks = 1
        gb = self.batch_size * self.world
        self.num_batches = self.num_samples // gb if self.drop_last else int(np.ceil(self.num_samples * 1.0 / gb))
        self._slots = None
        self._ring_backed = bool(shuffle)

    def _spans(self):
        """(lo, hi) row ranges, in visiting order, of this rank's share of each global batch."""
        n, B, gb = self.num_samples, self.batch_size, self.batch_size * self.world
        for g0 in range(0, n, gb):
            rows = min(gb, n - g0)
            if rows < gb and self.drop_last:
                return
            if rows == gb:
                yield g0 + self.rank * B, g0 + (self.rank + 1) * B
            else:       # incomplete tail kept: split its rows evenly, earlier ranks take the remainder
                base, extra = divmod(rows, self.world)
                lo = self.rank * base + min(self.rank, extra)
                yield g0 + lo, g0 + lo + base + (1 if self.rank < extra else 0)

    def matrices(self):
        if not self.shuffle:
            for lo, hi in self._spans():
                yield self.matrix[lo:hi]                # zero-copy slice of the pinned split
            return
        perm = torch_loader_permutation(self.num_samples)   # on the caller's thread: global RNG order as torch's
        if self._slots is None:
            self._slots = self._ring_slots(self.matrix.shape[1], self.matrix.numpy().dtype)

        def produce():
            for k, (lo, hi) in enumerate(self._spans()):
                idx = perm[lo:hi]
                slot = self._slots[k % self.ring][:idx.numel()]
                torch.index_select(self.matrix, 0, idx, out=slot)
                yield slot
        for mat in _Prefetcher(produce, self.prefetch):
            yield mat


class NpzDataLoader(MatrixDataLoader):
    """fuxictr.pytorch.dataloaders.NpzDataLoader (npz_dataloader.py:69-97).  num_workers is accepted
    and ignored: there is no per-row work left to parallelise."""

    def __init__(self, feature_map, data_path, batch_size=32, shuffle=False, num_workers=1, pin="auto", shard=None,
                 drop_last=None, **kwargs):
        if not data_path.endswith(".npz"):
            data_path += ".npz"
        super(NpzDataLoader, self).__init__(feature_map, load_npz_matrix(feature_map, data_path), batch_size=batch_size,
                                           shuffle=shuffle, pin=pin, shard=shard, drop_last=drop_last)


class ParquetDataLoader(MatrixDataLoader):
    """fuxictr.pytorch.dataloaders.ParquetDataLoader (parquet_dataloader.py:77-106)."""

    def __init__(self, feature_map, data_path, batch_size=32, shuffle=False, num_workers=1, pin="auto", shard=None,
                 drop_last=None, **kwargs):
        if not data_path.endswith(".parquet"):
            data_path += ".parquet"
        super(ParquetDataLoader, self).__init__(feature_map, load_parquet_matrix(feature_map, data_path), batch_size=batch_size,
                                           shuffle=shuffle, pin=pin, shard=shard, drop_last=drop_last)


# ----------------------------------------------------------------------------------------------
# Block ("streaming") splits (NpzBlockDataLoader / ParquetBlockDataLoader)
# ----------------------------------------------------------------------------------------------
class BlockMatrixDataLoader(_MatrixLoaderBase):
    """A directory of part files read one at a time.  Unshuffled order = the reference's chained
    datapipe with a single worker (npz_block_dataloader.py:52-80): blocks sorted by name, rows in
    file order, batches running across block boundaries.  shuffle=True mixes every block with the
    `buffer_size` rows held back from the previous ones — the role of the reference's
    `datapipe.shuffle(buffer_size)`; the permutation comes from this loader's own generator (seeded
    from the global torch RNG), not from torch's datapipe internals, so shuffled block runs match the
    reference in distribution, not row for row."""
    _pattern = "*"

    def __init__(self, feature_map, data_path, split="train", batch_size=32, shuffle=False, num_workers=1,
                 buffer_size=100000, pin="auto", **kwargs):
        super(BlockMatrixDataLoader, self).__init__(feature_map, batch_size, pin)
        if not data_path.endswith(self._pattern[1:]):
            data_path = os.path.join(data_path, self._pattern)
        self.data_blocks = sorted(glob.glob(data_path))
        assert len(self.data_blocks) > 0, "invalid data_path: %s" % data_path
        self.num_blocks = len(self.data_blocks)
        self.shuffle, self.buffer_size = shuffle, int(buffer_size)
        self.num_samples = sum(self._block_rows(p) for p in self.data_blocks)
        self.num_batches = int(np.ceil(self.num_samples / self.batch_size))

    def _load(self, path):
        raise NotImplementedError

    def _block_rows(self, path):
        raise NotImplementedError

    def matrices(self):
        B = self.batch_size
        seed = int(torch.empty((), dtype=torch.int64).random_().item()) if self.shuffle else 0
        state = {"slots": None}

        def emit(rows, k):
            if state["slots"] is None:
                state["slots"] = self._ring_slots(rows.shape[1], rows.dtype)
            slot = state["slots"][k % self.ring][:rows.shape[0]]
            slot.copy_(torch.from_numpy(rows))
            return slot

        def produce():
            rng = np.random.default_rng(seed)
            pool, k = None, 0               # rows read but not yet emitted
            # shuffle: every new block is merged into the pool and the pool is permuted once (O(pool)
            # per block, not per batch); batches leave from the front while at least buffer_size rows
            # stay behind to mix with the next block.
            hold = self.buffer_size if self.shuffle else 0
            for path in self.data_blocks:
                block = self._load(path)
                pool = block if pool is None or pool.shape[0] == 0 else np.concatenate([pool, block])
                if self.shuffle:
                    pool = pool[rng.permutation(pool.shape[0])]
                full = max(pool.shape[0] - hold, 0) // B * B
                for lo in range(0, full, B):
                    yield emit(pool[lo:lo + B], k)
                    k += 1
                pool = pool[full:]
            if pool is not None:
                for lo in range(0, pool.shape[0], B):
                    yield emit(pool[lo:lo + B], k)
                    k += 1
        for mat in _Prefetcher(produce, self.prefetch):
            yield mat


class NpzBlockDataLoader(BlockMatrixDataLoader):
    """fuxictr.pytorch.dataloaders.NpzBlockDataLoader (npz_block_dataloader.py:83-150)."""
    _pattern = "*.npz"

    def _load(self, path):
        return load_npz_matrix(self.feature_map, path)

    def _block_rows(self, path):
        return np.load(path)[self.feature_map.labels[0]].shape[0]


class ParquetBlockDataLoader(BlockMatrixDataLoader):
    """fuxictr.pytorch.dataloaders.ParquetBlockDataLoader (parquet_block_dataloader.py:91-160); row
    counts come from the parquet footer (pyarrow) instead of a polars scan."""
    _pattern = "*.parquet"

    def _load(self, path):
        return load_parquet_matrix(self.feature_map, path)

    def _block_rows(self, path):
        import pyarrow.parquet as pq
        return pq.ParquetFile(path).metadata.num_rows


# ----------------------------------------------------------------------------------------------
# RankDataLoader (rank_dataloader.py:24-96)
# ----------------------------------------------------------------------------------------------
class RankDataLoader(object):
    """fuxictr.pytorch.dataloaders.RankDataLoader (rank_dataloader.py:24-96): picks the loader class
    from (data_format, streaming) — or takes `data_loader=` — and builds the generators `stage` needs.
    Training data is shuffled if asked; validation and test never are."""
    _LOADERS = {("npz", False): NpzDataLoader, ("npz", True): NpzBlockDataLoader,
                ("parquet", False): ParquetDataLoader, ("parquet", True): ParquetBlockDataLoader}

    def __init__(self, feature_map, stage="both", train_data=None, valid_data=None, test_data=None,
                 batch_size=32, shuffle=True, streaming=False, data_format="npz", **kwargs):
        loader_cls = kwargs.get("data_loader") or \
            self._LOADERS[("npz" if data_format == "npz" else "parquet", bool(streaming))]
        self.stage = stage
        wanted = {"train": stage in ("both", "train") and train_data is not None,
                  "valid": stage in ("both", "train") and bool(valid_data),
                  "test": stage in ("both", "test") and bool(test_data)}
        paths = {"train": train_data, "valid": valid_data, "test": test_data}
        gens = {}
        for split in ("train", "valid", "test"):
            gens[split] = None
            if wanted[split]:
                gens[split] = loader_cls(feature_map, paths[split], split=split, batch_size=batch_size,
                                         shuffle=(shuffle and split == "train"), **kwargs)
                logging.info("%s samples: total/%d, blocks/%d", split, gens[split].num_samples,
                             gens[split].num_blocks)
        self.train_gen, self.valid_gen, self.test_gen = gens["train"], gens["valid"], gens["test"]

    def make_iterator(self):
        """(train, valid) for stage "train", test for "test", all three otherwise."""
        by_stage = {"train": (self.train_gen, self.valid_gen), "test": self.test_gen}
        return by_stage.get(self.stage, (self.train_gen, self.valid_gen, self.test_gen))

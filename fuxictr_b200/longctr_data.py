"""The LongCTR input path (model_zoo/LongCTR/longctr_dataloader.py) with the user histories and item features in HBM.

The reference's `BatchCollator` builds every batch's triple (batch_dict, item_dict, mask) on the CPU: it pads each
sample's history `full_seq[user_index][:seq_len]` with keras `pad_sequences(maxlen=L, value=0, padding=p,
truncating=p)`, looks up B (L + 1) rows of item_info with `iloc` (positional) and hands the model int64 tensors that
`get_inputs` copies to the device one feature at a time.  At B 4096, L 1024 and three item columns that is 117 MB of
H2D per batch.  Here:

  * `LongCTRStore` holds every user's full history (CSR: int64 offsets, int32 item ids) and the item columns (an
    (N_items, C) int32 matrix) in HBM, loaded once and checked once;
  * per batch only the batch matrix travels (B rows of the data file's columns);
  * one kernel (`b2_longctr_collate`) writes the padded histories' item columns and the mask, element for element
    what the reference's collator writes.

`LongCTRDataLoader` takes the reference's constructor and yields the triple on the device; `matrices()` yields the
pinned host matrices with their L for `pipeline.LongCTRPipeline`.
"""
import collections

import numpy as np
import torch

from . import _lib
from .dataloader import _MatrixLoaderBase, _Prefetcher, _to_host_tensor, torch_loader_permutation

PADDING = {"pre": _lib.B2_LONGCTR_PAD_PRE, "post": _lib.B2_LONGCTR_PAD_POST}
_INT32_END = 1 << 31
_DTYPE_CODE = {torch.int64: _lib.B2_I64, torch.int32: _lib.B2_I32}


def load_parquet_columns(data_path):
    """ParquetDataset.load_data (longctr_dataloader.py): every column in the file's order, list-valued columns
    expanded into consecutive matrix columns.  Returns (matrix, column_index)."""
    import pandas as pd
    df = pd.read_parquet(data_path)
    arrays, column_index, idx = [], {}, 0
    for col in df.columns:
        if df[col].dtype == "object":
            array = np.array(df[col].to_list())
            column_index[col] = list(range(idx, idx + array.shape[1]))
            idx += array.shape[1]
        else:
            array = df[col].to_numpy()
            column_index[col] = idx
            idx += 1
        arrays.append(array)
    return np.column_stack(arrays), column_index


def _wanted_columns(feature_map):
    return set(list(feature_map.features.keys()) + list(feature_map.labels))


class LongCTRStore(object):
    """Every user's history and the item columns of item_info, checked on the host and copied to HBM on first use.

    user_info: parquet with a list-valued `full_item_seq` column, row u = user_index u.  item_info: parquet with an
    `item_index` column (dropped, as `set_index` drops it) and the item columns; row r is item r (the reference reads
    it with `iloc`).  The item columns kept are those the feature map names, in the file's order."""

    def __init__(self, feature_map, user_info, item_info):
        import pandas as pd
        seqs = pd.read_parquet(user_info)["full_item_seq"].values
        lens = np.fromiter((len(s) for s in seqs), dtype=np.int64, count=len(seqs))
        if len(seqs) == 0:
            raise ValueError("LongCTR store: %s holds no users" % user_info)
        self.offsets = np.zeros(len(seqs) + 1, dtype=np.int64)
        np.cumsum(lens, out=self.offsets[1:])
        hist = (np.concatenate([np.asarray(s, dtype=np.int64) for s in seqs if len(s)])
                if self.offsets[-1] else np.zeros(0, dtype=np.int64))
        items = pd.read_parquet(item_info).set_index("item_index")
        wanted = _wanted_columns(feature_map)
        self.item_columns = [c for c in items.columns if c in wanted]
        if not self.item_columns:
            raise ValueError("LongCTR store: no column of %s is a feature of the feature map" % item_info)
        cols = []
        for c in self.item_columns:
            s = items[c]
            if s.dtype == "object" and len(s) and isinstance(s.iloc[0], (list, np.ndarray)):
                raise NotImplementedError("LongCTR store: item column %s is list-valued; only scalar integer item "
                                          "columns are supported" % c)
            if not np.issubdtype(s.dtype, np.integer):
                raise ValueError("LongCTR store: item column %s has dtype %s; item columns must be integer ids"
                                 % (c, s.dtype))
            v = s.to_numpy().astype(np.int64)
            if v.size and (v.min() < -_INT32_END or v.max() >= _INT32_END):
                raise ValueError("LongCTR store: item column %s holds values outside int32" % c)
            cols.append(v)
        self.num_users, self.num_items = len(seqs), len(items)
        if self.num_items == 0:
            raise ValueError("LongCTR store: %s holds no items" % item_info)
        if hist.size:
            lo, hi = int(hist.min()), int(hist.max())
            if lo < 0 or hi >= self.num_items or hi >= _INT32_END:
                raise ValueError("LongCTR store: history item ids span [%d, %d], outside [0, %d) (the rows of "
                                 "item_info; ids at or above 2^31 would wrap in the reference's int32 padding)"
                                 % (lo, hi, self.num_items))
        self.hist = hist.astype(np.int32)
        self.table = np.ascontiguousarray(np.stack(cols, axis=1).astype(np.int32))
        self._dev = {}

    def on(self, device):
        """(offsets, hist, table) as device tensors; copied once per device."""
        device = torch.device(device)
        if device not in self._dev:
            hist = self.hist if self.hist.size else np.zeros(1, dtype=np.int32)   # a valid pointer when empty
            self._dev[device] = tuple(torch.from_numpy(a).to(device) for a in (self.offsets, hist, self.table))
        return self._dev[device]

    def collate(self, matrix, L, cols, padding, mask=None, items=None):
        """The triple's mask (B, L) float32 and item columns (C, B (L + 1)) int64 of a device batch matrix, written by
        one b2_longctr_collate launch into `mask` / `items` (allocated when None)."""
        from .functional import _ptr, _stream
        offsets, hist, table = self.on(matrix.device)
        B = matrix.shape[0]
        if mask is None:
            mask = torch.empty((B, L), dtype=torch.float32, device=matrix.device)
        if items is None:
            items = torch.empty((len(self.item_columns), B * (L + 1)), dtype=torch.int64, device=matrix.device)
        if matrix.dtype not in _DTYPE_CODE or matrix.stride(1) != 1:
            raise ValueError("LongCTR collate: the batch matrix must be a row-major int64 or int32 tensor, got %s"
                             % matrix.dtype)
        _lib.call("b2_longctr_collate", _ptr(matrix), _DTYPE_CODE[matrix.dtype], B, matrix.stride(0), cols[0],
                  cols[1], cols[2], _ptr(offsets), _ptr(hist), self.num_users, _ptr(table), self.num_items,
                  len(self.item_columns), L, PADDING[padding], _ptr(mask) if L else _ptr(None), _ptr(items), _stream())
        return mask, items


class LongCTRDataLoader(_MatrixLoaderBase):
    """model_zoo/LongCTR/longctr_dataloader.py LongCTRDataLoader: same constructor, `num_samples`, `num_blocks`,
    `num_batches`, `len()` and batch order (drop_last=False; shuffled order = `DataLoader(shuffle=True)`'s draw from
    the global torch RNG).  Iterating yields (batch_dict, item_dict, mask) on the device: batch_dict holds column
    views of the device batch matrix (the file's columns that the feature map names, in the matrix's dtype),
    item_dict one int64 tensor of B (L + 1) ids per item column, mask (B, L) float32, with
    L = min(max(seq_len of the batch), max_len).  num_workers is accepted and ignored.  `gpu` (a keyword of the
    reference's params) picks the device, cuda:0 by default."""

    def __init__(self, feature_map, data_path, user_info, item_info, batch_size=32, shuffle=False, num_workers=1,
                 max_len=50, padding="pre", pin="auto", **kwargs):
        super(LongCTRDataLoader, self).__init__(feature_map, batch_size, pin)
        if padding not in PADDING:
            raise ValueError("LongCTRDataLoader: padding must be 'pre' or 'post', got %r" % (padding,))
        if int(max_len) < 1 or int(max_len) > _lib.B2_LONGCTR_MAX_LEN:
            raise ValueError("LongCTRDataLoader: max_len must lie in [1, %d], got %s" % (_lib.B2_LONGCTR_MAX_LEN,
                                                                                       max_len))
        if not data_path.endswith(".parquet"):
            data_path += ".parquet"
        matrix, self.column_index = load_parquet_columns(data_path)
        wanted = _wanted_columns(feature_map)
        self.batch_columns = [c for c in self.column_index if c in wanted]
        for c in ("user_index", "item_index", "seq_len"):
            if c not in self.batch_columns or isinstance(self.column_index[c], list):
                raise ValueError("LongCTRDataLoader: %s needs a scalar %s column that the feature map names"
                                 % (data_path, c))
        if matrix.dtype not in (np.int64, np.int32):
            raise ValueError("LongCTRDataLoader: the columns of %s stack to %s; the reference's collator indexes "
                             "user_info and item_info with them and needs integer columns" % (data_path, matrix.dtype))
        self.store = LongCTRStore(feature_map, user_info, item_info)
        self.cols = tuple(self.column_index[c] for c in ("user_index", "item_index", "seq_len"))
        users, targets, seq = (matrix[:, c].astype(np.int64) for c in self.cols)
        if users.size and (users.min() < 0 or users.max() >= self.store.num_users):
            raise ValueError("LongCTRDataLoader: user_index spans [%d, %d], outside [0, %d) (the rows of user_info)"
                             % (users.min(), users.max(), self.store.num_users))
        if targets.size and (targets.min() < 0 or targets.max() >= self.store.num_items):
            raise ValueError("LongCTRDataLoader: item_index spans [%d, %d], outside [0, %d) (the rows of item_info)"
                             % (targets.min(), targets.max(), self.store.num_items))
        if seq.size and (seq.min() < 0 or seq.max() >= _INT32_END):
            raise ValueError("LongCTRDataLoader: seq_len spans [%d, %d], outside [0, 2^31)" % (seq.min(), seq.max()))
        self._seq = seq
        self.shuffle, self.max_len, self.padding = bool(shuffle), int(max_len), padding
        self.matrix = _to_host_tensor(matrix, False if (shuffle and pin == "auto") else pin)
        self.num_samples = matrix.shape[0]
        self.num_blocks = 1
        self.num_batches = int(np.ceil(self.num_samples / self.batch_size))
        gpu = int(kwargs.get("gpu", 0))
        self.device = torch.device("cuda", gpu if gpu >= 0 else 0)
        self._slots = None

    @property
    def item_columns(self):
        return self.store.item_columns

    def batch_dict(self, matrix):
        """The reference's batch_dict: the feature map's columns of the file, as column views of `matrix`."""
        out = {}
        for c in self.batch_columns:
            idx = self.column_index[c]
            out[c] = matrix[:, idx[0]:idx[-1] + 1] if isinstance(idx, list) else matrix[:, idx]
        return out

    def seq_max_len(self, rows):
        """L of a batch from its host seq_len values (`rows`: a slice or an index tensor)."""
        return min(int(self._seq[rows].max()), self.max_len)

    def matrices(self):
        """(pinned host batch matrix, L) per batch, in the reference's order.  Shuffled batches come from a pinned
        ring: a consumer must finish its H2D of a matrix before it asks for the ring's next-but-two batch (at most
        two copies in flight), as TrainPipeline.step does."""
        n, B = self.num_samples, self.batch_size
        if not self.shuffle:
            for lo in range(0, n, B):
                hi = min(lo + B, n)
                yield self.matrix[lo:hi], self.seq_max_len(slice(lo, hi))
            return
        perm = torch_loader_permutation(n)          # on the caller's thread: the global RNG order torch's is
        if self._slots is None:
            self._slots = self._ring_slots(self.matrix.shape[1], self.matrix.numpy().dtype)

        def produce():
            for k, lo in enumerate(range(0, n, B)):
                idx = perm[lo:lo + B]
                slot = self._slots[k % self.ring][:idx.numel()]
                torch.index_select(self.matrix, 0, idx, out=slot)
                yield slot, self.seq_max_len(idx.numpy())
        for item in _Prefetcher(produce, self.prefetch):
            yield item

    def collate(self, dev_matrix, L, mask=None, items=None):
        """The triple of a batch matrix already in HBM, written into `mask` / `items` when given."""
        mask, items = self.store.collate(dev_matrix, L, self.cols, self.padding, mask, items)
        return (self.batch_dict(dev_matrix), collections.OrderedDict(zip(self.item_columns, items.unbind(0))), mask)

    def __iter__(self):
        in_flight = collections.deque()
        self.store.on(self.device)
        for mat, L in self.matrices():
            dev = mat.to(self.device, non_blocking=True)
            done = torch.cuda.Event()
            done.record()
            in_flight.append(done)
            if len(in_flight) > 2:          # a ring slot is refilled only after its copy has left it
                in_flight.popleft().synchronize()
            yield self.collate(dev, L)

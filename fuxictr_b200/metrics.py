"""Device-resident evaluation (SURVEY.md 8f row 3): the twin of fuxictr/metrics.py:26-48 and of
the accumulation loop in BaseModel.evaluate (fuxictr/pytorch/models/rank_model.py:350-381).

The reference syncs after every validation batch (`.cpu().numpy()`), extends Python lists, and
calls sklearn on float64 copies.  Here predictions and labels are appended to HBM buffers without
a sync, and `logloss` / `AUC` are computed by csrc/metrics.cu (fp64 log-loss sum; exact integer
Mann-Whitney statistic through a radix sort), so an epoch's evaluation costs one 48-byte D2H.
Group metrics (gAUC, avgAUC, MRR, NDCG@k) are per-user host code in the reference
(metrics.py:49-72) and are outside the hot path: they raise NotImplementedError here.
"""
import ctypes
from collections import OrderedDict

import torch

from . import _lib
from . import functional as F2

_DEVICE_METRICS = ("logloss", "binary_crossentropy", "AUC")


def _check_metrics(metrics):
    for m in metrics:
        if m in _DEVICE_METRICS:
            continue
        if m in ("gAUC", "avgAUC", "MRR") or m.startswith("NDCG"):
            raise NotImplementedError("metric={} is a per-group host metric of the reference "
                                      "(fuxictr/metrics.py:49-72); not on the H100 path.".format(m))
        raise ValueError("metric={} not supported.".format(m))       # metrics.py:52


def evaluate_metrics(y_true, y_pred, metrics, group_id=None):
    """Same signature and return type as fuxictr.metrics.evaluate_metrics, on fp32 CUDA tensors."""
    _check_metrics(metrics)
    F2._require_cuda(y_pred, y_true)
    y_pred = F2._f32c(y_pred.detach().reshape(-1))
    y_true = F2._f32c(y_true.detach().reshape(-1))
    if y_pred.numel() != y_true.numel():
        raise ValueError("Found input variables with inconsistent numbers of samples: [%d, %d]"
                         % (y_true.numel(), y_pred.numel()))
    n = y_pred.numel()
    want_ll = any(m in ("logloss", "binary_crossentropy") for m in metrics)
    want_auc = "AUC" in metrics
    out = torch.zeros(6, dtype=torch.int64, device=y_pred.device)     # [0:5] b2_auc result, [5] logloss sum (f64 bits)
    if want_ll:
        _lib.call("b2_logloss_sum", F2._ptr(y_pred), F2._ptr(y_true), n,
                  ctypes.c_void_p(out.data_ptr() + 40), F2._stream())
    if want_auc:
        if n < 1:
            raise ValueError("AUC of an empty prediction set is undefined")
        nbytes = ctypes.c_int64(0)
        _lib.call("b2_auc_workspace_bytes", n, ctypes.byref(nbytes))
        ws = torch.empty(nbytes.value, dtype=torch.uint8, device=y_pred.device)   # caching allocator: 512-byte aligned
        _lib.call("b2_auc", F2._ptr(y_pred), F2._ptr(y_true), n, F2._ptr(ws), nbytes.value, F2._ptr(out),
                  F2._stream())
    host = out.cpu()                                                   # the one D2H of the evaluation
    n_neg, n_pos, n_nan, n_bad, twice_u = (int(v) for v in host[:5])
    result = OrderedDict()
    for m in metrics:
        if m in ("logloss", "binary_crossentropy"):
            result[m] = float(host[5:6].view(torch.float64)) / max(n, 1)
        elif m == "AUC":
            if n_nan:
                raise ValueError("Input contains NaN.")                # sklearn's check_array message
            if n_bad:
                raise ValueError("AUC needs binary {0, 1} labels (%d other values found)" % n_bad)
            if n_pos == 0 or n_neg == 0:
                raise ValueError("Only one class present in y_true. ROC AUC score is not defined in that case.")
            result[m] = twice_u / (2.0 * n_pos * n_neg)
    return result


class DeviceMetrics(object):
    """Append-only HBM buffers for an evaluation pass; no host sync until compute()."""

    def __init__(self, device, capacity=1 << 20):
        self.device = device
        self._pred = torch.empty(capacity, dtype=torch.float32, device=device)
        self._true = torch.empty(capacity, dtype=torch.float32, device=device)
        self.n = 0

    def _reserve(self, extra):
        need = self.n + extra
        if need <= self._pred.numel():
            return
        cap = self._pred.numel()
        while cap < need:
            cap *= 2
        for name in ("_pred", "_true"):
            grown = torch.empty(cap, dtype=torch.float32, device=self.device)
            grown[:self.n].copy_(getattr(self, name)[:self.n])
            setattr(self, name, grown)

    def append(self, y_pred, y_true=None):
        y_pred = y_pred.detach().reshape(-1)
        k = y_pred.numel()
        self._reserve(k)
        self._pred[self.n:self.n + k].copy_(y_pred, non_blocking=True)
        if y_true is not None:
            self._true[self.n:self.n + k].copy_(y_true.detach().reshape(-1), non_blocking=True)   # f64 -> f32 cast on device
        self.n += k

    def predictions(self):
        return self._pred[:self.n]

    def labels(self):
        return self._true[:self.n]

    def compute(self, metrics):
        return evaluate_metrics(self._true[:self.n], self._pred[:self.n], metrics)


def device_metrics_supported(metrics, group_id=None):
    """True when every requested metric is one of the pointwise device metrics."""
    return group_id is None and all(m in _DEVICE_METRICS for m in metrics)


def evaluate_generator(model, data_generator, metrics):
    """The loop of BaseModel.evaluate (rank_model.py:360-381) with device-resident accumulation:
    `model` needs .forward(batch) -> {"y_pred"}, .get_labels(batch), .device, .eval()."""
    model.eval()
    with torch.no_grad():
        acc = DeviceMetrics(model.device)
        for batch_data in data_generator:
            acc.append(model.forward(batch_data)["y_pred"], model.get_labels(batch_data))
        return acc.compute(metrics)


def predict_generator(model, data_generator):
    """BaseModel.predict (rank_model.py:383-398): flattened float64 numpy array, one D2H."""
    model.eval()
    with torch.no_grad():
        acc = DeviceMetrics(model.device)
        for batch_data in data_generator:
            acc.append(model.forward(batch_data)["y_pred"])
        return acc.predictions().cpu().numpy().astype("float64")

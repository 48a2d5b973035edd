"""enable(): route the UNMODIFIED reference's hot-path layers through the H100 kernels.

On a machine that has reczoo/FuxiCTR installed, ``import fuxictr_b200.patch as p; p.enable()``
(before or after building a model) swaps the ``forward`` of the reference's own layer classes —
class identity, parameters, ``state_dict`` keys, initialisation order and the
``type(module) == FeatureEmbeddingDict`` test of the regulariser (rank_model.py:107) are untouched,
so any ``model_zoo`` model keeps running from its YAML config.  A patched forward uses the kernels
when its tensors are CUDA tensors and the configuration is one the kernels cover; otherwise it
calls the reference's original forward (the reference's own code, not a fallback of ours).

Patched: FeatureEmbedding, FeatureEmbeddingDict, LogisticRegression, InnerProductInteraction,
CrossNet, CrossNetV2, CrossNetMix, CompressedInteractionNet, DIN_Attention, MultiHeadTargetAttention,
Dice, MLP_Block
(fuxictr/pytorch/layers/**, SURVEY.md 8a); and BaseModel.evaluate / BaseModel.predict
(fuxictr/pytorch/models/rank_model.py:350-398, SURVEY.md 8f row 3): for a model on a CUDA device
whose metrics are logloss / AUC (no group metrics) the predictions stay in HBM and
csrc/metrics.cu computes the numbers; any other case runs the reference's own method.
"""
import logging
import functools

import torch

from . import layers as M

_ORIGINALS = {}
_STATE = {"enabled": False, "calls": {}}


def _tensors(args, kwargs):
    for a in list(args) + list(kwargs.values()):
        if isinstance(a, torch.Tensor):
            yield a
        elif isinstance(a, dict):
            for v in a.values():
                if isinstance(v, torch.Tensor):
                    yield v


def _on_cuda(args, kwargs):
    ts = list(_tensors(args, kwargs))
    return bool(ts) and all(t.is_cuda for t in ts)


def _wrap(ref_cls, mirror_forward, supported=None):
    name = ref_cls.__name__
    original = ref_cls.forward
    _ORIGINALS[ref_cls] = original

    @functools.wraps(original)
    def forward(self, *args, **kwargs):
        if _STATE["enabled"] and _on_cuda(args, kwargs) and (supported is None or supported(self)):
            _STATE["calls"][name] = _STATE["calls"].get(name, 0) + 1
            return mirror_forward(self, *args, **kwargs)
        return original(self, *args, **kwargs)
    ref_cls.forward = forward


def _graft_methods(ref_cls, mirror_cls, names):
    for n in names:
        setattr(ref_cls, n, getattr(mirror_cls, n))


def _fed_supported(self):
    if not hasattr(self, "_plans"):
        self._plans = {}
    return True


def _mlp_supported(self):
    return True


def _crossnet_mix_supported(self):
    """The kernels' range of low_rank and num_experts (include/fuxictr_b200.h "CrossNetMix")."""
    from . import functional as F2
    if self.layer_num == 0:
        return True
    return F2.crossnet_mix_bound(self.U_list[0].shape[2], self.num_experts) is None


def _target_attention_supported(self):
    """The kernels' row width and head count (include/fuxictr_b200.h "MultiHeadTargetAttention"), and no
    attention dropout in training mode."""
    from . import functional as F2
    if self.dot_attention.dropout is not None and self.training:
        return False
    width = self.num_heads * self.W_q.in_features if self.use_qkvo else self.num_heads * self.head_dim
    return F2.target_attention_bound(width, self.num_heads) is None


def _wrap_base_model(base_cls):
    from . import metrics as DM
    orig_evaluate, orig_predict = base_cls.evaluate, base_cls.predict
    _ORIGINALS[(base_cls, "evaluate")], _ORIGINALS[(base_cls, "predict")] = orig_evaluate, orig_predict

    def _device_model(self):
        return _STATE["enabled"] and getattr(self, "device", None) is not None and self.device.type == "cuda"

    @functools.wraps(orig_evaluate)
    def evaluate(self, data_generator, metrics=None):
        names = metrics if metrics is not None else self.validation_metrics
        if _device_model(self) and DM.device_metrics_supported(names, getattr(self.feature_map, "group_id", None)):
            _STATE["calls"]["evaluate"] = _STATE["calls"].get("evaluate", 0) + 1
            val_logs = DM.evaluate_generator(self, data_generator, names)
            logging.info("[Metrics] " + " - ".join("{}: {:.6f}".format(k, v) for k, v in val_logs.items()))
            return val_logs
        return orig_evaluate(self, data_generator, metrics)

    @functools.wraps(orig_predict)
    def predict(self, data_generator):
        if _device_model(self):
            _STATE["calls"]["predict"] = _STATE["calls"].get("predict", 0) + 1
            return DM.predict_generator(self, data_generator)
        return orig_predict(self, data_generator)
    base_cls.evaluate, base_cls.predict = evaluate, predict


def enable():
    """Patch the reference classes in place (idempotent).  Raises ImportError when the reference
    package is not importable — this module is only meaningful next to it."""
    import fuxictr.pytorch.layers as R
    if _ORIGINALS:
        _STATE["enabled"] = True
        return
    from fuxictr.pytorch.models.rank_model import BaseModel
    _wrap_base_model(BaseModel)
    # helper methods the mirrored forwards call on `self`
    _graft_methods(R.FeatureEmbeddingDict, M.FeatureEmbeddingDict,
                   ["_active_features", "_is_fusable", "_plan", "_fused_arena", "forward_tensor"])
    _wrap(R.FeatureEmbeddingDict, M.FeatureEmbeddingDict.forward, _fed_supported)
    _wrap(R.FeatureEmbedding, M.FeatureEmbedding.forward, lambda s: _fed_supported(s.embedding_layer))

    def lr_ok(self):
        if not hasattr(self, "_lr_plans"):
            self._lr_plans = {}
        return _fed_supported(self.embedding_layer.embedding_layer)
    _wrap(R.LogisticRegression, M.LogisticRegression.forward, lr_ok)
    _wrap(R.InnerProductInteraction, M.InnerProductInteraction.forward)
    _wrap(R.CrossNet, M.CrossNet.forward)
    _wrap(R.CrossNetV2, M.CrossNetV2.forward)
    _wrap(R.CrossNetMix, M.CrossNetMix.forward, _crossnet_mix_supported)
    _wrap(R.CompressedInteractionNet, M.CompressedInteractionNet.forward)
    _wrap(R.DIN_Attention, M.DIN_Attention.forward)
    _wrap(R.MultiHeadTargetAttention, M.MultiHeadTargetAttention.forward, _target_attention_supported)
    _wrap(R.Dice, M.Dice.forward)
    _graft_methods(R.MLP_Block, M.MLP_Block, ["chain_layers"])     # the tensor-core modes' one-node chain
    _wrap(R.MLP_Block, M.MLP_Block.forward, _mlp_supported)
    _STATE["enabled"] = True


def disable():
    """Back to the reference's own forwards (the patches stay installed but inert)."""
    _STATE["enabled"] = False


def call_counts():
    """How many times each patched forward took the kernel path (for tests / diagnostics)."""
    return dict(_STATE["calls"])

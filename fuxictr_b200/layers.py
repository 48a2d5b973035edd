"""Drop-in torch.nn.Module mirrors of the reference's hot-path layers.

Same class names, constructor signatures, child-module names (hence state_dict keys),
initialisation order and forward signatures as ``fuxictr.pytorch.layers`` — the modules
are *parameter containers*; their forwards dispatch to the sm_90a kernels of
libfuxictr_b200.so through fuxictr_b200.functional.  CUDA tensors are required: a CPU
tensor raises (there is no CPU implementation on this path).

Reference files (relative to the reference root):
  FeatureEmbedding / FeatureEmbeddingDict  fuxictr/pytorch/layers/embeddings/feature_embedding.py:30-297
  MaskedAveragePooling / MaskedSumPooling  fuxictr/pytorch/layers/pooling.py:23-73
  LogisticRegression                       fuxictr/pytorch/layers/blocks/logistic_regression.py:24-59
  FactorizationMachine                     fuxictr/pytorch/layers/blocks/factorization_machine.py:25-59
  InnerProductInteraction                  fuxictr/pytorch/layers/interactions/inner_product.py:23-70
  CrossInteraction / CrossNet / CrossNetV2 fuxictr/pytorch/layers/interactions/cross_net.py:24-129
  CompressedInteractionNet                 fuxictr/pytorch/layers/interactions/compressed_interaction_net.py:23-76
  DIN_Attention                            fuxictr/pytorch/layers/attentions/target_attention.py:26-92
  MultiHeadTargetAttention                 fuxictr/pytorch/layers/attentions/target_attention.py:95-172
  ScaledDotProductAttention                fuxictr/pytorch/layers/attentions/dot_product_attention.py:24-58
  Dice                                     fuxictr/pytorch/layers/activations.py:24-51
  MLP_Block                                fuxictr/pytorch/layers/blocks/mlp_block.py:24-96
  FeatureSelection / InteractionAggregation model_zoo/FinalMLP/src/FinalMLP.py
  MaskBlock / SerialMaskNet / ParallelMaskNet model_zoo/MaskNet/src/MaskNet.py
  MultiHeadSelfAttention                   model_zoo/AutoInt/src/AutoInt.py
  FactorizationMachineBlock / LinearCompressionBlock / WuKongLayer model_zoo/WuKong/src/WuKong.py
  FeatureGating / FactorizedInteraction / FinalBlock model_zoo/FinalNet/src/FinalNet.py
  TransformerBlock / BehaviorTransformer   model_zoo/BST/src/BST.py
"""
import sys
from collections import OrderedDict
from functools import partial  # noqa: F401  (initializer strings use it)

import numpy as np  # noqa: F401
import torch
from torch import nn

from . import _lib
from . import functional as F2
from ._lib import (B2_POOL_NONE, B2_POOL_SUM, B2_POOL_MEAN, B2_ACT_NONE, B2_ACT_RELU,
                   B2_ACT_SIGMOID, B2_ACT_LEAKY_RELU, FM_PRODUCT_SUM, FM_BI_INTERACTION, FM_INNER_PRODUCT)

layers = sys.modules[__name__]  # so feature_encoder strings like "layers.MaskedSumPooling()" resolve


def not_in_whitelist(element, whitelist=[]):
    """fuxictr/utils.py: an empty whitelist admits everything; a scalar whitelist is a 1-list."""
    if not whitelist:
        return False
    allowed = whitelist if isinstance(whitelist, list) else [whitelist]
    return element not in allowed


def get_initializer(initializer):
    """torch_utils.py:175-194: the YAML carries initializers as Python expressions over `nn` / `partial`."""
    if not isinstance(initializer, str):
        return initializer
    try:
        return eval(initializer)
    except Exception:
        raise ValueError("initializer={} is not supported.".format(initializer))


_NAMED_ACTIVATIONS = {
    "relu": lambda units: nn.ReLU(),
    "sigmoid": lambda units: nn.Sigmoid(),
    "tanh": lambda units: nn.Tanh(),
    "softmax": lambda units: nn.Softmax(dim=-1),
    "prelu": lambda units: nn.PReLU(units, init=0.1),
    "dice": lambda units: Dice(units),
}


def get_activation(activation, hidden_units=None):
    """torch_utils.py:137-173: name -> module; a list of names maps element-wise (per-layer widths
    for the two activations that own parameters); anything else (a module, None) passes through."""
    if isinstance(activation, list):
        if hidden_units is None:
            return [get_activation(a) for a in activation]
        assert len(activation) == len(hidden_units)
        return [get_activation(a, u) for a, u in zip(activation, hidden_units)]
    if not isinstance(activation, str):
        return activation
    key = activation.lower()
    if key in ("prelu", "dice"):
        assert type(hidden_units) == int
    make = _NAMED_ACTIVATIONS.get(key)
    return make(hidden_units) if make is not None else getattr(nn, activation)()


# --------------------------------------------------------------------------------------
# Pooling encoders (fused into the gather when used as a feature_encoder)
# --------------------------------------------------------------------------------------
class MaskedAveragePooling(nn.Module):
    """pooling.py:33-49.  As a sequence feature's encoder it is fused into the gather; called directly on
    a materialised (B, L, D) tensor these are glue ops.  Positions count when their VECTOR is non-zero."""

    def forward(self, embedding_matrix, mask=None):
        if mask is None:
            mask = embedding_matrix.sum(dim=-1) != 0
        count = mask.float().sum(-1, keepdim=True)
        return embedding_matrix.sum(dim=1) / (count + 1e-12)


class MaskedSumPooling(nn.Module):
    """pooling.py:62-73."""

    def forward(self, embedding_matrix):
        return embedding_matrix.sum(dim=1)


# --------------------------------------------------------------------------------------
# Embeddings
# --------------------------------------------------------------------------------------
class FeatureEmbeddingDict(nn.Module):
    """feature_embedding.py:91-297.  Construction contract (pinned seed-for-seed against the live
    reference by tests/test_host_logic.py): features are visited in FeatureMap order; a feature's
    encoder module (if any) is registered BEFORE its table; a `share_embedding` feature aliases the
    earlier feature's module; LR mode (embedding_dim == 1 without pretrain+sharing) forces width 1
    and sum-pools sequences; afterwards every owned nn.Embedding is re-initialised (padding row kept)."""

    def __init__(self, feature_map, embedding_dim,
                 embedding_initializer="partial(nn.init.normal_, std=1e-4)",
                 required_feature_columns=None, not_required_feature_columns=None,
                 use_pretrain=True, use_sharing=True):
        super(FeatureEmbeddingDict, self).__init__()
        self._feature_map = feature_map
        self.required_feature_columns = required_feature_columns
        self.not_required_feature_columns = not_required_feature_columns
        self.use_pretrain = use_pretrain
        self.embedding_initializer = get_initializer(embedding_initializer)
        self.embedding_layers = nn.ModuleDict()
        self.feature_encoders = nn.ModuleDict()
        self._plans = {}
        lr_mode = embedding_dim == 1 and not (use_pretrain and use_sharing)
        for name, spec in feature_map.features.items():
            if not self.is_required(name):
                continue
            kind = spec["type"]
            width = 1 if lr_mode else spec.get("embedding_dim", embedding_dim)
            encoder = self._make_encoder(spec, kind, width, lr_mode)
            if encoder is not None:
                self.feature_encoders[name] = encoder
            donor = spec.get("share_embedding") if use_sharing else None
            if donor is not None and donor in self.embedding_layers:
                self.embedding_layers[name] = self.embedding_layers[donor]     # one module, two names
                continue
            table = self._make_table(name, spec, kind, width)
            if table is not None:
                self.embedding_layers[name] = table
        self.init_weights()

    def _make_encoder(self, spec, kind, width, lr_mode):
        if lr_mode:
            return MaskedSumPooling() if kind == "sequence" else None
        if spec.get("feature_encoder", None):
            return self.get_feature_encoder(spec["feature_encoder"])
        if kind == "embedding":     # a dense vector feature is projected to the embedding width
            return nn.Linear(spec.get("pretrain_dim", width), width, bias=False)
        return None

    def _make_table(self, name, spec, kind, width):
        if kind == "numeric":
            return nn.Linear(1, width, bias=False)
        if kind == "embedding":
            return nn.Identity()
        if kind in ("categorical", "sequence"):
            if self.use_pretrain and "pretrained_emb" in spec:
                raise NotImplementedError(
                    "feature %s: pretrained_emb is outside the H100 hot path "
                    "(SURVEY.md section 2 row 2); keep the reference module for it" % name)
            return nn.Embedding(spec["vocab_size"], width, padding_idx=spec.get("padding_idx", None))
        return None

    def get_feature_encoder(self, encoder):
        """Encoder strings are Python expressions over this module (`layers.MaskedSumPooling()`, `nn.*`)."""
        try:
            if type(encoder) == list:
                return nn.Sequential(*[eval(expr) for expr in encoder])
            return eval(encoder)
        except Exception:
            raise ValueError("feature_encoder={} is not supported.".format(encoder))

    def init_weights(self):
        specs = self._feature_map.features
        for name, module in self.embedding_layers.items():
            if "share_embedding" in specs[name] or type(module) != nn.Embedding:
                continue
            # rows 1.. only when a padding row exists (the reference assumes padding_idx == 0)
            target = module.weight if module.padding_idx is None else module.weight[1:, :]
            self.embedding_initializer(target)

    def is_required(self, feature):
        if self._feature_map.features[feature]["type"] == "meta":
            return False
        wanted, unwanted = self.required_feature_columns, self.not_required_feature_columns
        if wanted and feature not in wanted:
            return False
        return not (unwanted and feature in unwanted)

    def dict2tensor(self, embedding_dict, flatten_emb=False, feature_list=[], feature_source=[],
                    feature_type=[]):
        """FeatureMap order, three optional whitelists; concat on the last dim or stack on dim 1."""
        picked = []
        for name, spec in self._feature_map.features.items():
            if name not in embedding_dict:
                continue
            if (feature_list and not_in_whitelist(name, feature_list)) or \
                    (feature_source and not_in_whitelist(spec["source"], feature_source)) or \
                    (feature_type and not_in_whitelist(spec["type"], feature_type)):
                continue
            picked.append(embedding_dict[name])
        return torch.cat(picked, dim=-1) if flatten_emb else torch.stack(picked, dim=1)

    # ---- fused path -------------------------------------------------------------------
    def _active_features(self, inputs, feature_source, feature_type):
        """Input keys (caller's order) that own a table and pass the source / type whitelists."""
        specs = self._feature_map.features

        def admitted(name):
            if name not in self.embedding_layers:
                return False
            spec = specs[name]
            return not ((feature_source and not_in_whitelist(spec["source"], feature_source)) or
                        (feature_type and not_in_whitelist(spec["type"], feature_type)))
        return [name for name in inputs.keys() if admitted(name)]

    # value transform the reference applies before a feature's table, by feature type
    # (feature_embedding.py:279-291); only features OUTSIDE the fused kernel go through it
    _CASTS = {
        "numeric": lambda t: t.float().view(-1, 1),
        "categorical": lambda t: t.long(),
        "sequence": lambda t: t.long(),
        "embedding": lambda t: t.float(),
    }

    def _unfused_lookup(self, name, column):
        kind = self._feature_map.features[name]["type"]
        if kind not in self._CASTS:
            raise NotImplementedError
        out = self.embedding_layers[name](self._CASTS[kind](column))
        return self.feature_encoders[name](out) if name in self.feature_encoders else out

    def _is_fusable(self, feature):
        """Plain nn.Embedding lookup, optionally followed by a Masked{Sum,Average}Pooling."""
        spec = self._feature_map.features[feature]
        if spec["type"] not in ("categorical", "sequence"):
            return False
        if type(self.embedding_layers[feature]) != nn.Embedding:
            return False
        if feature in self.feature_encoders:
            enc = self.feature_encoders[feature]
            # by name: the reference's own pooling classes qualify too (fuxictr_b200.patch)
            if not (spec["type"] == "sequence" and
                    type(enc).__name__ in ("MaskedSumPooling", "MaskedAveragePooling")):
                return False
        return True

    def _plan(self, names, order):
        """Build (and cache) the launch plan for the fusable features `names` laid out in `order`."""
        key = (tuple(names), tuple(order))
        plan = self._plans.get(key)
        if plan is not None:
            return plan
        tables, slot_of, fields = [], {}, []
        for feature in order:
            spec = self._feature_map.features[feature]
            emb = self.embedding_layers[feature]
            if id(emb) not in slot_of:
                slot_of[id(emb)] = len(tables)
                tables.append(emb)
            seq_len = spec["max_len"] if spec["type"] == "sequence" else 1
            pool = B2_POOL_NONE
            if feature in self.feature_encoders:
                pool = B2_POOL_SUM if type(self.feature_encoders[feature]).__name__ == "MaskedSumPooling" \
                    else B2_POOL_MEAN
            fields.append(F2.GatherField(feature, slot_of[id(emb)], emb.embedding_dim, seq_len, pool,
                                         emb.padding_idx))
        plan = (F2.GatherPlan(fields), tables)
        self._plans[key] = plan
        return plan

    def _fused_arena(self, inputs, order):
        plan, tables = self._plan(order, order)
        idx = [inputs[f] for f in order]
        arena = F2.embed_gather(plan, idx, [t.weight for t in tables])
        return plan, arena

    def forward(self, inputs, feature_source=[], feature_type=[]):
        names = self._active_features(inputs, feature_source, feature_type)
        feature_emb_dict = OrderedDict()
        fusable = [f for f in names if self._is_fusable(f)]
        fused_out = {}
        if fusable:
            plan, arena = self._fused_arena(inputs, fusable)
            B = arena.shape[0]
            parts = arena.split(plan.widths, dim=1) if len(fusable) > 1 else (arena,)
            for field, part in zip(plan.fields, parts):
                if field.seq_len > 1 and field.pool == B2_POOL_NONE:
                    part = part.reshape(B, field.seq_len, field.dim)
                fused_out[field.name] = part
        for name in names:      # numeric / embedding-type / custom-encoder features: stock module calls
            feature_emb_dict[name] = fused_out[name] if name in fused_out else self._unfused_lookup(name, inputs[name])
        return feature_emb_dict

    def forward_tensor(self, inputs, feature_source=[], feature_type=[], flatten_emb=False):
        """FeatureEmbedding.forward in one launch: the gather writes the stacked (B,F,D) /
        concatenated (B, sum D) tensor directly (no dict, no torch.stack/cat)."""
        names = self._active_features(inputs, feature_source, feature_type)
        order = [f for f in self._feature_map.features.keys() if f in set(names)]
        if order and all(self._is_fusable(f) for f in order):
            plan, arena = self._fused_arena(inputs, order)
            unpooled = any(f.seq_len > 1 and f.pool == B2_POOL_NONE for f in plan.fields)
            if flatten_emb and not unpooled:
                return arena
            dims = set(f.dim for f in plan.fields)
            if not flatten_emb and not unpooled and len(dims) == 1:
                return arena.view(arena.shape[0], len(plan.fields), plan.fields[0].dim)
        feature_emb_dict = self.forward(inputs, feature_source=feature_source, feature_type=feature_type)
        return self.dict2tensor(feature_emb_dict, flatten_emb=flatten_emb)


def front_plan(embedding_layer, lr_layer, X):
    """(order, plan, tables, lr_plan, lr_tables) of the launch fused_front makes for inputs X, or None when the
    configuration needs the general path (sequence / numeric features, mixed dims, dim % 4 != 0)."""
    fed = embedding_layer.embedding_layer
    names = fed._active_features(X, [], [])
    order = [f for f in fed._feature_map.features.keys() if f in set(names)]
    if not order or not all(fed._is_fusable(f) for f in order):
        return None
    plan, tables = fed._plan(order, order)
    lr_plan = lr_tables = None
    if lr_layer is not None:
        lfed = lr_layer.embedding_layer.embedding_layer
        lnames = lfed._active_features(X, [], [])
        lorder = [f for f in lfed._feature_map.features.keys() if f in set(lnames)]
        if lorder != order or not all(lfed._is_fusable(f) for f in lorder):
            return None
        lr_plan, lr_tables = lfed._plan(lorder, lorder)
    if not F2.front_supported(plan, lr_plan):
        return None
    return order, plan, tables, lr_plan, lr_tables


def fused_front(embedding_layer, lr_layer, X, want_fm):
    """One launch for FeatureEmbedding + (FM product_sum) + (LogisticRegression): returns
    (feature_emb (B,F,D), logit (B,1)), or None when the configuration needs the general path."""
    fp = front_plan(embedding_layer, lr_layer, X)
    if fp is None:
        return None
    order, plan, tables, lr_plan, lr_tables = fp
    bias = lr_layer.bias if lr_layer is not None else None
    arena, logit = F2.front(plan, lr_plan, [X[f] for f in order], [t.weight for t in tables],
                            [t.weight for t in lr_tables] if lr_tables else [], bias, want_fm)
    return arena.view(arena.shape[0], len(plan.fields), plan.fields[0].dim), logit


class FeatureEmbedding(nn.Module):
    """feature_embedding.py:30-88: a FeatureEmbeddingDict (child name `embedding_layer`) whose forward
    returns the stacked / concatenated tensor."""

    def __init__(self, feature_map, embedding_dim, embedding_initializer="partial(nn.init.normal_, std=1e-4)",
                 required_feature_columns=None, not_required_feature_columns=None, use_pretrain=True,
                 use_sharing=True):
        super(FeatureEmbedding, self).__init__()
        self.embedding_layer = FeatureEmbeddingDict(
            feature_map, embedding_dim, embedding_initializer=embedding_initializer,
            required_feature_columns=required_feature_columns,
            not_required_feature_columns=not_required_feature_columns,
            use_pretrain=use_pretrain, use_sharing=use_sharing)

    def forward(self, X, feature_source=[], feature_type=[], flatten_emb=False):
        return self.embedding_layer.forward_tensor(X, feature_source=feature_source,
                                                   feature_type=feature_type, flatten_emb=flatten_emb)


# --------------------------------------------------------------------------------------
# LR / FM
# --------------------------------------------------------------------------------------
class LogisticRegression(nn.Module):
    """logistic_regression.py:24-59: first-order term = width-1 embedding tables summed over the fields
    (+ bias).  `bias` is registered before the tables (state_dict / RNG order of the reference)."""

    def __init__(self, feature_map, use_bias=True):
        super(LogisticRegression, self).__init__()
        self.bias = nn.Parameter(torch.zeros(1), requires_grad=True) if use_bias else None
        self.embedding_layer = FeatureEmbedding(feature_map, 1, use_pretrain=False, use_sharing=False)
        self._lr_plans = {}

    def forward(self, X):
        fed = self.embedding_layer.embedding_layer
        names = fed._active_features(X, [], [])
        order = [f for f in fed._feature_map.features.keys() if f in set(names)]
        if order and all(fed._is_fusable(f) for f in order):
            key = tuple(order)
            if key not in self._lr_plans:
                self._lr_plans[key] = fed._plan(order, order)
            plan, tables = self._lr_plans[key]
            return F2.lr_forward(plan, [X[f] for f in order], [t.weight for t in tables], self.bias)
        embed_weights = self.embedding_layer(X)
        output = embed_weights.sum(dim=1)
        if self.bias is not None:
            output = output + self.bias
        return output


class InnerProductInteraction(nn.Module):
    """inner_product.py:23-70.  output: product_sum (B,1) | bi_interaction (B,D) | inner_product
    (B, F(F-1)/2) | elementwise_product (B, F(F-1)/2, D).  The pair-selection buffers are frozen
    Parameters like the reference's (they appear in state_dict)."""

    _OUTPUTS = ("product_sum", "bi_interaction", "inner_product", "elementwise_product")

    def __init__(self, num_fields, output="product_sum"):
        super(InnerProductInteraction, self).__init__()
        if output not in self._OUTPUTS:
            raise ValueError("InnerProductInteraction output={} is not supported.".format(output))
        self._output_type = output
        if output == "inner_product":
            self.interaction_units = int(num_fields * (num_fields - 1) / 2)
            upper = torch.triu(torch.ones(num_fields, num_fields), 1).bool()
            self.triu_mask = nn.Parameter(upper, requires_grad=False)
        elif output == "elementwise_product":
            pairs = torch.triu_indices(num_fields, num_fields, offset=1)
            self.triu_index = nn.Parameter(pairs, requires_grad=False)

    def forward(self, feature_emb):
        if self._output_type == "product_sum":
            return F2.fm_interaction(feature_emb, FM_PRODUCT_SUM)
        elif self._output_type == "bi_interaction":
            return F2.fm_interaction(feature_emb, FM_BI_INTERACTION)
        elif self._output_type == "inner_product":
            return F2.fm_interaction(feature_emb, FM_INNER_PRODUCT)
        else:  # elementwise_product (PNN family, outside the five in-scope models): glue ops
            emb1 = torch.index_select(feature_emb, 1, self.triu_index[0])
            emb2 = torch.index_select(feature_emb, 1, self.triu_index[1])
            return emb1 * emb2


class FactorizationMachine(nn.Module):
    """factorization_machine.py:25-59: second-order product_sum + LogisticRegression."""

    def __init__(self, feature_map):
        super(FactorizationMachine, self).__init__()
        self.fm_layer = InnerProductInteraction(feature_map.num_fields, output="product_sum")
        self.lr_layer = LogisticRegression(feature_map, use_bias=True)

    def forward(self, X, feature_emb):
        return self.fm_layer(feature_emb) + self.lr_layer(X)


# --------------------------------------------------------------------------------------
# Cross networks
# --------------------------------------------------------------------------------------
class CrossInteraction(nn.Module):
    """cross_net.py:24-55: one rank-1 cross layer; parameters `weight` (Linear(d, 1), no bias) and `bias` (d)."""

    def __init__(self, input_dim):
        super(CrossInteraction, self).__init__()
        self.weight = nn.Linear(input_dim, 1, bias=False)
        self.bias = nn.Parameter(torch.zeros(input_dim))

    def forward(self, X_0, X_i):
        # stand-alone use only: CrossNet runs all of its CrossInteraction layers in one launch
        return F2.linear_act(X_i, self.weight.weight, None, B2_ACT_NONE) * X_0 + self.bias


class CrossNet(nn.Module):
    """cross_net.py:58-92: x_{i+1} = x_i + (w_i . x_i) x_0 + b_i; all layers in one kernel each way."""

    def __init__(self, input_dim, num_layers):
        super(CrossNet, self).__init__()
        self.num_layers = num_layers
        self.cross_net = nn.ModuleList([CrossInteraction(input_dim) for _ in range(num_layers)])

    def forward(self, X_0):
        if self.num_layers == 0:
            return X_0
        w = torch.cat([layer.weight.weight for layer in self.cross_net], dim=0)     # (L, d)
        b = torch.stack([layer.bias for layer in self.cross_net], dim=0)             # (L, d)
        return F2.crossnet(X_0, w, b)


class CrossNetV2(nn.Module):
    """cross_net.py:95-129: x_{i+1} = x_i + x_0 * (W_i x_i + b_i); each layer is ONE GEMM whose epilogue
    applies the cross (add + mul * (acc + bias))."""

    def __init__(self, input_dim, num_layers):
        super(CrossNetV2, self).__init__()
        self.num_layers = num_layers
        self.cross_layers = nn.ModuleList([nn.Linear(input_dim, input_dim) for _ in range(num_layers)])

    def forward(self, X_0):
        X_i = X_0
        for layer in self.cross_layers:
            X_i = F2.cross_v2_layer(X_0, X_i, layer.weight, layer.bias)
        return X_i


class CrossNetMix(nn.Module):
    """cross_net.py:132-201 (DCN-Mix): per layer a softmax-gated mixture of E low-rank experts,
    x_{l+1} = x_l + sum_e p_e x_0 * (U_e tanh(C_e tanh(V_e^T x_l)) + b).  Each layer is one autograd node:
    two GEMMs around the per-row expert kernel (functional._CrossMixLayer).  Parameters, their names,
    registration order and initialisation draws are the reference's; the output is squeezed like its
    `x_l.squeeze()`."""

    def __init__(self, in_features, layer_num=2, low_rank=32, num_experts=4):
        super(CrossNetMix, self).__init__()
        bound = F2.crossnet_mix_bound(low_rank, num_experts)
        if bound is not None:
            raise NotImplementedError("CrossNetMix kernels: " + bound)
        self.layer_num = layer_num
        self.num_experts = num_experts
        self.U_list = torch.nn.ParameterList([nn.Parameter(nn.init.xavier_normal_(
            torch.empty(num_experts, in_features, low_rank))) for i in range(self.layer_num)])
        self.V_list = torch.nn.ParameterList([nn.Parameter(nn.init.xavier_normal_(
            torch.empty(num_experts, in_features, low_rank))) for i in range(self.layer_num)])
        self.C_list = torch.nn.ParameterList([nn.Parameter(nn.init.xavier_normal_(
            torch.empty(num_experts, low_rank, low_rank))) for i in range(self.layer_num)])
        self.gating = nn.ModuleList([nn.Linear(in_features, 1, bias=False) for i in range(self.num_experts)])
        self.bias = torch.nn.ParameterList([nn.Parameter(nn.init.zeros_(
            torch.empty(in_features, 1))) for i in range(self.layer_num)])

    def forward(self, inputs):
        x_l = inputs
        if self.layer_num > 0:
            gates = torch.cat([g.weight for g in self.gating], dim=0)        # (E, d), shared by every layer
            for i in range(self.layer_num):
                x_l = F2.crossnet_mix_layer(inputs, x_l, self.U_list[i], self.V_list[i], self.C_list[i], gates,
                                            self.bias[i])
        return x_l.squeeze()


class GateCorssLayer(nn.Module):
    """GDCN's gated cross network (model_zoo/GDCN/src/GDCN.py, GateCorssLayer; the reference's spelling),
    x_{i+1} = x_0 * (W_i x_i + b_i) * sigmoid(Wg_i x_i) + x_i.  Each layer is one autograd node: one GEMM on the
    stacked [W_i; Wg_i] and one row kernel (functional._GatedCrossLayer).  Children `w`, `wg` (bias-free Linears),
    `b` (uniform in [0, 1)) and `activation`, registered and drawn in the reference's order."""

    def __init__(self, input_dim, cn_layers=3):
        super(GateCorssLayer, self).__init__()
        self.cn_layers = cn_layers
        self.w = nn.ModuleList([nn.Linear(input_dim, input_dim, bias=False) for _ in range(cn_layers)])
        self.wg = nn.ModuleList([nn.Linear(input_dim, input_dim, bias=False) for _ in range(cn_layers)])
        self.b = nn.ParameterList([nn.Parameter(torch.zeros(input_dim)) for _ in range(cn_layers)])
        for p in self.b:
            nn.init.uniform_(p.data)
        self.activation = nn.Sigmoid()

    def forward(self, x):
        x0 = x
        for i in range(self.cn_layers):
            x = F2.gated_cross_layer(x0, x, self.w[i].weight, self.wg[i].weight, self.b[i])
        return x


def _mask_act(module):
    """The B2_ACT_* code of a MaskBlock's hidden activation module; the row kernel implements ReLU and Sigmoid."""
    if type(module) == nn.ReLU:
        return B2_ACT_RELU
    if type(module) == nn.Sigmoid:
        return B2_ACT_SIGMOID
    raise NotImplementedError("MaskBlock: hidden activation %s is not implemented on the H100 path (ReLU and "
                              "Sigmoid are)" % type(module).__name__)


class MaskBlock(nn.Module):
    """MaskNet's mask block (model_zoo/MaskNet/src/MaskNet.py, MaskBlock):
    out = hidden_layer(mask_layer(V_emb) * V_hidden), mask_layer = Linear -> ReLU -> Linear,
    hidden_layer = Linear(bias=False) -> [LayerNorm] -> activation -> [Dropout].  Children, registration order and
    initial draws are the reference's.  The forward runs on the kernels (functional.mask_blocks): three GEMMs and one
    row kernel for LayerNorm, activation and dropout.  Output widths beyond the row kernel's bound and activations
    other than ReLU and Sigmoid are refused here, before any CUDA call."""

    def __init__(self, input_dim, hidden_dim, output_dim, hidden_activation="ReLU", reduction_ratio=1,
                 dropout_rate=0, layer_norm=True):
        super(MaskBlock, self).__init__()
        bound = F2.masknet_width_bound(output_dim, "MaskBlock output_dim")
        if bound:
            raise ValueError(bound)
        self.mask_layer = nn.Sequential(nn.Linear(input_dim, int(hidden_dim * reduction_ratio)),
                                        nn.ReLU(),
                                        nn.Linear(int(hidden_dim * reduction_ratio), hidden_dim))
        hidden_layers = [nn.Linear(hidden_dim, output_dim, bias=False)]
        if layer_norm:
            hidden_layers.append(nn.LayerNorm(output_dim))
        hidden_layers.append(get_activation(hidden_activation))
        if dropout_rate > 0:
            hidden_layers.append(nn.Dropout(p=dropout_rate))
        self.hidden_layer = nn.Sequential(*hidden_layers)
        self._act = _mask_act(hidden_layers[2 if layer_norm else 1])
        if dropout_rate > 0:
            F2.dropout_consts(dropout_rate)         # a rate outside (0, 1) is refused here, as nn.Dropout does

    def block_params(self):
        """(W1, b1, W2, b2, W3, gamma, beta) of functional.mask_blocks."""
        ln = self.hidden_layer[1] if type(self.hidden_layer[1]) == nn.LayerNorm else None
        return (self.mask_layer[0].weight, self.mask_layer[0].bias, self.mask_layer[2].weight, self.mask_layer[2].bias,
                self.hidden_layer[0].weight, ln.weight if ln is not None else None, ln.bias if ln is not None else None)

    def dropout_rate(self):
        """The block's dropout probability in training mode, 0 in eval mode (nn.Dropout is then the identity)."""
        last = self.hidden_layer[-1]
        return last.p if (type(last) == nn.Dropout and last.training) else 0.0

    def forward(self, V_emb, V_hidden):
        return _run_mask_blocks([self], V_emb, V_hidden)


def _masknet_eps(blocks):
    ln = blocks[0].hidden_layer[1]
    return ln.eps if type(ln) == nn.LayerNorm else 1e-5


def _run_mask_blocks(blocks, V_emb, V_hidden, sink=None, snapshot=None, first_layer=0, want_aux=False):
    """The outputs of `blocks` (same act, dropout, LayerNorm and output width) on (V_emb, V_hidden), side by side.
    sink: the EmbeddingGrad of a shared_grad view V_emb; None: a view and buffer of these blocks alone.
    V_hidden is V_emb: the blocks' input gradient goes to V_emb's buffer too."""
    same = V_hidden is V_emb
    if sink is None:
        V_emb, sink = F2.shared_grad(V_emb)
    p = blocks[0].dropout_rate()
    if p > 0 and snapshot is None:
        snapshot, first_layer = F2.dropout_snapshot(V_emb.device, len(blocks)), 0
    return F2.mask_blocks(V_emb, sink, None if same else V_hidden, [b.block_params() for b in blocks], blocks[0]._act,
                          eps=_masknet_eps(blocks), dropout=p, snapshot=snapshot, first_layer=first_layer,
                          want_aux=want_aux)


class SerialMaskNet(nn.Module):
    """MaskNet.py, SerialMaskNet: MaskBlocks chained over [input_dim] + hidden_units, every block's mask MLP reading
    V_emb, then fc = Linear(h_last, output_dim) -> output activation.  One dropout snapshot per forward: block i
    draws the mask of layer i."""

    def __init__(self, input_dim, output_dim=None, output_activation=None, hidden_units=[],
                 hidden_activations="ReLU", reduction_ratio=1, dropout_rates=0, layer_norm=True):
        super(SerialMaskNet, self).__init__()
        if not isinstance(dropout_rates, list):
            dropout_rates = [dropout_rates] * len(hidden_units)
        if not isinstance(hidden_activations, list):
            hidden_activations = [hidden_activations] * len(hidden_units)
        self.hidden_units = [input_dim] + hidden_units
        self.mask_blocks = nn.ModuleList()
        for idx in range(len(self.hidden_units) - 1):
            self.mask_blocks.append(MaskBlock(input_dim,
                                              self.hidden_units[idx],
                                              self.hidden_units[idx + 1],
                                              hidden_activations[idx],
                                              reduction_ratio,
                                              dropout_rates[idx],
                                              layer_norm))
        fc_layers = []
        if output_dim is not None:
            fc_layers.append(nn.Linear(self.hidden_units[-1], output_dim))
        if output_activation is not None:
            fc_layers.append(get_activation(output_activation))
        self.fc = None
        if len(fc_layers) > 0:
            self.fc = nn.Sequential(*fc_layers)

    def blocks_out(self, V_emb, V_hidden, sink=None):
        """The last block's output (what fc reads)."""
        same = V_hidden is V_emb
        if sink is None:
            V_emb, sink = F2.shared_grad(V_emb)
        n_drop = sum(1 for b in self.mask_blocks if b.dropout_rate() > 0)
        snap = F2.dropout_snapshot(V_emb.device, n_drop) if n_drop else None
        v_out, ordinal = (V_emb if same else V_hidden), 0
        for blk in self.mask_blocks:
            v_out = _run_mask_blocks([blk], V_emb, v_out, sink, snap, ordinal)
            ordinal += 1 if blk.dropout_rate() > 0 else 0
        return v_out

    def forward(self, V_emb, V_hidden):
        v_out = self.blocks_out(V_emb, V_hidden)
        if self.fc is not None:
            lin = self.fc[0] if type(self.fc[0]) == nn.Linear else None
            if lin is not None:
                act = B2_ACT_SIGMOID if (len(self.fc) > 1 and type(self.fc[1]) == nn.Sigmoid) else B2_ACT_NONE
                v_out = F2.linear_act(v_out, lin.weight, lin.bias, act)
                rest = list(self.fc)[2 if act != B2_ACT_NONE else 1:]
            else:
                rest = list(self.fc)
            for m in rest:
                v_out = m(v_out)
        return v_out


class ParallelMaskNet(nn.Module):
    """MaskNet.py, ParallelMaskNet: num_blocks MaskBlock(input_dim, input_dim, block_dim) on the same (V_emb,
    V_hidden), concatenated, then MLP_Block to output_dim.  The blocks run as one autograd node that writes each
    output straight into its column slice of the concatenation, with the MLP's first-GEMM operand copy."""

    def __init__(self, input_dim, output_dim=None, output_activation=None, num_blocks=1, block_dim=64,
                 hidden_units=[], hidden_activations="ReLU", reduction_ratio=1, dropout_rates=0,
                 layer_norm=True):
        super(ParallelMaskNet, self).__init__()
        self.num_blocks = num_blocks
        self.mask_blocks = nn.ModuleList([MaskBlock(input_dim,
                                                    input_dim,
                                                    block_dim,
                                                    hidden_activations,
                                                    reduction_ratio,
                                                    dropout_rates,
                                                    layer_norm) for _ in range(num_blocks)])

        self.dnn = MLP_Block(input_dim=block_dim * num_blocks,
                             output_dim=output_dim,
                             hidden_units=hidden_units,
                             hidden_activations=hidden_activations,
                             output_activation=output_activation,
                             dropout_rates=dropout_rates)

    def blocks_out(self, V_emb, V_hidden, sink=None):
        """The concatenated block outputs (what dnn reads)."""
        return _run_mask_blocks(list(self.mask_blocks), V_emb, V_hidden, sink, want_aux=True)

    def forward(self, V_emb, V_hidden):
        return self.dnn(self.blocks_out(V_emb, V_hidden))


class FeatureSelection(nn.Module):
    """FinalMLP's feature selection (model_zoo/FinalMLP/src/FinalMLP.py, FeatureSelection): per stream s, a gate MLP
    ending in a sigmoid gives g_s and the stream's input is flat_emb * (2 g_s).  A stream without context features
    feeds its gate the learned row fs<s>_ctx_bias; the reference repeats that row over the batch, here the gate MLP
    runs once on the one row and the gating kernel broadcasts it (functional._FsGate).  Children and initial draws in
    the reference's order."""

    def __init__(self, feature_map, feature_dim, embedding_dim, fs_hidden_units=[], fs1_context=[], fs2_context=[]):
        super(FeatureSelection, self).__init__()
        self.fs1_context = fs1_context
        if len(fs1_context) == 0:
            self.fs1_ctx_bias = nn.Parameter(torch.zeros(1, embedding_dim))
        else:
            self.fs1_ctx_emb = FeatureEmbedding(feature_map, embedding_dim, required_feature_columns=fs1_context)
        self.fs2_context = fs2_context
        if len(fs2_context) == 0:
            self.fs2_ctx_bias = nn.Parameter(torch.zeros(1, embedding_dim))
        else:
            self.fs2_ctx_emb = FeatureEmbedding(feature_map, embedding_dim, required_feature_columns=fs2_context)
        self.fs1_gate = MLP_Block(input_dim=embedding_dim * max(1, len(fs1_context)), output_dim=feature_dim,
                                  hidden_units=fs_hidden_units, hidden_activations="ReLU", output_activation="Sigmoid",
                                  batch_norm=False)
        self.fs2_gate = MLP_Block(input_dim=embedding_dim * max(1, len(fs2_context)), output_dim=feature_dim,
                                  hidden_units=fs_hidden_units, hidden_activations="ReLU", output_activation="Sigmoid",
                                  batch_norm=False)

    def forward(self, X, flat_emb):
        if len(self.fs1_context) == 0:
            g1 = self.fs1_gate(self.fs1_ctx_bias)
        else:
            g1 = self.fs1_gate(self.fs1_ctx_emb(X, flatten_emb=True))
        if len(self.fs2_context) == 0:
            g2 = self.fs2_gate(self.fs2_ctx_bias)
        else:
            g2 = self.fs2_gate(self.fs2_ctx_emb(X, flatten_emb=True))
        return F2.fs_gate(flat_emb, g1, g2)


class InteractionAggregation(nn.Module):
    """FinalMLP's fusion of its two towers (model_zoo/FinalMLP/src/FinalMLP.py, InteractionAggregation):
    w_x(x) + w_y(y) + the multi-head bilinear sum_h x_h^T W_h y_h, one autograd node (functional.
    _InteractionAggregation).  `w_xy` gets its xavier draw here, as in the reference; a model's reset_parameters
    re-draws only the two Linears.  FinalMLP builds it with output_dim 1 only, the one width implemented."""

    def __init__(self, x_dim, y_dim, output_dim=1, num_heads=1):
        super(InteractionAggregation, self).__init__()
        assert x_dim % num_heads == 0 and y_dim % num_heads == 0, \
            "Input dim must be divisible by num_heads!"
        if output_dim != 1:
            raise NotImplementedError("InteractionAggregation is implemented for output_dim 1 (FinalMLP's), got %r"
                                      % (output_dim,))
        self.num_heads = num_heads
        self.output_dim = output_dim
        self.head_x_dim = x_dim // num_heads
        self.head_y_dim = y_dim // num_heads
        self.w_x = nn.Linear(x_dim, output_dim)
        self.w_y = nn.Linear(y_dim, output_dim)
        self.w_xy = nn.Parameter(torch.Tensor(num_heads * self.head_x_dim * self.head_y_dim, output_dim))
        nn.init.xavier_normal_(self.w_xy)

    def forward(self, x, y):
        return F2.interaction_aggregation(x, y, self.w_x.weight, self.w_x.bias, self.w_y.weight, self.w_y.bias,
                                          self.w_xy, self.num_heads)


# --------------------------------------------------------------------------------------
# CIN
# --------------------------------------------------------------------------------------
class CompressedInteractionNet(nn.Module):
    """compressed_interaction_net.py:23-76.  Layer k is a 1x1 Conv1d over the F * H_{k-1} outer-product
    channels (H_0 = F); `fc` over the concatenated sum-pooled maps is registered first."""

    def __init__(self, num_fields, cin_hidden_units, output_dim=1):
        super(CompressedInteractionNet, self).__init__()
        self.cin_hidden_units = cin_hidden_units
        self.fc = nn.Linear(sum(cin_hidden_units), output_dim)
        self.cin_layer = nn.ModuleDict()
        width_in = num_fields
        for k, width_out in enumerate(cin_hidden_units, start=1):
            self.cin_layer["layer_%d" % k] = nn.Conv1d(num_fields * width_in, width_out, kernel_size=1)
            width_in = width_out

    def forward(self, feature_emb):
        return F2.cin_forward(feature_emb,
                              [self.cin_layer["layer_" + str(i + 1)] for i in range(len(self.cin_hidden_units))],
                              self.fc)


# --------------------------------------------------------------------------------------
# Dice / MLP / DIN attention
# --------------------------------------------------------------------------------------
class Dice(nn.Module):
    """activations.py:24-51: p = sigmoid(BN(x)) with a non-affine BatchNorm1d(eps, momentum 0.01);
    out = p x + alpha (1 - p) x.  Statistics + gate are one kernel each way."""

    def __init__(self, input_dim, eps=1e-9):
        super(Dice, self).__init__()
        self.bn = nn.BatchNorm1d(input_dim, affine=False, eps=eps, momentum=0.01)
        self.alpha = nn.Parameter(torch.zeros(input_dim))

    def forward(self, X):
        return F2.dice_forward(X, self.bn, self.alpha, self.training)


class MLP_Block(nn.Module):
    """mlp_block.py:24-96.  `self.mlp` is the reference's Sequential: optional leading BatchNorm1d
    (`bn_only_once`), then per hidden layer Linear -> [BatchNorm1d] -> [activation] -> [Dropout], then the
    optional output Linear and output activation — module order fixes state_dict keys and init order."""

    def __init__(self, input_dim, hidden_units=[], hidden_activations="ReLU", output_dim=None,
                 output_activation=None, dropout_rates=0.0, batch_norm=False, bn_only_once=False,
                 use_bias=True):
        super(MLP_Block, self).__init__()
        depth = len(hidden_units)
        rates = dropout_rates if isinstance(dropout_rates, list) else [dropout_rates] * depth
        names = hidden_activations if isinstance(hidden_activations, list) else [hidden_activations] * depth
        acts = get_activation(names, hidden_units)
        widths = [input_dim] + hidden_units
        stack = [nn.BatchNorm1d(input_dim)] if (batch_norm and bn_only_once) else []
        for k in range(depth):
            stack.append(nn.Linear(widths[k], widths[k + 1], bias=use_bias))
            if batch_norm and not bn_only_once:
                stack.append(nn.BatchNorm1d(widths[k + 1]))
            if acts[k]:
                stack.append(acts[k])
            if rates[k] > 0:
                stack.append(nn.Dropout(p=rates[k]))
        if output_dim is not None:
            stack.append(nn.Linear(widths[-1], output_dim, bias=use_bias))
        if output_activation is not None:
            stack.append(get_activation(output_activation))
        self.mlp = nn.Sequential(*stack)

    def chain_layers(self):
        """The stack as F2.mlp_chain layers when it is Linear -> [ReLU|Sigmoid] -> [Dropout(0 < p < 1)] throughout,
        else None.  A Dropout in training mode passes its p to the chain (the mask of the chain's epilogues); in
        eval mode it is the identity and the plain chain runs."""
        mods = list(self.mlp)
        layers, i = [], 0
        while i < len(mods):
            if type(mods[i]) != nn.Linear:
                return None
            act = B2_ACT_NONE
            if i + 1 < len(mods) and type(mods[i + 1]) == nn.ReLU:
                act = B2_ACT_RELU
            elif i + 1 < len(mods) and type(mods[i + 1]) == nn.Sigmoid:
                act = B2_ACT_SIGMOID
            layer = (mods[i].weight, mods[i].bias, act)
            i += 2 if act != B2_ACT_NONE else 1
            if i < len(mods) and type(mods[i]) == nn.Dropout:
                if not 0.0 < mods[i].p < 1.0:
                    return None
                if mods[i].training:
                    layer += (mods[i].p,)
                i += 1
            layers.append(layer)
        return layers or None

    def forward(self, inputs):
        mods = list(self.mlp)
        x = inputs
        if F2.mlp_chain_supported() and inputs.is_cuda:
            # such a stack runs as ONE autograd node (cross-layer epilogue fusion)
            layers = self.chain_layers()
            if layers is not None:
                return F2.mlp_chain(x, layers)
        i = 0
        while i < len(mods):
            m = mods[i]
            if type(m) == nn.Linear:
                act = B2_ACT_NONE
                if i + 1 < len(mods) and type(mods[i + 1]) == nn.ReLU:
                    act = B2_ACT_RELU
                elif i + 1 < len(mods) and type(mods[i + 1]) == nn.Sigmoid:
                    act = B2_ACT_SIGMOID
                x = F2.linear_act(x, m.weight, m.bias, act)   # Linear + activation fused
                i += 2 if act != B2_ACT_NONE else 1
            else:
                # BatchNorm1d / Dropout / PReLU / Tanh ...: applied as the reference does
                # (mlp_block.py:72-80); Dice dispatches to its own kernel.
                x = m(x)
                i += 1
        return x


class DIN_Attention(nn.Module):
    """target_attention.py:26-92: scores = MLP([t, h, t-h, t*h]) per history position, masked (optionally
    softmaxed), weighted sum of the history.  "Dice" builds one Dice per attention layer."""

    def __init__(self, embedding_dim=64, attention_units=[32], hidden_activations="ReLU", output_activation=None,
                 dropout_rate=0, batch_norm=False, use_softmax=False):
        super(DIN_Attention, self).__init__()
        self.embedding_dim = embedding_dim
        self.use_softmax = use_softmax
        if isinstance(hidden_activations, str) and hidden_activations.lower() == "dice":
            hidden_activations = [Dice(width) for width in attention_units]
        self.attention_layer = MLP_Block(input_dim=4 * embedding_dim, output_dim=1, hidden_units=attention_units,
                                         hidden_activations=hidden_activations, output_activation=output_activation,
                                         dropout_rates=dropout_rate, batch_norm=batch_norm)

    def forward(self, target_item, history_sequence, mask=None):
        return F2.din_attention(self, target_item, history_sequence, mask)


class ScaledDotProductAttention(nn.Module):
    """dot_product_attention.py:24-58, as a child of MultiHeadTargetAttention: the same constructor and
    `dropout` child.  Its arithmetic runs inside MultiHeadTargetAttention's kernels, which fold the
    projections around it; on its own it has no kernel and raises."""

    def __init__(self, dropout_rate=0.):
        super(ScaledDotProductAttention, self).__init__()
        self.dropout = nn.Dropout(dropout_rate) if dropout_rate > 0 else None

    def forward(self, Q, K, V, scale=None, mask=None):
        raise NotImplementedError("ScaledDotProductAttention runs on the kernels only inside "
                                  "MultiHeadTargetAttention")


class MultiHeadTargetAttention(nn.Module):
    """target_attention.py:95-172: the target item attends over its history, per head, with optional Q, K, V, O
    projections.  One autograd node (functional._TargetAttention): with the projections, two GEMMs on weights
    folded per head around the row kernel, so the history is never projected; without them, the row kernel
    alone.  Parameters, child names, registration order and initialisation draws are the reference's.
    Attention dropout in training mode has no kernel and raises."""

    def __init__(self, input_dim=64, attention_dim=64, num_heads=1, dropout_rate=0, use_scale=True, use_qkvo=True):
        super(MultiHeadTargetAttention, self).__init__()
        if not use_qkvo:
            attention_dim = input_dim
        assert attention_dim % num_heads == 0, \
            "attention_dim={} is not divisible by num_heads={}".format(attention_dim, num_heads)
        bound = F2.target_attention_bound(num_heads * input_dim if use_qkvo else input_dim, num_heads)
        if bound is not None:
            raise NotImplementedError("MultiHeadTargetAttention kernels: " + bound)
        self.num_heads = num_heads
        self.head_dim = attention_dim // num_heads
        self.scale = self.head_dim ** 0.5 if use_scale else None
        self.use_qkvo = use_qkvo
        if use_qkvo:
            self.W_q = nn.Linear(input_dim, attention_dim, bias=False)
            self.W_k = nn.Linear(input_dim, attention_dim, bias=False)
            self.W_v = nn.Linear(input_dim, attention_dim, bias=False)
            self.W_o = nn.Linear(attention_dim, input_dim, bias=False)
        self.dot_attention = ScaledDotProductAttention(dropout_rate)

    def forward(self, target_item, history_sequence, mask=None):
        if self.dot_attention.dropout is not None and self.training:
            raise NotImplementedError("MultiHeadTargetAttention kernels: attention dropout in training mode "
                                      "has no kernel")
        weights = (self.W_q.weight, self.W_k.weight, self.W_v.weight, self.W_o.weight) if self.use_qkvo else ()
        return F2.target_attention(target_item, history_sequence, mask, self.num_heads, self.scale is not None,
                                   *weights)


class MultiHeadTopKAttention(nn.Module):
    """model_zoo/LongCTR/TWIN/TWIN.py, MultiHeadTopKAttention: per head, the target scores the whole history, the top k
    scores are kept and softmaxed, and their values are pooled.  The constructor, its assert, the children W_q, W_h,
    W_v, W_o (registration order, state_dict keys, initial draws) and `dropout` are the reference's.  It runs inside
    TWIN's interest block, one autograd node on the kernels (functional.twin_interest); Kc > 0 (cross features, which
    the reference can only broadcast at L = 1) and attention dropout have no kernel and raise."""

    def __init__(self, input_dim=64, Kc=0, embedding_dim=16, attention_dim=64, topk=50, num_heads=1, dropout_rate=0):
        super(MultiHeadTopKAttention, self).__init__()
        assert attention_dim % num_heads == 0, \
            "attention_dim={} is not divisible by num_heads={}".format(attention_dim, num_heads)
        if Kc > 0:
            raise NotImplementedError("MultiHeadTopKAttention kernels: Kc_cross_features > 0 is not supported: the "
                                      "reference's cross_feat_seq.view(B, Kc, -1) * W_c broadcasts only at L = 1")
        if dropout_rate:
            raise NotImplementedError("MultiHeadTopKAttention kernels: attention dropout has no kernel")
        self.num_heads = num_heads
        self.topk = topk
        self.head_dim = attention_dim // num_heads
        self.scale = self.head_dim ** 0.5
        self.Kc = Kc
        self.Kc_dim = 0
        self.Kh_dim = input_dim
        self.W_q = nn.Linear(input_dim, attention_dim, bias=False)
        self.W_h = nn.Linear(input_dim, attention_dim, bias=False)
        self.W_v = nn.Linear(input_dim, attention_dim, bias=False)
        self.W_o = nn.Linear(attention_dim, input_dim, bias=False)
        self.dropout = None

    def weights(self):
        return self.W_q.weight, self.W_h.weight, self.W_v.weight, self.W_o.weight

    def forward(self, target_item, item_sequence, mask=None):
        raise NotImplementedError("MultiHeadTopKAttention runs inside TWIN's interest block: call "
                                  "functional.twin_interest on item_feat_emb (B, L + 1, d) with the target last")


class FilterLayer2(nn.Module):
    """model_zoo/LongCTR/MIRRN/MIRRN.py, FilterLayer2: LN(dropout(irfft(rfft(u) W, n=k)) + u) over the k retrieved rows
    u (B, k, d), FFTs along the slot axis.  The reference's einsum keeps the diagonal of each of the n_block blocks of
    complex_weight, so the filter is one complex weight per channel and needs no FFT on the device
    (functional.mirrn_filter_table).  complex_weight (n_block, d / n_block, d / n_block, 2), out_dropout and the
    TF-style LayerNorm child (eps 1e-12, nn.LayerNorm's formula) keep the reference's registration order, state_dict
    keys and initial draws.  It runs inside MIRRN's interest block (functional.mirrn_interest), which needs
    n_block = 4."""

    def __init__(self, max_length, hidden_size, hidden_dropout_prob, n_block):
        super(FilterLayer2, self).__init__()
        if n_block != 4 or hidden_size % n_block:
            raise NotImplementedError("FilterLayer2 kernels: n_block must be 4 and divide hidden_size, got n_block %d, "
                                      "hidden_size %d" % (n_block, hidden_size))
        self.complex_weight = nn.Parameter(
            torch.randn(n_block, hidden_size // n_block, hidden_size // n_block, 2, dtype=torch.float32) * 0.02)
        self.out_dropout = nn.Dropout(hidden_dropout_prob)
        self.LayerNorm = nn.LayerNorm(hidden_size, eps=F2.MIRRN_LN_EPS)
        self.n = n_block

    def forward(self, input_tensor):
        raise NotImplementedError("FilterLayer2 runs inside MIRRN's interest block: call functional.mirrn_interest on "
                                  "item_feat_emb (B, L + 1, d) with the target last")


class MultiHeadSelfAttention(nn.Module):
    """model_zoo/AutoInt/src/AutoInt.py, MultiHeadSelfAttention: field-wise multi-head self-attention with an optional
    residual (X, or X W_res^T when input_dim != attention_dim), LayerNorm and a final ReLU.  One autograd node per layer
    (functional._SelfAttentionLayer): one GEMM on the stacked [W_q; W_k; W_v (; W_res)] and one row kernel that never
    writes the (B, H, F, F) attention weights.  The constructor, its assert, the children (`dot_attention` is the
    ScaledDotProductAttention mirror and holds the dropout), their registration order and initial draws are the
    reference's."""

    def __init__(self, input_dim, attention_dim=None, num_heads=1, dropout_rate=0., use_residual=True,
                 use_scale=False, layer_norm=False):
        super(MultiHeadSelfAttention, self).__init__()
        if attention_dim is None:
            attention_dim = input_dim
        assert attention_dim % num_heads == 0, \
            "attention_dim={} is not divisible by num_heads={}".format(attention_dim, num_heads)
        bound = F2.autoint_bound(1, attention_dim, num_heads)
        if bound is not None:
            raise NotImplementedError("MultiHeadSelfAttention kernels: " + bound)
        self.head_dim = attention_dim // num_heads
        self.num_heads = num_heads
        self.use_residual = use_residual
        self.scale = self.head_dim ** 0.5 if use_scale else None
        self.W_q = nn.Linear(input_dim, attention_dim, bias=False)
        self.W_k = nn.Linear(input_dim, attention_dim, bias=False)
        self.W_v = nn.Linear(input_dim, attention_dim, bias=False)
        if self.use_residual and input_dim != attention_dim:
            self.W_res = nn.Linear(input_dim, attention_dim, bias=False)
        else:
            self.W_res = None
        self.dot_attention = ScaledDotProductAttention(dropout_rate)
        self.layer_norm = nn.LayerNorm(attention_dim) if layer_norm else None

    def forward(self, X, snapshot=None, layer=0, want_aux=False):
        """X (B, F, input_dim) -> (B, F, attention_dim).  In training mode with dropout the attention weights take the
        mask of layer `layer` of `snapshot` (functional.dropout_snapshot; None: one of its own).  want_aux: also write
        the output's GEMM operand copy for a following layer."""
        drop = self.dot_attention.dropout
        p = drop.p if (drop is not None and self.training) else 0.0
        ln = self.layer_norm
        return F2.self_attention_layer(X, self.W_q.weight, self.W_k.weight, self.W_v.weight,
                                       self.W_res.weight if self.W_res is not None else None,
                                       num_heads=self.num_heads, use_residual=self.use_residual,
                                       use_scale=self.scale is not None,
                                       gamma=ln.weight if ln is not None else None,
                                       beta=ln.bias if ln is not None else None,
                                       eps=ln.eps if ln is not None else 1e-5, dropout=p, snapshot=snapshot,
                                       layer=layer, want_aux=want_aux)


class FactorizationMachineBlock(nn.Module):
    """model_zoo/WuKong/src/WuKong.py, FactorizationMachineBlock: the rank-k FM x (x^T proj_Y), its LayerNorm over
    F k and an MLP to fmb D with a ReLU output.  The constructor, its draws (proj_Y = randn(F, k), then the MLP's
    Linears), the children and their registration order are the reference's; the forward runs inside
    WuKongLayer.forward (functional.wukong_layer).  rank_k=None (the vanilla FM, F^2 wide) is refused."""

    def __init__(self, input_features=16, output_features=16, embedding_dim=16, rank_k=8, mlp_hidden_units=[16, 16],
                 mlp_hidden_activations="relu", mlp_dropout=0):
        super(FactorizationMachineBlock, self).__init__()
        if rank_k is None:
            raise NotImplementedError("FactorizationMachineBlock kernels: " + F2.wukong_bound(input_features,
                                                                                              output_features, 1, None))
        self.embedding_dim = embedding_dim
        self.output_features = output_features
        self.rank_k = rank_k
        self.input_features = input_features
        self.proj_Y = nn.Parameter(torch.randn(self.input_features, self.rank_k))
        fm_out_dim = input_features * rank_k
        self.layer_norm = nn.LayerNorm(fm_out_dim)
        self.mlp = MLP_Block(input_dim=fm_out_dim, output_dim=output_features * embedding_dim,
                             hidden_units=mlp_hidden_units, hidden_activations=mlp_hidden_activations,
                             output_activation="relu", dropout_rates=mlp_dropout)

    def first_linear(self):
        return next(m for m in self.mlp.mlp if type(m) == nn.Linear)


class LinearCompressionBlock(nn.Module):
    """model_zoo/WuKong/src/WuKong.py, LinearCompressionBlock: Linear(F -> lcb, bias=False) over the field axis; it
    runs as the LCB columns of WuKongLayer's field-axis GEMM."""

    def __init__(self, input_features=16, output_features=8):
        super(LinearCompressionBlock, self).__init__()
        self.linear = nn.Linear(input_features, output_features, bias=False)


class WuKongLayer(nn.Module):
    """model_zoo/WuKong/src/WuKong.py, WuKongLayer: out = [LayerNorm(D)](cat(FMB(x), LCB(x)) + residual), the residual
    x itself or, when input_features != lcb + fmb, residual_proj over the field axis.  Constructor, children, their
    registration order and draws are the reference's.  One layer is the FM row kernel, the FMB's MLP, one field-axis
    GEMM and the combine row kernel (functional.wukong_layer); between layers of a stack the activations stay in the
    (B D, fp) layout (forward_stack)."""

    def __init__(self, input_features=16, lcb_features=8, fmb_features=8, embedding_dim=16, fmp_rank_k=4,
                 fmb_mlp_units=[16, 16], fmb_mlp_activations="relu", fmb_dropout=0.1, layer_norm=True):
        super(WuKongLayer, self).__init__()
        bound = F2.wukong_bound(input_features, lcb_features + fmb_features, embedding_dim, fmp_rank_k)
        if bound is None and (lcb_features < 1 or fmb_features < 1):
            bound = "lcb_features and fmb_features must be at least 1, got %d and %d" % (lcb_features, fmb_features)
        if bound is not None:
            raise NotImplementedError("WuKongLayer kernels: " + bound)
        self.fmb = FactorizationMachineBlock(input_features, fmb_features, embedding_dim, fmp_rank_k, fmb_mlp_units,
                                             fmb_mlp_activations, fmb_dropout)
        self.lcb = LinearCompressionBlock(input_features, lcb_features)
        self.layer_norm = nn.LayerNorm(embedding_dim) if layer_norm else None
        if input_features != lcb_features + fmb_features:
            self.residual_proj = nn.Linear(input_features, lcb_features + fmb_features)

    def run(self, x, sink=None, last=True, want_aux=False):
        """functional.wukong_layer on x (the embedding (B, F, D), or X' with its shared_grad sink)."""
        fmb, ln = self.fmb, self.layer_norm
        res = getattr(self, "residual_proj", None)
        return F2.wukong_layer(x, fmb.proj_Y, fmb.layer_norm.weight, fmb.layer_norm.bias, fmb.mlp,
                               self.lcb.linear.weight, res.weight if res is not None else None,
                               res.bias if res is not None else None, ln.weight if ln is not None else None,
                               ln.bias if ln is not None else None, fm_eps=fmb.layer_norm.eps,
                               eps=ln.eps if ln is not None else 1e-5, embedding_dim=fmb.embedding_dim, sink=sink,
                               last=last, fm_aux=F2._tc_layer_ok(fmb.first_linear().weight), want_aux=want_aux)

    def forward(self, x):
        """x (B, F, D) -> (B, lcb + fmb, D)."""
        out = self.run(x)
        return out.view(x.shape[0], -1, self.fmb.embedding_dim)


def wukong_stack(layers, feature_emb, want_aux=False):
    """The WuKong layers `layers` on feature_emb (B, F, D) -> the last layer's (B, Fo D) flatten [b, f, d].  Between
    layers the activations stay as X' (B D, fp), whose gradient is one buffer (functional.shared_grad) that the
    combine backward, the dgrad and the FM backward all add into.  want_aux: the flatten's GEMM operand copy."""
    x, sink = feature_emb, None
    for i, layer in enumerate(layers):
        last = i + 1 == len(layers)
        if last:
            return layer.run(x, sink, last=True, want_aux=want_aux)
        nxt = layers[i + 1]
        res = getattr(nxt, "residual_proj", None)
        n = nxt.lcb.linear.weight.shape[0] + (res.weight.shape[0] if res is not None else 0)
        x = layer.run(x, sink, last=False, want_aux=F2._wukong_tc_shape(n, F2.wukong_pitch(nxt.fmb.input_features)))
        x, sink = F2.shared_grad(x)


# --------------------------------------------------------------------------------------
# FinalNet (model_zoo/FinalNet/src/FinalNet.py)
# --------------------------------------------------------------------------------------
def _finalnet_act(module):
    """The B2_ACT_* code of a FinalBlock activation module (get_activation's result), refusing what the kernels lack."""
    if module is None:
        return B2_ACT_NONE
    if type(module) == nn.ReLU:
        return B2_ACT_RELU
    if type(module) == nn.Sigmoid:
        return B2_ACT_SIGMOID
    raise NotImplementedError("FinalBlock kernels: activation %s is not supported (None, ReLU and Sigmoid are)"
                              % type(module).__name__)


class FeatureGating(nn.Module):
    """model_zoo/FinalNet/src/FinalNet.py, FeatureGating: gates = Linear(F, F) over the field axis, out =
    cat([e, e * gates], dim=1) (gate_residual "concat"; "sum" is refused).  init_weights sets the gate's weight to 0
    and its bias to 1, as the reference's.  One row kernel each way (functional.feature_gating)."""

    def __init__(self, num_fields, gate_residual="concat"):
        super(FeatureGating, self).__init__()
        self.linear = nn.Linear(num_fields, num_fields)
        assert gate_residual in ["concat", "sum"]
        if gate_residual != "concat":
            raise NotImplementedError("FeatureGating kernels: gate_residual='sum' is not supported ('concat' is)")
        self.gate_residual = gate_residual

    def init_weights(self):
        nn.init.zeros_(self.linear.weight)
        nn.init.ones_(self.linear.bias)

    def run(self, feature_emb, sink=None, want_aux=False):
        """(B, 2 F D): the flattened output block 1 reads; feature_emb (B, F, D), or its (B, F D) shared_grad view."""
        return F2.feature_gating(feature_emb, self.linear.weight, self.linear.bias, sink=sink, want_aux=want_aux)

    def forward(self, feature_emb):
        """(B, F, D) -> (B, 2 F, D)."""
        return self.run(feature_emb).view(feature_emb.shape[0], -1, feature_emb.shape[2])


class FactorizedInteraction(nn.Module):
    """model_zoo/FinalNet/src/FinalNet.py, FactorizedInteraction: h = Linear(x), h2, h1 = chunk(h, 2),
    cat([h2, h1 * h2]) (concat, which asserts an even output_dim) or h2 + h1 * h2 (sum, whose Linear is 2 output_dim
    wide).  One GEMM and one row kernel (functional.factorized_interaction)."""

    def __init__(self, input_dim, output_dim, bias=True, residual_type="sum"):
        super(FactorizedInteraction, self).__init__()
        self.residual_type = residual_type
        if residual_type == "sum":
            output_dim = output_dim * 2
        else:
            assert output_dim % 2 == 0, "output_dim should be divisible by 2."
        self.linear = nn.Linear(input_dim, output_dim, bias=bias)

    def forward(self, x):
        return F2.factorized_interaction(x, self.linear.weight, self.linear.bias, self.residual_type)


class FinalBlock(nn.Module):
    """model_zoo/FinalNet/src/FinalNet.py, FinalBlock: per layer FactorizedInteraction, then BatchNorm1d (the real
    nn.BatchNorm1d children, whose running statistics the kernels update in place), the activation and dropout.  As in
    the reference, layer i applies self.dropout[i] whenever there is one, and self.dropout only holds the rates > 0: per
    layer rates [0, 0.5] put the 0.5 after layer 0.  Activations: None, ReLU, Sigmoid; others are refused here."""

    def __init__(self, input_dim, hidden_units=[], hidden_activations=None, dropout_rates=[], batch_norm=True,
                 residual_type="sum"):
        super(FinalBlock, self).__init__()
        if type(dropout_rates) != list:
            dropout_rates = [dropout_rates] * len(hidden_units)
        if type(hidden_activations) != list:
            hidden_activations = [hidden_activations] * len(hidden_units)
        bound = F2.finalnet_bound(hidden_units)
        if bound is not None:
            raise NotImplementedError("FinalBlock kernels: " + bound)
        self.layer = nn.ModuleList()
        self.norm = nn.ModuleList()
        self.dropout = nn.ModuleList()
        self.activation = nn.ModuleList()
        hidden_units = [input_dim] + hidden_units
        for idx in range(len(hidden_units) - 1):
            self.layer.append(FactorizedInteraction(hidden_units[idx], hidden_units[idx + 1],
                                                    residual_type=residual_type))
            if batch_norm:
                self.norm.append(nn.BatchNorm1d(hidden_units[idx + 1]))
            if dropout_rates[idx] > 0:
                self.dropout.append(nn.Dropout(dropout_rates[idx]))
            self.activation.append(get_activation(hidden_activations[idx]))
        self._acts = [_finalnet_act(a) for a in self.activation]

    def run(self, X, sink=None, want_aux=False):
        """The block on X (B, input_dim); sink: X is a shared_grad view.  want_aux: the output's operand copy."""
        L = len(self.layer)
        rates = [self.dropout[i].p if len(self.dropout) > i else 0.0 for i in range(L)]
        snap = None
        if self.training and any(p > 0 for p in rates):
            snap = F2.dropout_snapshot(X.device, L)
        x = X
        for i in range(L):
            lin = self.layer[i].linear
            norm = (self.norm[i], self.norm[i].training) if len(self.norm) > i else None
            drop = (snap, i, rates[i]) if snap is not None and rates[i] > 0 else None
            aux = F2._tc_layer_ok(self.layer[i + 1].linear.weight) if i + 1 < L else want_aux
            x = F2.factorized_interaction(x, lin.weight, lin.bias, self.layer[i].residual_type,
                                          sink=sink if i == 0 else None, batch_norm=norm, act=self._acts[i],
                                          dropout=drop, want_aux=aux)
        return x

    def forward(self, X):
        return self.run(X)


class TransformerBlock(nn.Module):
    """model_zoo/BST/src/BST.py, TransformerBlock: s = LN1(x [+ dropout1(MHA(x))]), out = LN2(s [+ dropout2(FFN(s))]) with
    FFN = Linear -> LeakyReLU -> Linear.  `attention` is a real nn.MultiheadAttention and holds the projections
    (in_proj_weight = [W_q; W_k; W_v], in_proj_bias, out_proj) and the attention dropout; the kernels read it, its
    forward is never called.  On the kernels (run): the in-projection GEMM, the masked attention row kernel, the
    out-projection GEMM, the residual + dropout + LayerNorm row kernel, the FFN as one MLP chain with LeakyReLU
    (B2_ACT_LEAKY_RELU) in its first epilogue and dropout2 in its second, and the residual + LayerNorm row kernel.
    Constructor, children, registration order and initial draws are the reference's."""

    def __init__(self, model_dim=64, ffn_dim=64, num_heads=8, attn_dropout=0.0, net_dropout=0.0, layer_norm=True,
                 use_residual=True):
        super(TransformerBlock, self).__init__()
        self.attention = nn.MultiheadAttention(model_dim, num_heads=num_heads, dropout=attn_dropout, batch_first=True)
        self.ffn = nn.Sequential(nn.Linear(model_dim, ffn_dim), nn.LeakyReLU(), nn.Linear(ffn_dim, model_dim))
        self.use_residual = use_residual
        self.dropout1 = nn.Dropout(net_dropout)
        self.dropout2 = nn.Dropout(net_dropout)
        self.layer_norm1 = nn.LayerNorm(model_dim) if layer_norm else None
        self.layer_norm2 = nn.LayerNorm(model_dim) if layer_norm else None

    def _p(self, drop):
        return drop.p if (drop.training and drop.p > 0) else 0.0

    def run(self, x, valid, batch, seq_len, causal=False, snapshot=None, layer=0, want_aux=False):
        """x (B L, model_dim) -> (B L, model_dim).  valid (B, L - 1) uint8: 1 for a real history slot.  In training
        mode with dropout the attention weights take the mask of layer `layer` of `snapshot` and dropout1 that of
        layer + 1 (functional.dropout_snapshot; None: their own); dropout2 is the MLP chain's, drawn from the chain's
        own snapshot (its layer 0).  want_aux: also
        write the output's GEMM operand copy for a following block.  An empty batch makes no launch."""
        att = self.attention
        if not isinstance(self.ffn[1], nn.LeakyReLU) or self.ffn[1].negative_slope != 0.01:
            raise NotImplementedError("TransformerBlock kernels: the FFN activation must be nn.LeakyReLU(0.01)")
        if batch == 0:
            return x.view_as(x)
        ln1, ln2 = self.layer_norm1, self.layer_norm2
        W1, W2 = self.ffn[0], self.ffn[2]
        qkv = F2.linear_act(x, att.in_proj_weight, att.in_proj_bias)
        ctx = F2.bst_attention(qkv, valid, batch, seq_len, att.num_heads, causal=causal,
                               dropout=att.dropout if self.training else 0.0, snapshot=snapshot, layer=layer,
                               want_aux=F2._tc_layer_ok(att.out_proj.weight))
        attn = F2.linear_act(ctx, att.out_proj.weight, att.out_proj.bias)
        s = F2.bst_add_norm(attn, x if self.use_residual else None, ln1.weight if ln1 is not None else None,
                            ln1.bias if ln1 is not None else None, ln1.eps if ln1 is not None else 1e-5,
                            dropout=self._p(self.dropout1), snapshot=snapshot, layer=layer + 1,
                            want_aux=F2._tc_layer_ok(W1.weight))
        p2 = self._p(self.dropout2)
        f = F2.mlp_chain(s, [(W1.weight, W1.bias, B2_ACT_LEAKY_RELU), (W2.weight, W2.bias, B2_ACT_NONE, p2)])
        return F2.bst_add_norm(f, s if self.use_residual else None, ln2.weight if ln2 is not None else None,
                               ln2.bias if ln2 is not None else None, ln2.eps if ln2 is not None else 1e-5,
                               want_aux=want_aux)

    def forward(self, x, attn_mask=None):
        raise NotImplementedError("TransformerBlock runs on the kernels through run(x, valid, ...), which takes the "
                                  "key-padding mask as a (B, L - 1) byte mask instead of a (B H, L, L) attn_mask")


class BehaviorTransformer(nn.Module):
    """model_zoo/BST/src/BST.py, BehaviorTransformer: [tokens | position_emb] through stacked TransformerBlocks.
    position_emb (seq_len, position_dim) is a trained parameter initialised sinusoidally by its own reset_parameters
    (RankModel.reset_parameters does not touch it).  In training mode with dropout the blocks draw their attention and
    dropout1 masks from one dropout snapshot, two layers per block (each FFN chain takes a snapshot of its own)."""

    def __init__(self, seq_len=1, model_dim=64, num_heads=8, stacked_transformer_layers=1, attn_dropout=0.0,
                 net_dropout=0.0, use_position_emb=True, position_dim=4, layer_norm=True, use_residual=True):
        super(BehaviorTransformer, self).__init__()
        self.position_dim = position_dim
        self.use_position_emb = use_position_emb
        self.transformer_blocks = nn.ModuleList(TransformerBlock(model_dim=model_dim, ffn_dim=model_dim,
                                                                 num_heads=num_heads, attn_dropout=attn_dropout,
                                                                 net_dropout=net_dropout, layer_norm=layer_norm,
                                                                 use_residual=use_residual)
                                                for _ in range(stacked_transformer_layers))
        if self.use_position_emb:
            self.position_emb = nn.Parameter(torch.Tensor(seq_len, position_dim))
            self.reset_parameters()

    def reset_parameters(self):
        """The sinusoidal table: pe[t, 2k] = sin(t w_k), pe[t, 2k + 1] = cos(t w_k), w_k = 10000^(-2k / dim)."""
        seq_len = self.position_emb.size(0)
        pe = torch.zeros(seq_len, self.position_dim)
        position = torch.arange(0, seq_len).float().unsqueeze(1)
        freq = torch.exp(torch.arange(0, self.position_dim, 2).float() * (-np.log(10000.0) / self.position_dim))
        pe[:, 0::2] = torch.sin(position * freq)
        pe[:, 1::2] = torch.cos(position * freq)
        self.position_emb.data = pe

    def run(self, sequence_embs, target_embs, valid, causal=False, want_aux=False):
        """The (B L, model_dim) output of the stack on one (target, sequence) pair: sequence_embs the nf (B, L - 1, D)
        embeddings of the sequence fields, target_embs the nf (B, D) ones of the target fields, valid (B, L - 1)
        uint8.  want_aux: also write the output's GEMM operand copy."""
        blocks = list(self.transformer_blocks)
        B, Lm1 = valid.shape
        L = Lm1 + 1
        x = F2.bst_tokens(sequence_embs, target_embs, self.position_emb if self.use_position_emb else None,
                          want_aux=bool(blocks) and F2._tc_layer_ok(blocks[0].attention.in_proj_weight))
        snap = None
        if self.training and blocks and (blocks[0].attention.dropout > 0 or blocks[0]._p(blocks[0].dropout1) > 0):
            snap = F2.dropout_snapshot(x.device, 2 * len(blocks))
        for k, blk in enumerate(blocks):
            last = k + 1 == len(blocks)
            x = blk.run(x, valid, B, L, causal=causal, snapshot=snap, layer=2 * k,
                        want_aux=want_aux if last else F2._tc_layer_ok(blocks[k + 1].attention.in_proj_weight))
        return x

    def forward(self, x, attn_mask=None):
        raise NotImplementedError("BehaviorTransformer runs on the kernels through run(sequence_embs, target_embs, "
                                  "valid)")


class TransActTransformer(nn.Module):
    """model_zoo/TransAct/src/TransAct.py, TransActTransformer: the early-fusion tokens [sequence | target] of the L
    slots through a post-norm nn.TransformerEncoder with a key-padding mask (an empty history keeps its last slot),
    the output zeroed at padded slots, then [last first_k_cols slots | out_linear(max over L)].
    `transformer_encoder` is a real nn.TransformerEncoder and holds the parameters (its layers start as copies of one
    layer, as in the reference); its forward is never called.  On the kernels (run), each layer is the in-projection
    GEMM, the key-tiled attention (functional.transact_attention), out_proj, the residual + dropout1 + norm1 row
    kernel, the FFN as one MLP chain (ReLU and the inner dropout in its first epilogue, dropout2 in its second) and the
    residual + norm2 row kernel.  Refused: use_time_window_mask=True (the reference's forward never passes
    time_interval_seq, so it cannot train)."""

    def __init__(self, transformer_in_dim, dim_feedforward=64, num_heads=1, dropout=0, transformer_layers=1,
                 use_time_window_mask=False, time_window_ms=86400000, first_k_cols=1, concat_max_pool=True):
        super(TransActTransformer, self).__init__()
        if use_time_window_mask:
            raise NotImplementedError("TransAct use_time_window_mask=True is not supported: the reference's forward "
                                      "never passes time_interval_seq, so its mask compares None with an int")
        self.use_time_window_mask = use_time_window_mask
        self.time_window_ms = time_window_ms
        self.concat_max_pool = concat_max_pool
        self.first_k_cols = first_k_cols
        encoder_layer = nn.TransformerEncoderLayer(d_model=transformer_in_dim, nhead=num_heads,
                                                   dim_feedforward=dim_feedforward, dropout=dropout, batch_first=True)
        self.transformer_encoder = nn.TransformerEncoder(encoder_layer, num_layers=transformer_layers)
        if self.concat_max_pool:
            self.out_linear = nn.Linear(transformer_in_dim, transformer_in_dim)

    @staticmethod
    def _p(drop):
        return drop.p if (drop.training and drop.p > 0) else 0.0

    def run_layers(self, x, valid, batch, seq_len, want_aux=False):
        """The encoder stack on the tokens x (B L, md) with the adjusted mask valid (B, L) uint8.  Rows of padded slots
        come out finite but not the reference's: the model zeroes them.  In training mode with dropout, layer k's
        attention weights take the mask of snapshot layer 2 k and its dropout1 that of 2 k + 1; the FFN chains draw
        their own."""
        lyrs = list(self.transformer_encoder.layers)
        if batch == 0 or not lyrs:
            return x
        snap = None
        if self.training and (lyrs[0].self_attn.dropout > 0 or self._p(lyrs[0].dropout1) > 0):
            snap = F2.dropout_snapshot(x.device, 2 * len(lyrs))
        for k, lyr in enumerate(lyrs):
            if lyr.norm_first or lyr.activation_relu_or_gelu != 1:
                raise NotImplementedError("TransActTransformer kernels: post-norm layers with ReLU only")
            att = lyr.self_attn
            last = k + 1 == len(lyrs)
            qkv = F2.linear_act(x, att.in_proj_weight, att.in_proj_bias)
            ctx = F2.transact_attention(qkv, valid, batch, seq_len, att.num_heads,
                                        dropout=att.dropout if self.training else 0.0, snapshot=snap, layer=2 * k,
                                        want_aux=F2._tc_layer_ok(att.out_proj.weight))
            a = F2.linear_act(ctx, att.out_proj.weight, att.out_proj.bias)
            s = F2.bst_add_norm(a, x, lyr.norm1.weight, lyr.norm1.bias, lyr.norm1.eps, dropout=self._p(lyr.dropout1),
                                snapshot=snap, layer=2 * k + 1, want_aux=F2._tc_layer_ok(lyr.linear1.weight))
            p0, p2 = self._p(lyr.dropout), self._p(lyr.dropout2)
            f = F2.mlp_chain(s, [(lyr.linear1.weight, lyr.linear1.bias, B2_ACT_RELU) + ((p0,) if p0 > 0 else ()),
                                 (lyr.linear2.weight, lyr.linear2.bias, B2_ACT_NONE) + ((p2,) if p2 > 0 else ())])
            nxt = want_aux if last else F2._tc_layer_ok(lyrs[k + 1].self_attn.in_proj_weight)
            x = F2.bst_add_norm(f, s, lyr.norm2.weight, lyr.norm2.bias, lyr.norm2.eps, want_aux=nxt)
        return x

    def run(self, sequence_embs, target_embs, ids):
        """The (B, (first_k_cols + concat_max_pool) md) output on one (target, sequence) pair: sequence_embs the ns
        (B, L, D) embeddings of the sequence fields, target_embs the nt (B, D) ones of the target fields, ids (B, L)
        the first sequence field's ids (0 = padding)."""
        lyrs = list(self.transformer_encoder.layers)
        B, L = ids.shape[0], ids.shape[1]
        x, valid = F2.transact_tokens(sequence_embs, target_embs, ids,
                                      want_aux=bool(lyrs) and F2._tc_layer_ok(lyrs[0].self_attn.in_proj_weight))
        y = self.run_layers(x, valid, B, L)
        if not self.concat_max_pool:
            return F2.transact_output(y, valid, B, L, self.first_k_cols, max_pool=False)
        last, maxv = F2.transact_output(y, valid, B, L, self.first_k_cols, max_pool=True,
                                        want_aux=F2._tc_layer_ok(self.out_linear.weight))
        return torch.cat([last, F2.linear_act(maxv, self.out_linear.weight, self.out_linear.bias)], dim=-1)

    def forward(self, target_emb, sequence_emb, time_interval_seq=None, mask=None):
        raise NotImplementedError("TransActTransformer runs on the kernels through run(sequence_embs, target_embs, ids)")


class AGRUCell(nn.Module):
    """model_zoo/DIEN/src/DIEN.py, AGRUCell: h' = h + a (n - h), r = s(i_r + h_r), n = tanh(i_n + r h_n), with the
    chunks u, r, n of x2h(x) and h2h(h) (u unused).  The kernels read x2h and h2h (functional.gru_sequence)."""

    def __init__(self, input_size, hidden_size, bias=True):
        super(AGRUCell, self).__init__()
        self.x2h = nn.Linear(input_size, 3 * hidden_size, bias=bias)
        self.h2h = nn.Linear(hidden_size, 3 * hidden_size, bias=bias)

    def forward(self, x, hx, attn):
        raise NotImplementedError("AGRUCell runs over whole sequences on the kernels (DynamicGRU.run)")


class AUGRUCell(AGRUCell):
    """model_zoo/DIEN/src/DIEN.py, AUGRUCell: h' = h + a s(i_u + h_u) (n - h), r and n as AGRUCell's."""

    def forward(self, x, hx, attn):
        raise NotImplementedError("AUGRUCell runs over whole sequences on the kernels (DynamicGRU.run)")


class DynamicGRU(nn.Module):
    """model_zoo/DIEN/src/DIEN.py, DynamicGRU with an AUGRU or AGRU cell: the recurrence over each sample's first len
    positions from h = 0, one kernel launch each way (functional.gru_sequence) instead of a Python loop over time."""

    def __init__(self, input_size, hidden_size, bias=True, gru_type="AUGRU"):
        super(DynamicGRU, self).__init__()
        self.hidden_size = hidden_size
        self.gru_type = gru_type
        if gru_type == "AUGRU":
            self.gru_cell = AUGRUCell(input_size, hidden_size, bias=bias)
        elif gru_type == "AGRU":
            self.gru_cell = AGRUCell(input_size, hidden_size, bias=bias)

    def run(self, x, mask, attn, sink=None):
        """h_last (B, H) of the cell over x (B, L, H) with the attention attn (B, L); mask (B, L) uint8 gives the
        lengths.  sink: x is a shared_grad view (functional.gru_sequence)."""
        cell = self.gru_cell
        if cell.x2h.bias is None or cell.h2h.bias is None:
            raise NotImplementedError("DynamicGRU kernels: the cell's Linears need their biases (bias=True)")
        return F2.gru_sequence(x, mask, cell.x2h.weight, cell.x2h.bias, cell.h2h.weight, cell.h2h.bias,
                               cell=self.gru_type, att=attn, sink=sink)[1]

    def forward(self, packed_seq_emb, attn_score=None, h=None):
        raise NotImplementedError("DynamicGRU runs on the kernels through run(x, mask, attn), which takes padded "
                                  "sequences and a mask instead of PackedSequences")


class AttentionLayer(nn.Module):
    """model_zoo/DIEN/src/DIEN.py, AttentionLayer: the scores of the interests against the target, times the mask,
    optionally softmaxed.  bilinear_attention <h_t, W_kernel t> and dot_attention <h_t, t> are one kernel each way
    (functional.dien_scores); din_attention is the DIN input kernel, attn_mlp (an MLP_Block) and the masked softmax.
    A Dice attn_mlp is refused: the reference takes its batch statistics over the rows of non-empty histories only."""

    def __init__(self, model_dim, attention_type="bilinear_attention", attention_hidden_units=[80, 40],
                 attention_activation="Dice", use_attention_softmax=True, attention_dropout=0.0):
        super(AttentionLayer, self).__init__()
        assert attention_type in ["bilinear_attention", "dot_attention", "din_attention"], \
            "attention_type={} is not supported.".format(attention_type)
        self.attention_type = attention_type
        self.use_attention_softmax = use_attention_softmax
        if attention_type == "bilinear_attention":
            self.W_kernel = nn.Parameter(torch.eye(model_dim))
        elif attention_type == "din_attention":
            self.attn_mlp = MLP_Block(input_dim=model_dim * 4, output_dim=1, hidden_units=attention_hidden_units,
                                      hidden_activations=attention_activation, output_activation=None,
                                      dropout_rates=attention_dropout, batch_norm=False)

    def run(self, interest, target, mask, sink=None):
        """(B, L) scores of interest (B, L, H) (a shared_grad view with its sink, or None) against target (B, H);
        mask (B, L) uint8."""
        if self.attention_type == "din_attention":
            if any(type(m) == Dice for m in self.attn_mlp.modules()):
                raise NotImplementedError("DIEN din_attention: Dice in attn_mlp is not supported (the reference takes "
                                          "Dice's batch statistics over the rows of non-empty histories only)")
            if sink is None:
                raise ValueError("AttentionLayer din_attention: pass the interests' shared_grad sink")
            B, L = mask.shape
            w = self.attn_mlp(F2.dien_din_input(target, interest, sink)).view(B, L)
            if not self.use_attention_softmax:
                return w * mask
        else:
            w = F2.dien_scores(interest, target, mask,
                               self.W_kernel if self.attention_type == "bilinear_attention" else None, sink=sink)
        return F2.dien_softmax(w, mask) if self.use_attention_softmax else w

    def forward(self, sequence_emb, target_emb, mask=None):
        raise NotImplementedError("AttentionLayer runs on the kernels through run(interest, target, mask)")

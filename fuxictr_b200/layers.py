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
  Dice                                     fuxictr/pytorch/layers/activations.py:24-51
  MLP_Block                                fuxictr/pytorch/layers/blocks/mlp_block.py:24-96
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
                   B2_ACT_SIGMOID, FM_PRODUCT_SUM, FM_BI_INTERACTION, FM_INNER_PRODUCT)

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


def fused_front(embedding_layer, lr_layer, X, want_fm):
    """One launch for FeatureEmbedding + (FM product_sum) + (LogisticRegression): returns
    (feature_emb (B,F,D), logit (B,1)), or None when the configuration needs the general path
    (sequence / numeric features, mixed dims, dim % 4 != 0)."""
    fed = embedding_layer.embedding_layer
    names = fed._active_features(X, [], [])
    order = [f for f in fed._feature_map.features.keys() if f in set(names)]
    if not order or not all(fed._is_fusable(f) for f in order):
        return None
    plan, tables = fed._plan(order, order)
    lr_plan = lr_tables = bias = None
    if lr_layer is not None:
        lfed = lr_layer.embedding_layer.embedding_layer
        lnames = lfed._active_features(X, [], [])
        lorder = [f for f in lfed._feature_map.features.keys() if f in set(lnames)]
        if lorder != order or not all(lfed._is_fusable(f) for f in lorder):
            return None
        lr_plan, lr_tables = lfed._plan(lorder, lorder)
        bias = lr_layer.bias
    if not F2.front_supported(plan, lr_plan):
        return None
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

    def forward(self, inputs):
        mods = list(self.mlp)
        x = inputs
        if F2.mlp_chain_supported() and inputs.is_cuda:
            # a pure Linear(+ReLU/Sigmoid) stack runs as ONE autograd node (cross-layer epilogue fusion)
            layers, i, pure = [], 0, len(mods) > 0
            while i < len(mods):
                if type(mods[i]) != nn.Linear:
                    pure = False
                    break
                act = B2_ACT_NONE
                if i + 1 < len(mods) and type(mods[i + 1]) == nn.ReLU:
                    act = B2_ACT_RELU
                elif i + 1 < len(mods) and type(mods[i + 1]) == nn.Sigmoid:
                    act = B2_ACT_SIGMOID
                layers.append((mods[i].weight, mods[i].bias, act))
                i += 2 if act != B2_ACT_NONE else 1
            if pure:
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

"""CPU ORACLE — test infrastructure only, never the product path.

A plain restatement of the reference's hot-path arithmetic (reczoo/FuxiCTR v2.3.10) as
stateless functions over a {state_dict key: tensor} mapping, using the same stock ATen
ops the reference calls (the reference has no native code: its "kernels" ARE these ops —
SURVEY.md section 2.2), plus a numpy restatement of the integer part (index cast + row
gather) for bit-exact checks.  Each function cites the reference file:line it follows.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs
may import this module.  Nothing under fuxictr_b200/ does.

Pinning: tests/golden/*.npz hold inputs, weights, outputs and gradients produced by the
REAL reference modules (imported from /root/reference by tests/golden/make_golden.py in the
build container); tests/test_oracle_golden.py checks every function here against them.
"""
from collections import OrderedDict

import numpy as np
import torch
import torch.nn.functional as F


# ----------------------------------------------------------------------------------------
# Integer part, numpy: `.long()` truncation + row gather  (bit-exact contract)
# ----------------------------------------------------------------------------------------
def np_gather(table, ids):
    """feature_embedding.py:283-288: ids (any float/int dtype) -> int64 by truncation toward
    zero (torch .long()), then a pure row copy (aten::embedding == index_select)."""
    rows = np.trunc(np.asarray(ids, dtype=np.float64)).astype(np.int64) if \
        np.issubdtype(np.asarray(ids).dtype, np.floating) else np.asarray(ids).astype(np.int64)
    return np.asarray(table)[rows]


def np_feature_embedding(specs, tables, batch_matrix, column_index, flatten_emb=False):
    """feature_embedding.py:261-297 + :230-259 for categorical features, numpy only.
    specs: ordered {name: spec}; tables: {name: (V, D) array}; batch_matrix: (B, W) array."""
    outs = []
    for name, spec in specs.items():
        assert spec["type"] == "categorical"
        table = tables[spec.get("share_embedding", name)] if spec.get("share_embedding") in tables else tables[name]
        outs.append(np_gather(table, batch_matrix[:, column_index[name]]))
    return np.concatenate(outs, axis=-1) if flatten_emb else np.stack(outs, axis=1)


# ----------------------------------------------------------------------------------------
# Layer restatements (torch CPU ops, autograd gives the backward the reference gets)
# ----------------------------------------------------------------------------------------
def _emb_key(prefix, feature):
    return "%sembedding_layers.%s.weight" % (prefix, feature)


def table_owner(specs, feature, use_sharing=True):
    """feature_embedding.py:149-151: a feature with share_embedding uses the owner's table."""
    owner = specs[feature].get("share_embedding")
    return owner if (use_sharing and owner in specs) else feature


def feature_embedding_dict(specs, state, prefix, inputs, feature_source=(), feature_type=(),
                           lr_mode=False, use_sharing=True):
    """FeatureEmbeddingDict.forward, feature_embedding.py:261-297.
    `state[prefix + 'embedding_layers.<feat>.weight']` are the tables; numeric features use
    Linear(1, D, bias=False) (:280-282); sequence features optionally pooled by the encoder in
    spec['feature_encoder'] (:294-295) or by MaskedSumPooling in LR mode (:135-138)."""
    out = OrderedDict()
    for feature in inputs.keys():
        spec = specs[feature]
        if feature_source and spec.get("source") not in feature_source:
            continue
        if feature_type and spec["type"] not in feature_type:
            continue
        key = _emb_key(prefix, table_owner(specs, feature, use_sharing))
        if key not in state:
            continue
        if spec["type"] == "numeric":
            emb = F.linear(inputs[feature].float().view(-1, 1), state[key])
        elif spec["type"] in ("categorical", "sequence"):
            emb = F.embedding(inputs[feature].long(), state[key], padding_idx=spec.get("padding_idx"))
        else:
            raise NotImplementedError(spec["type"])
        if spec["type"] == "sequence":
            if lr_mode:
                emb = masked_sum_pooling(emb)
            elif spec.get("feature_encoder") == "layers.MaskedAveragePooling()":
                emb = masked_average_pooling(emb)
            elif spec.get("feature_encoder") == "layers.MaskedSumPooling()":
                emb = masked_sum_pooling(emb)
        out[feature] = emb
    return out


def dict2tensor(specs, emb_dict, flatten_emb=False):
    """feature_embedding.py:230-259: FeatureMap order, cat(dim=-1) or stack(dim=1)."""
    lst = [emb_dict[f] for f in specs.keys() if f in emb_dict]
    return torch.cat(lst, dim=-1) if flatten_emb else torch.stack(lst, dim=1)


def feature_embedding(specs, state, prefix, inputs, flatten_emb=False, **kw):
    """FeatureEmbedding.forward, feature_embedding.py:73-88."""
    return dict2tensor(specs, feature_embedding_dict(specs, state, prefix + "embedding_layer.", inputs, **kw),
                       flatten_emb=flatten_emb)


def masked_average_pooling(emb, mask=None):
    """pooling.py:45-49."""
    sum_out = torch.sum(emb, dim=1)
    if mask is None:
        mask = emb.sum(dim=-1) != 0
    return sum_out / (mask.float().sum(-1, keepdim=True) + 1e-12)


def masked_sum_pooling(emb):
    """pooling.py:73."""
    return torch.sum(emb, dim=1)


def logistic_regression(specs, state, prefix, inputs):
    """logistic_regression.py:55-58: FeatureEmbedding(dim=1, use_pretrain=False,
    use_sharing=False) -> sum over fields -> += bias."""
    w = feature_embedding(specs, state, prefix + "embedding_layer.", inputs, lr_mode=True, use_sharing=False)
    out = w.sum(dim=1)
    if prefix + "bias" in state:
        out = out + state[prefix + "bias"]
    return out


def inner_product_interaction(feature_emb, output="product_sum"):
    """inner_product.py:55-70."""
    if output in ("product_sum", "bi_interaction"):
        sum_then_square = torch.sum(feature_emb, dim=1) ** 2
        square_then_sum = torch.sum(feature_emb ** 2, dim=1)
        bi = (sum_then_square - square_then_sum) * 0.5
        return bi if output == "bi_interaction" else bi.sum(dim=-1, keepdim=True)
    num_fields = feature_emb.shape[1]
    if output == "inner_product":
        mat = torch.bmm(feature_emb, feature_emb.transpose(1, 2))
        mask = torch.triu(torch.ones(num_fields, num_fields), 1).bool()
        return torch.masked_select(mat, mask).view(-1, num_fields * (num_fields - 1) // 2)
    if output == "elementwise_product":
        iu = torch.triu_indices(num_fields, num_fields, offset=1)
        return torch.index_select(feature_emb, 1, iu[0]) * torch.index_select(feature_emb, 1, iu[1])
    raise ValueError(output)


def factorization_machine(specs, state, prefix, inputs, feature_emb):
    """factorization_machine.py:56-59."""
    return inner_product_interaction(feature_emb, "product_sum") + \
        logistic_regression(specs, state, prefix + "lr_layer.", inputs)


def crossnet(x0, state, prefix, num_layers):
    """cross_net.py:89-92 with CrossInteraction :54."""
    xi = x0
    for i in range(num_layers):
        w = state["%scross_net.%d.weight.weight" % (prefix, i)]
        b = state["%scross_net.%d.bias" % (prefix, i)]
        xi = xi + (F.linear(xi, w) * x0 + b)
    return xi


def crossnet_v2(x0, state, prefix, num_layers):
    """cross_net.py:126-129."""
    xi = x0
    for i in range(num_layers):
        xi = xi + x0 * F.linear(xi, state["%scross_layers.%d.weight" % (prefix, i)],
                                state["%scross_layers.%d.bias" % (prefix, i)])
    return xi


def compressed_interaction_net(feature_emb, state, prefix, cin_hidden_units):
    """compressed_interaction_net.py:64-76."""
    pools = []
    x0 = feature_emb
    batch, _, dim = x0.shape
    xi = x0
    for i in range(len(cin_hidden_units)):
        had = torch.einsum("bhd,bmd->bhmd", x0, xi).view(batch, -1, dim)
        xi = F.conv1d(had, state["%scin_layer.layer_%d.weight" % (prefix, i + 1)],
                      state["%scin_layer.layer_%d.bias" % (prefix, i + 1)]).view(batch, -1, dim)
        pools.append(xi.sum(dim=-1))
    return F.linear(torch.cat(pools, dim=-1), state[prefix + "fc.weight"], state[prefix + "fc.bias"])


def dice(x, state, prefix, training, eps=1e-9, momentum=0.01):
    """activations.py:37,49-50: BatchNorm1d(affine=False, eps=1e-9, momentum=0.01) gate."""
    p = torch.sigmoid(F.batch_norm(x, state[prefix + "bn.running_mean"], state[prefix + "bn.running_var"],
                                   None, None, training, momentum, eps))
    alpha = state[prefix + "alpha"]
    return p * x + alpha * (1 - p) * x


def mlp_block(x, state, prefix, layout, training=True):
    """mlp_block.py:64-96.  `layout` lists the nn.Sequential children in order as tuples:
    ("linear",), ("relu",), ("sigmoid",), ("dice",), ("bn",); indices are the child indices."""
    for idx, kind in enumerate(layout):
        p = "%smlp.%d." % (prefix, idx)
        if kind == "linear":
            x = F.linear(x, state[p + "weight"], state.get(p + "bias"))
        elif kind == "relu":
            x = torch.relu(x)
        elif kind == "sigmoid":
            x = torch.sigmoid(x)
        elif kind == "dice":
            x = dice(x, state, p, training)
        elif kind == "bn":
            x = F.batch_norm(x, state[p + "running_mean"], state[p + "running_var"], state[p + "weight"],
                             state[p + "bias"], training, 0.1, 1e-5)
        else:
            raise ValueError(kind)
    return x


def mlp_layout(n_hidden, hidden_act="relu", has_output=True, output_act=None):
    """Child order produced by MLP_Block.__init__ without BN/dropout (mlp_block.py:73-85)."""
    layout = []
    for _ in range(n_hidden):
        layout.append("linear")
        if hidden_act:
            layout.append(hidden_act)
    if has_output:
        layout.append("linear")
    if output_act:
        layout.append(output_act)
    return layout


def din_attention(target, history, mask, state, prefix, layout, embedding_dim, use_softmax=False,
                  training=True):
    """target_attention.py:79-92."""
    seq_len = history.size(1)
    t = target.unsqueeze(1).expand(-1, seq_len, -1)
    att_in = torch.cat([t, history, t - history, t * history], dim=-1)
    w = mlp_block(att_in.view(-1, 4 * embedding_dim), state, prefix + "attention_layer.", layout, training)
    w = w.view(-1, seq_len)
    if mask is not None:
        w = w * mask.float()
    if use_softmax:
        if mask is not None:
            w = w + -1.e9 * (1 - mask.float())
        w = w.softmax(dim=-1)
    return (w.unsqueeze(-1) * history).sum(dim=1)


# ----------------------------------------------------------------------------------------
# Model forwards (callers) and one training step
# ----------------------------------------------------------------------------------------
def split_inputs(specs, labels, batch):
    """BaseModel.get_inputs / get_labels, rank_model.py:169-203."""
    X = OrderedDict((k, v) for k, v in batch.items() if k not in labels and specs[k]["type"] != "meta")
    y = batch[labels[0]].float().view(-1, 1)
    return X, y


def deepfm_logit(specs, state, X, n_hidden):
    """DeepFM.forward, DeepFM.py:83-86 (pre-sigmoid)."""
    emb = feature_embedding(specs, state, "embedding_layer.", X)
    y = factorization_machine(specs, state, "fm.", X, emb)
    return y + mlp_block(emb.flatten(start_dim=1), state, "mlp.", mlp_layout(n_hidden))


def dcnv2_logit(specs, state, X, num_cross_layers, n_hidden):
    """DCNv2.forward (parallel structure), DCNv2.py:117-130 (pre-sigmoid)."""
    emb = feature_embedding(specs, state, "embedding_layer.", X, flatten_emb=True)
    cross = crossnet_v2(emb, state, "crossnet.", num_cross_layers)
    dnn = mlp_block(emb, state, "parallel_dnn.", mlp_layout(n_hidden, has_output=False))
    final = torch.cat([cross, dnn], dim=-1)
    return F.linear(final, state["fc.weight"], state["fc.bias"])


def dlrm_pred(specs, state, X, n_top_hidden):
    """DLRM.forward without dense features, DLRM.py:113-123 (top_mlp ends in sigmoid)."""
    emb = feature_embedding(specs, state, "embedding_layer.", X)
    inter = inner_product_interaction(emb, "inner_product")
    return mlp_block(inter, state, "top_mlp.", mlp_layout(n_top_hidden, output_act="sigmoid"))


def xdeepfm_logit(specs, state, X, cin_hidden_units, n_hidden):
    """xDeepFM.forward, xDeepFM.py:87-94 (pre-sigmoid)."""
    emb = feature_embedding(specs, state, "embedding_layer.", X)
    y = logistic_regression(specs, state, "lr_layer.", X) + \
        compressed_interaction_net(emb, state, "cin.", cin_hidden_units)
    return y + mlp_block(emb.flatten(start_dim=1), state, "dnn.", mlp_layout(n_hidden))


def din_pred(specs, state, X, embedding_dim, target_fields, sequence_fields, n_att_hidden, n_hidden,
             training=True, use_softmax=False):
    """DIN.forward, DIN.py:118-133 (dnn ends in sigmoid)."""
    emb = feature_embedding_dict(specs, state, "embedding_layer.", X)
    att_layout = mlp_layout(n_att_hidden, hidden_act="dice")
    for i, (tf, sf) in enumerate(zip(target_fields, sequence_fields)):
        tf_l = list(tf) if isinstance(tf, tuple) else [tf]
        sf_l = list(sf) if isinstance(sf, tuple) else [sf]
        target = torch.cat([emb[f] for f in tf_l], dim=-1)
        seq = torch.cat([emb[f] for f in sf_l], dim=-1)
        mask = X[sf_l[0]].long() != 0
        pooled = din_attention(target, seq, mask, state, "attention_layers.%d." % i, att_layout,
                               embedding_dim * len(tf_l), use_softmax, training)
        for f, part in zip(sf_l, pooled.split(embedding_dim, dim=-1)):
            emb[f] = part
    flat = dict2tensor(specs, emb, flatten_emb=True)
    return mlp_block(flat, state, "dnn.", mlp_layout(n_hidden, output_act="sigmoid"), training)


def bce_mean(y_pred, y_true):
    """BaseModel.add_loss, rank_model.py:130."""
    return F.binary_cross_entropy(y_pred, y_true, reduction="mean")


class OracleTrainer(object):
    """BaseModel.train_step (rank_model.py:316-323) over a functional model:
    zero_grad -> forward -> BCE -> backward -> clip_grad_norm_(10) -> torch.optim.Adam.step.
    `pred_fn(state, X)` returns y_pred (post-sigmoid)."""

    def __init__(self, state, pred_fn, specs, labels, lr=1e-3, max_norm=10.0):
        self.state = OrderedDict()
        for k, v in state.items():
            t = v.detach().clone()
            if t.is_floating_point() and "running_" not in k and "triu" not in k:
                t.requires_grad_(True)
            self.state[k] = t
        # share_embedding (feature_embedding.py:149-151): the reference registers ONE nn.Embedding
        # under both feature names, so its state_dict lists the same tensor twice.  Alias the
        # follower key to the owner's tensor (LogisticRegression builds its tables with
        # use_sharing=False, logistic_regression.py:44, so keys under "lr_layer." stay separate).
        for key in list(self.state.keys()):
            if ".embedding_layers." in key and key.endswith(".weight") and "lr_layer." not in key:
                head, feat = key[:-len(".weight")].rsplit(".embedding_layers.", 1)
                owner = table_owner(specs, feat) if feat in specs else feat
                if owner != feat:
                    self.state[key] = self.state["%s.embedding_layers.%s.weight" % (head, owner)]
        seen, self.params = set(), []
        for t in self.state.values():
            if t.requires_grad and id(t) not in seen:
                seen.add(id(t))
                self.params.append(t)
        self.pred_fn, self.specs, self.labels, self.max_norm = pred_fn, specs, labels, max_norm
        self.optimizer = torch.optim.Adam(self.params, lr=lr)

    def forward(self, batch):
        X, y = split_inputs(self.specs, self.labels, batch)
        return self.pred_fn(self.state, X), y

    def train_step(self, batch):
        self.optimizer.zero_grad()
        y_pred, y = self.forward(batch)
        loss = bce_mean(y_pred, y.to(y_pred.dtype))      # labels in the state's dtype (float64 runs)
        loss.backward()
        torch.nn.utils.clip_grad_norm_(self.params, self.max_norm)
        self.optimizer.step()
        return loss


# ----------------------------------------------------------------------------------------
# Evaluation metrics (fuxictr/metrics.py:45-48 as called by rank_model.py:350-381), numpy.
# The reference delegates to scikit-learn 1.x: log_loss (clip the float64 [1-p, p] rows to
# [eps, 1-eps], mean of -xlogy) and roc_auc_score (trapezoid over the ROC curve == tie-aware
# Mann-Whitney U / (P N)).  Restated here without sklearn and pinned to the real reference's output
# in tests/golden/metrics_eval.npz.
# ----------------------------------------------------------------------------------------
def logloss(y_true, y_pred):
    p = np.asarray(y_pred, dtype=np.float64).reshape(-1)
    y = np.asarray(y_true, dtype=np.float64).reshape(-1)
    eps = np.finfo(np.float64).eps
    p1 = np.clip(p, eps, 1 - eps)
    p0 = np.clip(1 - p, eps, 1 - eps)
    with np.errstate(divide="ignore", invalid="ignore"):
        terms = np.where(y != 0, y * np.log(p1), 0.0) + np.where(y != 1, (1 - y) * np.log(p0), 0.0)
    return float(-terms.mean())


def auc_twice_u(y_true, y_pred):
    """2U as an exact integer: sum over positives of #(neg < s) + #(neg <= s); also (P, N)."""
    p = np.asarray(y_pred).reshape(-1)
    y = np.asarray(y_true).reshape(-1)
    neg = np.sort(p[y == 0])
    pos = p[y == 1]
    lower = np.searchsorted(neg, pos, side="left").astype(np.int64)
    upper = np.searchsorted(neg, pos, side="right").astype(np.int64)
    return int(lower.sum() + upper.sum()), int(pos.size), int(neg.size)


def auc(y_true, y_pred):
    twice_u, n_pos, n_neg = auc_twice_u(y_true, y_pred)
    if n_pos == 0 or n_neg == 0:
        raise ValueError("Only one class present in y_true. ROC AUC score is not defined in that case.")
    return twice_u / (2.0 * n_pos * n_neg)


def evaluate_metrics(y_true, y_pred, metrics):
    """metrics.py:26-52 for the pointwise metrics."""
    out = OrderedDict()
    for m in metrics:
        if m in ("logloss", "binary_crossentropy"):
            out[m] = logloss(y_true, y_pred)
        elif m == "AUC":
            out[m] = auc(y_true, y_pred)
        else:
            raise ValueError("metric={} not supported.".format(m))
    return out


# ----------------------------------------------------------------------------------------
# Neighbouring interaction layers (SURVEY.md 8f row 4, second half) — restated ahead of their
# kernels so the parity gates exist first.  Pinned by tests/golden/next_*.npz.
# ----------------------------------------------------------------------------------------
def bilinear_interaction(state, prefix, feature_emb, bilinear_type):
    """BilinearInteraction / BilinearInteractionV2.forward (bilinear_interaction.py:63-78,128-141):
    out[:, p, :] = (e_i @ W_*) * e_j over the upper-triangular pairs p = (i < j); W_* is the one
    shared matrix (field_all), W[i] (field_each) or W[p] (field_interaction)."""
    W = state[prefix + "bilinear_W"]
    F_ = feature_emb.shape[1]
    iu = torch.triu_indices(F_, F_, offset=1)
    left, right = feature_emb[:, iu[0]], feature_emb[:, iu[1]]
    if bilinear_type == "field_all":
        hidden = torch.matmul(left, W)
    elif bilinear_type == "field_each":
        hidden = torch.einsum("bpd,pde->bpe", left, W[iu[0]])
    elif bilinear_type == "field_interaction":
        hidden = torch.einsum("bpd,pde->bpe", left, W)
    else:
        raise NotImplementedError
    return hidden * right


def squeeze_excitation(state, prefix, feature_emb, excitation_activation="ReLU"):
    """SqueezeExcitation.forward (squeeze_excitation.py:61-64): per-field mean over the embedding
    axis -> Linear(F, F/r) -> ReLU -> Linear(F/r, F) -> ReLU|Sigmoid -> rescale the fields."""
    z = feature_emb.mean(dim=-1)
    a = F.relu(F.linear(z, state[prefix + "excitation.0.weight"]))
    a = F.linear(a, state[prefix + "excitation.2.weight"])
    a = F.relu(a) if excitation_activation.lower() == "relu" else torch.sigmoid(a)
    return feature_emb * a.unsqueeze(-1)


def multi_head_target_attention(state, prefix, target_item, history_sequence, mask, num_heads,
                                use_scale=True, use_qkvo=True):
    """MultiHeadTargetAttention.forward + ScaledDotProductAttention (target_attention.py:141-172,
    dot_product_attention.py:48-58): one query (the target) per sample, masked positions filled with
    -1e9 before the softmax over the history, heads concatenated, optional W_o."""
    if use_qkvo:
        q = F.linear(target_item, state[prefix + "W_q.weight"])
        k = F.linear(history_sequence, state[prefix + "W_k.weight"])
        v = F.linear(history_sequence, state[prefix + "W_v.weight"])
    else:
        q, k, v = target_item, history_sequence, history_sequence
    B, L = k.shape[0], k.shape[1]
    hd = q.shape[-1] // num_heads
    q = q.view(B, 1, num_heads, hd).transpose(1, 2)
    k = k.view(B, L, num_heads, hd).transpose(1, 2)
    v = v.view(B, L, num_heads, hd).transpose(1, 2)
    scores = torch.matmul(q, k.transpose(-1, -2))                     # (B, H, 1, L)
    if use_scale:
        scores = scores / (hd ** 0.5)
    if mask is not None:
        scores = scores.masked_fill(mask.view(B, 1, 1, L).float() == 0, -1.e9)
    out = torch.matmul(scores.softmax(dim=-1), v)                     # (B, H, 1, hd)
    out = out.transpose(1, 2).contiguous().view(B, num_heads * hd)
    return F.linear(out, state[prefix + "W_o.weight"]) if use_qkvo else out


def crossnet_mix(state, prefix, x0, layer_num, num_experts):
    """CrossNetMix.forward (cross_net.py:168-201): per layer a softmax-gated mixture of low-rank
    experts  x0 * (U_e tanh(C_e tanh(V_e^T x_l)) + b),  residual added."""
    xl = x0
    for i in range(layer_num):
        outs, gates = [], []
        for e in range(num_experts):
            gates.append(F.linear(xl, state[prefix + "gating.%d.weight" % e]))          # (B, 1)
            U, V, C = (state[prefix + "%s_list.%d" % (n, i)][e] for n in ("U", "V", "C"))
            vx = torch.tanh(xl @ V)                                                       # (B, r)
            vx = torch.tanh(vx @ C.t())
            outs.append(x0 * (vx @ U.t() + state[prefix + "bias.%d" % i].view(1, -1)))
        outs = torch.stack(outs, 2)                                                       # (B, d, E)
        score = torch.stack(gates, 1).softmax(1)                                          # (B, E, 1)
        xl = torch.matmul(outs, score).squeeze(2) + xl
    return xl

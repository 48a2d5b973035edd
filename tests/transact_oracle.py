"""Float64 restatement of TransAct (model_zoo/TransAct/src/TransAct.py: TransActTransformer, TransAct) for the TransAct
tests, written from the model's math (nn.TransformerEncoderLayer: post-norm, ReLU, eps 1e-5), on the shared oracle's
embedding, CrossNetV2 and MLP restatements (oracle/fuxictr_oracle.py).  Test infrastructure only: nothing under
fuxictr_b200/ imports it."""
import math
import os
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle.fuxictr_oracle import crossnet_v2, feature_embedding_dict, mlp_block  # noqa: E402


def _flat(field):
    return list(field) if isinstance(field, (list, tuple)) else [field]


def adjusted_padding(ids):
    """(B, L) bool, True = padded: ids == 0, with the last slot of an all-padding row unmasked (adjust_mask)."""
    pad = ids == 0
    pad[pad.all(dim=-1), -1] = False
    return pad


def encoder_layer(x, pad, state, prefix, num_heads, attn_keep=None, p_attn=0.0, keep1=None, keep0=None, keep2=None,
                  p=0.0):
    """nn.TransformerEncoderLayer (post-norm, ReLU) on x (B, L, md) with key-padding mask pad (B, L).  attn_keep
    (B, H, L, L), keep1 / keep0 / keep2 (B, L, md | dim_feedforward): dropout masks of the attention weights, dropout1,
    the inner dropout and dropout2 (kept values scaled by 1 / (1 - p))."""
    B, L, md = x.shape
    dh = md // num_heads
    qkv = F.linear(x, state[prefix + "self_attn.in_proj_weight"], state[prefix + "self_attn.in_proj_bias"])
    q, k, v = (t.reshape(B, L, num_heads, dh).transpose(1, 2) for t in qkv.split(md, dim=-1))
    scores = torch.matmul(q * math.sqrt(1.0 / dh), k.transpose(-1, -2))
    scores = scores.masked_fill(pad.view(B, 1, 1, L), float("-inf"))
    att = scores.softmax(dim=-1)
    if attn_keep is not None:
        att = att * attn_keep.to(att.dtype) / (1.0 - p_attn)
    ctx = torch.matmul(att, v).transpose(1, 2).reshape(B, L, md)
    a = F.linear(ctx, state[prefix + "self_attn.out_proj.weight"], state[prefix + "self_attn.out_proj.bias"])
    if keep1 is not None:
        a = a * keep1.to(a.dtype) / (1.0 - p)
    s = F.layer_norm(x + a, (md,), state[prefix + "norm1.weight"], state[prefix + "norm1.bias"], 1e-5)
    h = torch.relu(F.linear(s, state[prefix + "linear1.weight"], state[prefix + "linear1.bias"]))
    if keep0 is not None:
        h = h * keep0.to(h.dtype) / (1.0 - p)
    f = F.linear(h, state[prefix + "linear2.weight"], state[prefix + "linear2.bias"])
    if keep2 is not None:
        f = f * keep2.to(f.dtype) / (1.0 - p)
    return F.layer_norm(s + f, (md,), state[prefix + "norm2.weight"], state[prefix + "norm2.bias"], 1e-5)


def encoder_output(seq, tgt, ids, state, prefix, num_heads, n_layers):
    """(y (B, L, md) zeroed at padded slots, pad (B, L)) of the encoder stack on [seq | tgt]."""
    L = seq.shape[1]
    x = torch.cat([seq, tgt.unsqueeze(1).expand(-1, L, -1)], dim=-1)
    pad = adjusted_padding(ids)
    for n in range(n_layers):
        x = encoder_layer(x, pad, state, prefix + "transformer_encoder.layers.%d." % n, num_heads)
    return x.masked_fill(pad.unsqueeze(-1), 0.0), pad


def transformer(seq, tgt, ids, state, prefix, num_heads, n_layers, first_k_cols=1, concat_max_pool=True):
    """TransActTransformer.forward(tgt, seq, mask=ids == 0): (B, (first_k_cols + concat_max_pool) md)."""
    y, pad = encoder_output(seq, tgt, ids, state, prefix, num_heads, n_layers)
    out = [y[:, -first_k_cols:].flatten(start_dim=1)]
    if concat_max_pool:
        pooled = y.masked_fill(pad.unsqueeze(-1), -1e9).max(dim=1).values
        out.append(F.linear(pooled, state[prefix + "out_linear.weight"], state[prefix + "out_linear.bias"]))
    return torch.cat(out, dim=-1)


def _mlp_layout(n_hidden, batch_norm, has_output):
    layout = []
    for _ in range(n_hidden):
        layout += ["linear"] + (["bn"] if batch_norm else []) + ["relu"]
    return layout + (["linear"] if has_output else [])


def transact_logit(specs, state, X, kw):
    """TransAct.forward (pre-sigmoid) with the reference keywords kw: per pair the transformer on the first sequence
    field's mask, its output after the remaining embeddings, then mlp(cat([CrossNetV2(x), parallel_dnn(x)]))."""
    emb = feature_embedding_dict(specs, state, "embedding_layer.", X)
    targets = kw.get("target_item_field", [("item_id", "cate_id")])
    sequences = kw.get("sequence_item_field", [("click_history", "cate_history")])
    targets = targets if isinstance(targets, list) else [targets]
    sequences = sequences if isinstance(sequences, list) else [sequences]
    outs = []
    for idx, (target, sequence) in enumerate(zip(targets, sequences)):
        tnames, snames = _flat(target), _flat(sequence)
        seq = torch.cat([emb[n] for n in snames], dim=-1)
        tgt = torch.cat([emb[n] for n in tnames], dim=-1)
        outs.append(transformer(seq, tgt, X[snames[0]].long(), state, "transformer_encoders.%d." % idx,
                                kw.get("num_heads", 1), kw.get("transformer_layers", 1), kw.get("first_k_cols", 1),
                                kw.get("concat_max_pool", True)))
    for sequence in sequences:
        for n in _flat(sequence):
            if specs[n]["type"] == "sequence":
                emb.pop(n, None)
    x = torch.cat(list(emb.values()) + outs, dim=-1)
    bn = kw.get("batch_norm", False)
    cross = crossnet_v2(x, state, "crossnet.", kw.get("dcn_cross_layers", 3))
    dnn = mlp_block(x, state, "parallel_dnn.", _mlp_layout(len(kw.get("dcn_hidden_units", [256, 128, 64])), bn, False))
    head = torch.cat([cross, dnn], dim=-1)
    return mlp_block(head, state, "mlp.", _mlp_layout(len(kw.get("mlp_hidden_units", [])), False, True))

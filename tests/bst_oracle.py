"""Float64 restatement of BST (model_zoo/BST/src/BST.py: TransformerBlock, BehaviorTransformer, BST) for the BST tests,
written from the model's math, on the shared oracle's embedding and MLP restatements (oracle/fuxictr_oracle.py).  Test
infrastructure only: nothing under fuxictr_b200/ imports it."""
import math
import os
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle.fuxictr_oracle import feature_embedding_dict, mlp_block, mlp_layout  # noqa: E402


def _flat(field):
    return list(field) if isinstance(field, (list, tuple)) else [field]


def attention_mask(valid, causal):
    """(B, L, L) bool, True = hidden: key j is hidden from query i != j when j is a padded history slot (valid (B, L - 1)
    bool, False = padding) or, causal, j > i.  The target (the last token) is never padding."""
    B, Lm1 = valid.shape
    L = Lm1 + 1
    pad = torch.cat([~valid.bool(), torch.zeros(B, 1, dtype=torch.bool)], dim=1)
    hide = pad.unsqueeze(1).expand(B, L, L).clone()
    if causal:
        hide = hide | torch.ones(L, L, dtype=torch.bool).triu(1).unsqueeze(0)
    return hide & ~torch.eye(L, dtype=torch.bool).unsqueeze(0)


def transformer_block(x, valid, state, prefix, num_heads, layer_norm=True, use_residual=True, causal=False,
                      attn_keep=None, p_attn=0.0, keep1=None, keep2=None, p_net=0.0):
    """TransformerBlock.forward on x (B, L, md).  attn_keep (B, H, L, L), keep1 / keep2 (B, L, md) bool: dropout masks of
    the attention weights, of dropout1 and of dropout2 (kept values scaled by 1 / (1 - p))."""
    B, L, md = x.shape
    dh = md // num_heads
    qkv = F.linear(x, state[prefix + "attention.in_proj_weight"], state[prefix + "attention.in_proj_bias"])
    q, k, v = (t.reshape(B, L, num_heads, dh).transpose(1, 2) for t in qkv.split(md, dim=-1))
    scores = torch.matmul(q * math.sqrt(1.0 / dh), k.transpose(-1, -2))
    scores = scores.masked_fill(attention_mask(valid, causal).unsqueeze(1), float("-inf"))
    att = scores.softmax(dim=-1)
    if attn_keep is not None:
        att = att * attn_keep.to(att.dtype) / (1.0 - p_attn)
    ctx = torch.matmul(att, v).transpose(1, 2).reshape(B, L, md)
    s = F.linear(ctx, state[prefix + "attention.out_proj.weight"], state[prefix + "attention.out_proj.bias"])
    if keep1 is not None:
        s = s * keep1.to(s.dtype) / (1.0 - p_net)
    if use_residual:
        s = s + x
    if layer_norm:
        s = F.layer_norm(s, (md,), state[prefix + "layer_norm1.weight"], state[prefix + "layer_norm1.bias"], 1e-5)
    h = F.leaky_relu(F.linear(s, state[prefix + "ffn.0.weight"], state[prefix + "ffn.0.bias"]), 0.01)
    out = F.linear(h, state[prefix + "ffn.2.weight"], state[prefix + "ffn.2.bias"])
    if keep2 is not None:
        out = out * keep2.to(out.dtype) / (1.0 - p_net)
    if use_residual:
        out = out + s
    if layer_norm:
        out = F.layer_norm(out, (md,), state[prefix + "layer_norm2.weight"], state[prefix + "layer_norm2.bias"], 1e-5)
    return out


def pooling(out, valid, kind):
    """BST.sequence_pooling: mean / sum over the real slots and the target (mean: / (count + 1e-12)), target, concat."""
    B = out.shape[0]
    w = torch.cat([valid.to(out.dtype), torch.ones(B, 1, dtype=out.dtype)], dim=1).unsqueeze(-1)
    if kind == "mean":
        return (out * w).sum(dim=1) / (w.sum(dim=1) + 1e-12)
    if kind == "sum":
        return (out * w).sum(dim=1)
    if kind == "target":
        return out[:, -1, :]
    return out.flatten(start_dim=1)


def bst_logit(specs, state, X, kw, n_blocks=None):
    """BST.forward (pre-sigmoid) with the reference keywords kw: tokens [sequence | target] (+ position embedding) per
    pair, the transformer stack, pooling, the pooled vectors after the remaining embeddings, the DNN."""
    emb = feature_embedding_dict(specs, state, "embedding_layer.", X)
    targets = kw.get("bst_target_field", [("item_id", "cate_id")])
    sequences = kw.get("bst_sequence_field", [("click_history", "cate_history")])
    targets = targets if isinstance(targets, list) else [targets]
    sequences = sequences if isinstance(sequences, list) else [sequences]
    heads = kw.get("num_heads", 2)
    n_blocks = kw.get("stacked_transformer_layers", 1) if n_blocks is None else n_blocks
    pooled = []
    for idx, (target, sequence) in enumerate(zip(targets, sequences)):
        tnames, snames = _flat(target), _flat(sequence)
        valid = X[snames[0]].long() != 0
        seq = torch.cat([emb[n] for n in snames], dim=-1)
        tgt = torch.cat([emb[n] for n in tnames], dim=-1)
        x = torch.cat([seq, tgt.unsqueeze(1)], dim=1)
        enc = "transformer_encoders.%d." % idx
        if kw.get("use_position_emb", True):
            pos = state[enc + "position_emb"]
            x = torch.cat([x, pos.unsqueeze(0).expand(x.shape[0], -1, -1)], dim=-1)
        for b in range(n_blocks):
            x = transformer_block(x, valid, state, enc + "transformer_blocks.%d." % b, heads,
                                  kw.get("layer_norm", True), kw.get("use_residual", True),
                                  kw.get("use_causal_mask", False))
        pooled.append(pooling(x, valid, kw.get("seq_pooling_type", "mean")))
    for sequence in sequences:
        for n in _flat(sequence):
            emb.pop(n, None)
    flat = torch.cat(list(emb.values()) + pooled, dim=-1)
    return mlp_block(flat, state, "dnn.", mlp_layout(len(kw.get("dnn_hidden_units", [256, 128, 64]))))

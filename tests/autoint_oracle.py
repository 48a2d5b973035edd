"""Float64 restatement of AutoInt (model_zoo/AutoInt/src/AutoInt.py: MultiHeadSelfAttention, AutoInt) for the AutoInt
tests, built on the shared oracle's embedding, LR and MLP restatements (oracle/fuxictr_oracle.py).  Test
infrastructure only: nothing under fuxictr_b200/ imports it."""
import os
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle.fuxictr_oracle import feature_embedding, logistic_regression, mlp_block, mlp_layout  # noqa: E402


def self_attention(X, state, prefix, num_heads, use_residual=True, use_scale=False, layer_norm=False, keep=None,
                   p=0.0):
    """MultiHeadSelfAttention.forward on X (B, F, d_in).  keep (B, H, F, F) bool: the dropout mask of the attention
    weights (kept weights scaled by 1 / (1 - p))."""
    W_q, W_k, W_v = (state[prefix + n + ".weight"] for n in ("W_q", "W_k", "W_v"))
    B, nf, _ = X.shape
    A = W_q.shape[0]
    dh = A // num_heads

    def heads(t):
        return t.view(B, nf, num_heads, dh).transpose(1, 2)
    q, k, v = heads(F.linear(X, W_q)), heads(F.linear(X, W_k)), heads(F.linear(X, W_v))
    scores = torch.matmul(q, k.transpose(-1, -2))
    if use_scale:
        scores = scores / dh ** 0.5
    att = scores.softmax(dim=-1)
    if keep is not None:
        att = att * keep.to(att.dtype) / (1.0 - p)
    out = torch.matmul(att, v).transpose(1, 2).reshape(B, nf, A)
    if use_residual:
        res = F.linear(X, state[prefix + "W_res.weight"]) if prefix + "W_res.weight" in state else X
        out = out + res
    if layer_norm:
        out = F.layer_norm(out, (A,), state[prefix + "layer_norm.weight"], state[prefix + "layer_norm.bias"], 1e-5)
    return out.relu()


def autoint_logit(specs, state, X, attention_layers, num_heads, n_hidden, use_residual=True, use_scale=False,
                  layer_norm=False, use_wide=False):
    """AutoInt.forward (pre-sigmoid): fc over the flattened attention stack, plus the DNN (n_hidden hidden layers;
    None: no DNN) and the LR term (use_wide)."""
    emb = feature_embedding(specs, state, "embedding_layer.", X)
    x = emb
    for i in range(attention_layers):
        x = self_attention(x, state, "self_attention.%d." % i, num_heads, use_residual, use_scale, layer_norm)
    y = F.linear(x.flatten(start_dim=1), state["fc.weight"], state["fc.bias"])
    if n_hidden is not None:
        y = y + mlp_block(emb.flatten(start_dim=1), state, "dnn.", mlp_layout(n_hidden))
    if use_wide:
        y = y + logistic_regression(specs, state, "lr_layer.", X)
    return y

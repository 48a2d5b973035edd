"""Float64 restatement of FinalMLP and DualMLP (model_zoo/FinalMLP/src: FeatureSelection, InteractionAggregation,
FinalMLP, DualMLP) for the FinalMLP tests, built on the shared oracle's embedding and MLP restatements
(oracle/fuxictr_oracle.py) and pinned to the reference's goldens by tests/test_finalmlp_host.py.  It runs the gates
as the reference does, over the context row repeated for every sample.  Test infrastructure only: nothing under
fuxictr_b200/ imports it."""
import os
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle.fuxictr_oracle import feature_embedding, mlp_block, mlp_layout  # noqa: E402


def interaction_aggregation(state, prefix, x, y, num_heads):
    """InteractionAggregation.forward at output_dim 1: w_x(x) + w_y(y) + sum_h x_h^T W_h y_h, (B, 1)."""
    B, dx = x.shape
    dy = y.shape[1]
    hx, hy = dx // num_heads, dy // num_heads
    W = state[prefix + "w_xy"].reshape(num_heads, hx, hy)
    xy = torch.einsum("bhi,hij,bhj->b", x.reshape(B, num_heads, hx), W, y.reshape(B, num_heads, hy))
    out = F.linear(x, state[prefix + "w_x.weight"], state[prefix + "w_x.bias"]) + \
        F.linear(y, state[prefix + "w_y.weight"], state[prefix + "w_y.bias"])
    return out + xy.unsqueeze(1)


def feature_selection(specs, state, prefix, X, flat_emb, contexts, n_hidden):
    """FeatureSelection.forward: (flat_emb * 2 g1, flat_emb * 2 g2), g_s the sigmoid gate of context s."""
    outs = []
    for s, ctx in ((1, contexts[0]), (2, contexts[1])):
        if ctx:
            sub = {k: specs[k] for k in specs if k in ctx}
            inp = feature_embedding(sub, state, "%sfs%d_ctx_emb." % (prefix, s), {k: X[k] for k in ctx},
                                    flatten_emb=True)
        else:
            inp = state["%sfs%d_ctx_bias" % (prefix, s)].repeat(flat_emb.shape[0], 1)
        g = mlp_block(inp, state, "%sfs%d_gate." % (prefix, s), mlp_layout(n_hidden, output_act="sigmoid"))
        outs.append(flat_emb * (g * 2))
    return tuple(outs)


def finalmlp_logit(specs, state, X, kw):
    """FinalMLP.forward (pre-sigmoid); kw: the model's constructor keywords."""
    emb = feature_embedding(specs, state, "embedding_layer.", X, flatten_emb=True)
    if kw.get("use_fs", True):
        f1, f2 = feature_selection(specs, state, "fs_module.", X, emb,
                                   (kw.get("fs1_context", []), kw.get("fs2_context", [])),
                                   len(kw.get("fs_hidden_units", [64])))
    else:
        f1 = f2 = emb
    x = mlp_block(f1, state, "mlp1.", mlp_layout(len(kw["mlp1_hidden_units"]), has_output=False))
    y = mlp_block(f2, state, "mlp2.", mlp_layout(len(kw["mlp2_hidden_units"]), has_output=False))
    return interaction_aggregation(state, "fusion_module.", x, y, kw.get("num_heads", 1))


def dualmlp_logit(specs, state, X, kw):
    """DualMLP.forward (pre-sigmoid): the two towers' logits, summed."""
    emb = feature_embedding(specs, state, "embedding_layer.", X, flatten_emb=True)
    return mlp_block(emb, state, "mlp1.", mlp_layout(len(kw["mlp1_hidden_units"]))) + \
        mlp_block(emb, state, "mlp2.", mlp_layout(len(kw["mlp2_hidden_units"])))

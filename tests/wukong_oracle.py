"""Float64 restatement of WuKong (model_zoo/WuKong/src/WuKong.py: FactorizationMachineBlock, LinearCompressionBlock,
WuKongLayer, WuKong) for the WuKong tests, built on the shared oracle's embedding and MLP restatements
(oracle/fuxictr_oracle.py).  Test infrastructure only: nothing under fuxictr_b200/ imports it."""
import os
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle.fuxictr_oracle import feature_embedding, mlp_block  # noqa: E402


def wukong_layer(x, state, prefix, n_fmb_hidden, layer_norm=True, margins=None):
    """WuKongLayer.forward on x (B, F, D); n_fmb_hidden: the FMB MLP's hidden layer count (no dropout).  margins: a
    list that receives, per sample, the smallest |pre-activation| of the FMB MLP's ReLUs (B,)."""
    B, nf, D = x.shape
    Y = state[prefix + "fmb.proj_Y"]
    fm = (x @ (x.transpose(1, 2) @ Y)).flatten(start_dim=1)
    fm = F.layer_norm(fm, (fm.shape[1],), state[prefix + "fmb.layer_norm.weight"],
                      state[prefix + "fmb.layer_norm.bias"], 1e-5)
    h = fm
    for i in range(n_fmb_hidden + 1):       # Linear, ReLU pairs: mlp_block with mlp_layout(n, output_act="relu")
        h = F.linear(h, state[prefix + "fmb.mlp.mlp.%d.weight" % (2 * i)], state[prefix + "fmb.mlp.mlp.%d.bias" % (2 * i)])
        if margins is not None:
            margins.append(h.detach().abs().amin(dim=1) if h.shape[0] else h.new_zeros(0))
        h = h.relu()
    fmb = h.reshape(B, h.shape[1] // D, D)
    lcb = F.linear(x.transpose(1, 2), state[prefix + "lcb.linear.weight"]).transpose(1, 2)
    out = torch.cat([fmb, lcb], dim=1)
    if prefix + "residual_proj.weight" in state:
        out = out + F.linear(x.transpose(1, 2), state[prefix + "residual_proj.weight"],
                             state[prefix + "residual_proj.bias"]).transpose(1, 2)
    else:
        out = out + x
    if layer_norm:
        out = F.layer_norm(out, (D,), state[prefix + "layer_norm.weight"], state[prefix + "layer_norm.bias"], 1e-5)
    return out


def fc_layout(n_hidden, batch_norm):
    layout = []
    for _ in range(n_hidden):
        layout += ["linear"] + (["bn"] if batch_norm else []) + ["relu"]
    return layout + ["linear"]


def wukong_logit(specs, state, X, num_layers, n_fmb_hidden, n_fc_hidden, batch_norm, layer_norm=True,
                 training=True):
    """WuKong.forward (pre-sigmoid): the layer stack, then fc over the flatten."""
    x = feature_embedding(specs, state, "embedding_layer.", X)
    for i in range(num_layers):
        x = wukong_layer(x, state, "wukong_stack.%d." % i, n_fmb_hidden, layer_norm)
    return mlp_block(x.flatten(start_dim=1), state, "fc.", fc_layout(n_fc_hidden, batch_norm), training)

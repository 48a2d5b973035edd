"""Float64 restatement of MaskNet (model_zoo/MaskNet/src/MaskNet.py: MaskBlock, SerialMaskNet, ParallelMaskNet,
MaskNet) for the MaskNet tests, built on the shared oracle's embedding and MLP restatements
(oracle/fuxictr_oracle.py) and pinned to the reference's goldens by tests/test_masknet_host.py.  Every block's mask
MLP reads the un-normalised V_emb, as the reference's does.  Test infrastructure only: nothing under fuxictr_b200/
imports it."""
import os
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle.fuxictr_oracle import feature_embedding, mlp_block, mlp_layout  # noqa: E402

ACTS = {"relu": torch.relu, "sigmoid": torch.sigmoid}


def mask_block(state, prefix, V_emb, V_hidden, act="relu", ln=True, keep=None, scale=1.0, eps=1e-5):
    """MaskBlock.forward; keep: the block's (B, n) dropout mask (1 kept, 0 dropped), kept values times scale."""
    h = torch.relu(F.linear(V_emb, state[prefix + "mask_layer.0.weight"], state[prefix + "mask_layer.0.bias"]))
    v_mask = F.linear(h, state[prefix + "mask_layer.2.weight"], state[prefix + "mask_layer.2.bias"])
    z = F.linear(v_mask * V_hidden, state[prefix + "hidden_layer.0.weight"])
    if ln:
        z = F.layer_norm(z, (z.shape[-1],), state[prefix + "hidden_layer.1.weight"],
                         state[prefix + "hidden_layer.1.bias"], eps)
    y = ACTS[act](z)
    if keep is not None:
        y = y * keep * scale
    return y


def field_layernorm(state, prefix, emb, num_fields, eps=1e-5):
    """cat_f LayerNorm_f(emb[:, f]) of the flattened (B, F D) embedding."""
    D = emb.shape[1] // num_fields
    parts = [F.layer_norm(emb[:, f * D:(f + 1) * D], (D,), state["%s%d.weight" % (prefix, f)],
                          state["%s%d.bias" % (prefix, f)], eps) for f in range(num_fields)]
    return torch.cat(parts, dim=1)


def masknet_logit(specs, state, X, kwargs, keeps=None, scale=1.0):
    """MaskNet.forward before the output sigmoid.  keeps: per block, its dropout mask or None."""
    emb = feature_embedding(specs, state, "embedding_layer.", X, flatten_emb=True)
    nf = len(specs)
    hidden = field_layernorm(state, "emb_norm.", emb, nf) if kwargs.get("emb_layernorm", True) else emb
    act = str(kwargs.get("dnn_hidden_activations", "ReLU")).lower()
    ln = kwargs.get("net_layernorm", True)
    units = list(kwargs.get("dnn_hidden_units", [64, 64, 64]))
    keeps = keeps or {}
    if kwargs.get("model_type", "SerialMaskNet") == "SerialMaskNet":
        v = hidden
        for i in range(len(units)):
            v = mask_block(state, "mask_net.mask_blocks.%d." % i, emb, v, act, ln, keeps.get(i), scale)
        return F.linear(v, state["mask_net.fc.0.weight"], state["mask_net.fc.0.bias"])
    nb = kwargs.get("parallel_num_blocks", 1)
    cat = torch.cat([mask_block(state, "mask_net.mask_blocks.%d." % i, emb, hidden, act, ln, keeps.get(i), scale)
                     for i in range(nb)], dim=1)
    return mlp_block(cat, state, "mask_net.dnn.", mlp_layout(len(units), hidden_act=act))

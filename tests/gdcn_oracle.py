"""Float64 restatement of GDCN (model_zoo/GDCN/src/GDCN.py: GateCorssLayer, GDCN, GDCNP) for the GDCN tests, built
on the shared oracle's embedding and MLP restatements (oracle/fuxictr_oracle.py) and pinned to the reference's
goldens by tests/test_gdcn_host.py.  Test infrastructure only: nothing under fuxictr_b200/ imports it."""
import os
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle.fuxictr_oracle import feature_embedding, mlp_block, mlp_layout  # noqa: E402


def gated_cross_layer(x0, xi, w, wg, b):
    """One GateCorssLayer step: x0 * (xi W^T + b) * sigmoid(xi Wg^T) + xi."""
    return x0 * (F.linear(xi, w) + b) * torch.sigmoid(F.linear(xi, wg)) + xi


def gate_cross_net(x0, state, prefix, cn_layers):
    """GateCorssLayer.forward."""
    x = x0
    for i in range(cn_layers):
        x = gated_cross_layer(x0, x, state["%sw.%d.weight" % (prefix, i)], state["%swg.%d.weight" % (prefix, i)],
                              state["%sb.%d" % (prefix, i)])
    return x


def gdcn_logit(specs, state, X, cn_layers, n_hidden):
    """GDCN.forward (pre-sigmoid): the DNN, which ends in the logit, over the gated cross network."""
    emb = feature_embedding(specs, state, "embedding_layer.", X, flatten_emb=True)
    return mlp_block(gate_cross_net(emb, state, "cross_net.", cn_layers), state, "dnn.", mlp_layout(n_hidden))


def gdcnp_logit(specs, state, X, cn_layers, n_hidden):
    """GDCNP.forward (pre-sigmoid): fc over [gated cross network | DNN tower]."""
    emb = feature_embedding(specs, state, "embedding_layer.", X, flatten_emb=True)
    cross = gate_cross_net(emb, state, "cross_net.", cn_layers)
    dnn = mlp_block(emb, state, "dnn.", mlp_layout(n_hidden, has_output=False))
    return F.linear(torch.cat([cross, dnn], dim=1), state["fc.weight"], state["fc.bias"])

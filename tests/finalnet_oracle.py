"""Float64 restatement of FinalNet (model_zoo/FinalNet/src/FinalNet.py: FeatureGating, FactorizedInteraction,
FinalBlock, FinalNet and its add_loss) for the FinalNet tests, built on the shared oracle's embedding restatement
(oracle/fuxictr_oracle.py).  Test infrastructure only: nothing under fuxictr_b200/ imports it."""
import os
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle.fuxictr_oracle import feature_embedding  # noqa: E402

ACTS = {None: lambda z: z, "ReLU": torch.relu, "relu": torch.relu, "Sigmoid": torch.sigmoid,
        "sigmoid": torch.sigmoid}


def feature_gating(e, state, prefix):
    """FeatureGating.forward (gate_residual "concat") on e (B, F, D) -> (B, 2 F, D)."""
    gates = F.linear(e.transpose(1, 2), state[prefix + "linear.weight"], state[prefix + "linear.bias"]).transpose(1, 2)
    return torch.cat([e, e * gates], dim=1)


def final_block(x, state, prefix, n_layers, residual_type, activations, batch_norm, training, eps=1e-5):
    """FinalBlock.forward without dropout on x (B, d_in): per layer the FactorizedInteraction, BatchNorm1d (batch
    statistics in training, the running ones in eval; no running-statistics update) and the activation."""
    if not isinstance(activations, list):
        activations = [activations] * n_layers
    for i in range(n_layers):
        h = F.linear(x, state[prefix + "layer.%d.linear.weight" % i], state[prefix + "layer.%d.linear.bias" % i])
        h2, h1 = torch.chunk(h, chunks=2, dim=-1)
        x = torch.cat([h2, h1 * h2], dim=-1) if residual_type == "concat" else h2 + h1 * h2
        if batch_norm:
            norm = prefix + "norm.%d." % i
            if training:
                mu, var = x.mean(0), x.var(0, unbiased=False)
            else:
                mu, var = state[norm + "running_mean"], state[norm + "running_var"]
            x = (x - mu) / torch.sqrt(var + eps) * state[norm + "weight"] + state[norm + "bias"]
        x = ACTS[activations[i]](x)
    return x


def finalnet_logits(specs, state, X, kw, training=True):
    """(y1, y2) of FinalNet.forward (y2 None with block_type "1B"); kw: the model's keyword arguments."""
    e = feature_embedding(specs, state, "embedding_layer.", X)
    bn, res = kw.get("batch_norm", True), kw.get("residual_type", "concat")
    u1 = kw.get("block1_hidden_units", [64, 64, 64])
    x1 = feature_gating(e, state, "feature_gating.") if kw.get("use_feature_gating", False) else e
    b1 = final_block(x1.flatten(start_dim=1), state, "block1.", len(u1), res, kw.get("block1_hidden_activations"),
                     bn, training)
    y1 = F.linear(b1, state["fc1.weight"], state["fc1.bias"])
    if kw.get("block_type", "2B") == "1B":
        return y1, None
    u2 = kw.get("block2_hidden_units", [64, 64, 64])
    b2 = final_block(e.flatten(start_dim=1), state, "block2.", len(u2), res, kw.get("block2_hidden_activations"),
                     bn, training)
    return y1, F.linear(b2, state["fc2.weight"], state["fc2.bias"])


def finalnet_loss(y1, y2, y):
    """(loss, y_pred) of FinalNet.add_loss."""
    if y2 is None:
        y_pred = torch.sigmoid(y1)
        return F.binary_cross_entropy(y_pred, y), y_pred
    y_pred = torch.sigmoid(0.5 * (y1 + y2))
    loss = F.binary_cross_entropy(y_pred, y)
    loss = loss + F.binary_cross_entropy(torch.sigmoid(y1), y_pred.detach())
    return loss + F.binary_cross_entropy(torch.sigmoid(y2), y_pred.detach()), y_pred

"""Float64 restatement of DIEN (model_zoo/DIEN/src/DIEN.py: the GRUs, AttentionLayer, DIEN) for the DIEN tests, written
from the model's math on padded sequences and masks (no packing), on the shared oracle's embedding and MLP
restatements (oracle/fuxictr_oracle.py).  Test infrastructure only: nothing under fuxictr_b200/ imports it."""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle.fuxictr_oracle import feature_embedding_dict, mlp_block  # noqa: E402


def _flat(field):
    return list(field) if isinstance(field, (list, tuple)) else [field]


def gru_sequence(x, mask, W_ih, b_ih, W_hh, b_hh, cell="GRU", att=None):
    """(h_seq, h_last): the recurrence over each sample's first len = mask.sum(1) positions from h = 0; h_seq zero from
    len on, h_last the state after step len - 1 (zero for an empty history)."""
    B, L, H = x.shape
    lens = mask.sum(dim=1)
    h = x.new_zeros(B, H)
    outs = []
    for t in range(L):
        i0, i1, i2 = (x[:, t] @ W_ih.t() + b_ih).chunk(3, 1)
        g0, g1, g2 = (h @ W_hh.t() + b_hh).chunk(3, 1)
        if cell == "GRU":
            r, z = torch.sigmoid(i0 + g0), torch.sigmoid(i1 + g1)
            n = torch.tanh(i2 + r * g2)
            hn = (1 - z) * n + z * h
        else:
            r = torch.sigmoid(i1 + g1)
            n = torch.tanh(i2 + r * g2)
            a = att[:, t].unsqueeze(-1)
            u = a * torch.sigmoid(i0 + g0) if cell == "AUGRU" else a
            hn = h + u * (n - h)
        on = (t < lens).unsqueeze(-1)
        h = torch.where(on, hn, h)
        outs.append(torch.where(on, hn, torch.zeros_like(hn)))
    return torch.stack(outs, dim=1), h


def attention(interest, target, mask, state, prefix, kw):
    """AttentionLayer.forward: bilinear, dot or din_attention scores, times the mask, optionally softmaxed."""
    kind = kw.get("attention_type", "bilinear_attention")
    B, L, H = interest.shape
    m = mask.to(interest.dtype)
    if kind == "dot_attention":
        s = (interest @ target.unsqueeze(-1)).view(B, L)
    elif kind == "bilinear_attention":
        s = ((interest @ state[prefix + "W_kernel"]) @ target.unsqueeze(-1)).view(B, L)
    else:
        t = target.unsqueeze(1).expand(-1, L, -1)
        din = torch.cat([t, interest, t - interest, t * interest], dim=-1).view(-1, 4 * H)
        act = str(kw.get("attention_activation", "Dice")).lower()
        layout = []
        for _ in kw.get("attention_hidden_units", [80, 40]):
            layout += ["linear", act]
        s = mlp_block(din, state, prefix + "attn_mlp.", layout + ["linear"]).view(B, L)
    s = s * m
    if kw.get("use_attention_softmax", True):
        s = (s + -1.e9 * (1 - m)).softmax(dim=-1)
    return s


def interest_stack(k, seq, target, mask, state, kw):
    """h_out (B, H) of pair k: extractor GRU, attention, evolution GRU (AUGRU, AGRU or GRU)."""
    ext, evo = "extraction_modules.%d." % k, "evolving_modules.%d." % k
    gru_type = kw.get("gru_type", "AUGRU")

    def w(p):
        return state[p + "weight_ih_l0"], state[p + "bias_ih_l0"], state[p + "weight_hh_l0"], state[p + "bias_hh_l0"]
    interest, _ = gru_sequence(seq, mask, *w(ext))
    if gru_type == "GRU":
        return gru_sequence(interest, mask, *w(evo))[1]
    att = attention(interest, target, mask, state, "attention_modules.%d." % k, kw)
    c = evo + "gru_cell."
    return gru_sequence(interest, mask, state[c + "x2h.weight"], state[c + "x2h.bias"], state[c + "h2h.weight"],
                        state[c + "h2h.bias"], cell=gru_type, att=att)[1]


def dnn_layout(kw):
    act = str(kw.get("dnn_activations", "ReLU")).lower()
    layout = []
    for _ in kw.get("dnn_hidden_units", [200, 80]):
        layout += ["linear"] + (["bn"] if kw.get("batch_norm", True) else []) + [act]
    return layout + ["linear"]


def dien_logit(specs, state, X, kw):
    """DIEN.forward (pre-sigmoid): per pair h_out (then the sum pooling and its product with the target), then the
    remaining 2-D embeddings in FeatureMap order without the neg-sequence fields, then the DNN."""
    emb = feature_embedding_dict(specs, state, "embedding_layer.", X)
    targets = kw.get("dien_target_field", [("item_id", "cate_id")])
    sequences = kw.get("dien_sequence_field", [("click_history", "cate_history")])
    targets = targets if isinstance(targets, list) else [targets]
    sequences = sequences if isinstance(sequences, list) else [sequences]
    negs = set(n for f in kw.get("dien_neg_seq_field", []) for n in _flat(f))
    parts = []
    for k, (target, sequence) in enumerate(zip(targets, sequences)):
        tgt = torch.cat([emb[n] for n in _flat(target)], dim=-1)
        seq = torch.cat([emb[n] for n in _flat(sequence)], dim=-1)
        mask = X[_flat(sequence)[0]].long() > 0
        parts.append(interest_stack(k, seq, tgt, mask, state, kw))
        if kw.get("enable_sum_pooling", False):
            pooled = seq.sum(dim=1)
            parts += [pooled, tgt * pooled]
    parts += [e for n, e in emb.items() if e.dim() == 2 and n not in negs]
    return mlp_block(torch.cat(parts, dim=-1), state, "dnn.", dnn_layout(kw))

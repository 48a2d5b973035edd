"""Float64 restatement of SIM's and TWIN's interest blocks (model_zoo/LongCTR/SIM/SIM.py, model_zoo/LongCTR/TWIN/TWIN.py)
for the SIM / TWIN tests, written from the models' math.  The top-k follows the project's tie rule: descending score,
ties to the lower position, -0.0 equal to +0.0.  Test infrastructure only: nothing under fuxictr_b200/ imports it."""
import torch

from longctr_oracle import mhta, short_window


def select(scores, k):
    """The k positions of largest score along the last axis, sorted by (score desc, position asc).  Comparisons are on
    values, so -0.0 and +0.0 tie."""
    L = scores.shape[-1]
    order = torch.arange(L, device=scores.device).expand(scores.shape)
    # a stable sort on the negated scores keeps equal scores in ascending position; + 0.0 folds -0.0 into +0.0
    idx = torch.sort(-scores + 0.0, dim=-1, stable=True).indices
    return torch.gather(order, -1, idx)[..., :k]


def sim_block(x, mask, short_seq_len, topk, heads, W_a, W_b, Ws, Wl):
    """(target, short, long, pooled, positions) of SIM's interest block on x (B, L + 1, d)."""
    target = x[:, -1]
    hs, ms = short_window(x, mask, short_seq_len)
    short = mhta(target, hs, ms, heads, True, Ws)
    hist = x[:, :-1]
    qk = torch.einsum("ba,bla->bl", target @ W_a.t(), hist @ W_b.t()) * (mask != 0).to(x.dtype)
    pooled = torch.einsum("bl,bld->bd", qk, hist)
    k = min(topk, mask.shape[1])
    pos = select(qk.detach(), k)
    emb = torch.gather(hist, 1, pos.unsqueeze(-1).expand(-1, -1, x.shape[-1]))
    long = mhta(target, emb, torch.gather(mask, 1, pos), heads, True, Wl)
    return target, short, long, pooled, pos


def topk_attention(target, hist, mask, heads, topk, W):
    """MultiHeadTopKAttention with Kc = 0 and no dropout; W = (W_q, W_h, W_v, W_o).  Returns (out, positions (B, H, k))."""
    B, L, _ = hist.shape
    A = W[0].shape[0]
    hd = A // heads
    q = (target @ W[0].t()).view(B, heads, 1, hd)
    kh = (hist @ W[1].t()).view(B, L, heads, hd).transpose(1, 2)
    v = (hist @ W[2].t()).view(B, L, heads, hd).transpose(1, 2)
    s = (q @ kh.transpose(-1, -2)).squeeze(2) / hd ** 0.5                     # (B, H, L)
    s = s.masked_fill(mask.view(B, 1, L) == 0, -1e9)
    k = min(topk, L)
    pos = select(s.detach(), k)
    a = torch.softmax(torch.gather(s, 2, pos), dim=-1)
    vv = torch.gather(v, 2, pos.unsqueeze(-1).expand(-1, -1, -1, hd))
    out = (a.unsqueeze(2) @ vv).squeeze(2).reshape(B, A)
    return out @ W[3].t(), pos


def twin_block(x, mask, short_seq_len, topk, heads, Ws, Wt):
    """(target, short, long, positions) of TWIN's interest block on x (B, L + 1, d)."""
    target = x[:, -1]
    hs, ms = short_window(x, mask, short_seq_len)
    short = mhta(target, hs, ms, heads, True, Ws)
    long, pos = topk_attention(target, x[:, :-1], mask, heads, topk, Wt)
    return target, short, long, pos


def model_logits(name, state, fm, triple, kw):
    """SIM's (main, auxiliary) or TWIN's (main,) pre-sigmoid logits (B, 1) on a LongCTR triple, from a float64 state:
    table lookups, the interest block, then the DNNs (Linear / ReLU, no batch norm)."""
    batch_dict, item_dict, mask = triple

    def lookup(f, ids):         # nn.Embedding(padding_idx): the padding row gets no gradient
        table = state["embedding_layer.embedding_layer.embedding_layers.%s.weight" % f]
        return torch.nn.functional.embedding(ids.long(), table, padding_idx=fm.features[f].get("padding_idx"))

    def dnn(prefix, h):
        i = 0
        while "%s.mlp.%d.weight" % (prefix, i) in state:
            h = torch.nn.functional.linear(h, state["%s.mlp.%d.weight" % (prefix, i)], state["%s.mlp.%d.bias" % (prefix, i)])
            if "%s.mlp.%d.weight" % (prefix, i + 2) in state:
                h = torch.relu(h)
            i += 2
        return h

    feats = list(fm.features.keys())
    batch = [lookup(f, batch_dict[f]) for f in feats if f in batch_dict and f not in fm.labels]
    items = torch.cat([lookup(f, item_dict[f]) for f in feats if f in item_dict], dim=-1)
    B = mask.shape[0]
    x = items.view(B, mask.shape[1] + 1, -1)
    att = lambda p, names=("W_q", "W_k", "W_v", "W_o"): tuple(state["%s.%s.weight" % (p, n)] for n in names)  # noqa
    if name == "SIM":
        target, short, long, pooled, _ = sim_block(x, mask, kw["short_seq_len"], kw["topk"], kw["num_heads"],
                                                   state["W_a.weight"], state["W_b.weight"], att("short_attention"),
                                                   att("long_attention"))
        return dnn("dnn", torch.cat(batch + [target, short, long], dim=-1)), \
            dnn("dnn_aux", torch.cat(batch + [target, pooled], dim=-1))
    target, short, long, _ = twin_block(x, mask, kw["short_seq_len"], kw["topk"], kw["num_heads"],
                                        att("short_attention"), att("long_attention", ("W_q", "W_h", "W_v", "W_o")))
    return (dnn("dnn", torch.cat(batch + [target, short, long], dim=-1)),)

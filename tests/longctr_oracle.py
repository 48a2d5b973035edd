"""Float64 restatement of ETA's and SDIM's interest blocks (model_zoo/LongCTR/ETA/ETA.py, model_zoo/LongCTR/SDIM/SDIM.py)
for the LongCTR tests, written from the models' math.  ETA's top-k follows the project's tie rule: ascending
(distance, position).  Test infrastructure only: nothing under fuxictr_b200/ imports it."""
import torch


def mhta(t, h, mask, heads, use_scale, W=None):
    """MultiHeadTargetAttention with ScaledDotProductAttention (no dropout); W = (W_q, W_k, W_v, W_o) or None."""
    if W is not None:
        q, k, v = t @ W[0].t(), h @ W[1].t(), h @ W[2].t()
    else:
        q, k, v = t, h, h
    B = q.shape[0]
    hd = q.shape[-1] // heads
    q = q.view(B, 1, heads, hd).transpose(1, 2)
    k = k.view(B, -1, heads, hd).transpose(1, 2)
    v = v.view(B, -1, heads, hd).transpose(1, 2)
    s = q @ k.transpose(-1, -2)
    if use_scale:
        s = s / hd ** 0.5
    s = s.masked_fill(mask.view(B, 1, 1, -1) == 0, -1e9)
    out = (torch.softmax(s, dim=-1) @ v).transpose(1, 2).reshape(B, heads * hd)
    return out @ W[3].t() if W is not None else out


def simhash(x, R):
    """Bits (..., L, n) of x (B, L, d) under R (1 or B, d, n): x . R[:, j] > 0."""
    return torch.einsum("bld,bdn->bln", x, R.expand(x.shape[0], *R.shape[1:])) > 0


def eta_distances(x, mask, R):
    """(B, L) Hamming distances of the history rows of x (B, L + 1, d) to the target, 1 + bits where masked."""
    code = simhash(x, R)
    dist = (code[:, :-1] ^ code[:, -1:]).sum(-1)
    return torch.where(mask != 0, dist, torch.full_like(dist, R.shape[-1] + 1))


def select(dist, k):
    """The k positions of smallest distance per row, sorted by (distance, position)."""
    L = dist.shape[1]
    key = dist.long() * (L + 1) + torch.arange(L, device=dist.device)
    return key.argsort(dim=1)[:, :k]


def short_window(x, mask, short_seq_len):
    s = short_seq_len
    return x[:, -s:-1], mask[:, -s:-1]


def eta_block(x, mask, R, short_seq_len, topk, heads, use_scale, Ws, Wl):
    """(target, short, long, positions) of ETA's interest block on x (B, L + 1, d)."""
    target = x[:, -1]
    hs, ms = short_window(x, mask, short_seq_len)
    short = mhta(target, hs, ms, heads, use_scale, Ws)
    k = min(topk, mask.shape[1])
    pos = select(eta_distances(x.detach(), mask, R), k)
    hist = x[:, :-1]
    emb = torch.gather(hist, 1, pos.unsqueeze(-1).expand(-1, -1, x.shape[-1]))
    long = mhta(target, emb, torch.gather(mask, 1, pos), heads, use_scale, Wl)
    return target, short, long, pos


def sdim_buckets(x, R):
    """(B, L + 1, num_hashes) integer buckets under R (1 or B, d, num_hashes, bits)."""
    B, L1, d = x.shape
    nh, bits = R.shape[-2], R.shape[-1]
    code = simhash(x, R.reshape(R.shape[0], d, nh * bits)).view(B, L1, nh, bits).long()
    return (code << torch.arange(bits, device=x.device)).sum(-1)


def sdim_block(x, mask, R, short_seq_len, l2_norm, heads, use_scale, Ws):
    """(target, short, long) of SDIM's interest block on x (B, L + 1, d)."""
    target = x[:, -1]
    hs, ms = short_window(x, mask, short_seq_len)
    short = mhta(target, hs, ms, heads, use_scale, Ws)
    bk = sdim_buckets(x.detach(), R)
    collide = (bk[:, :-1] == bk[:, -1:]) & (mask != 0).unsqueeze(-1)          # (B, L, nh)
    sums = torch.einsum("blh,bld->bhd", collide.to(x.dtype), x[:, :-1])
    if l2_norm:
        sums = torch.nn.functional.normalize(sums, dim=-1)
    return target, short, sums.mean(dim=1)


def model_logit(name, state, fm, triple, kw):
    """ETA's or SDIM's pre-sigmoid logit (B, 1) on a LongCTR triple, from a float64 state: table lookups, the interest
    block with the shared rotations, then the DNN (Linear / ReLU, no batch norm)."""
    batch_dict, item_dict, mask = triple
    def lookup(f, ids):         # nn.Embedding(padding_idx): the padding row gets no gradient
        table = state["embedding_layer.embedding_layer.embedding_layers.%s.weight" % f]
        return torch.nn.functional.embedding(ids.long(), table, padding_idx=fm.features[f].get("padding_idx"))
    feats = list(fm.features.keys())
    batch = [lookup(f, batch_dict[f]) for f in feats if f in batch_dict and f not in fm.labels]
    items = torch.cat([lookup(f, item_dict[f]) for f in feats if f in item_dict], dim=-1)
    B = mask.shape[0]
    x = items.view(B, mask.shape[1] + 1, -1)
    att = lambda p: tuple(state["%s.%s.weight" % (p, n)] for n in ("W_q", "W_k", "W_v", "W_o")) \
        if "%s.W_q.weight" % p in state else None                                             # noqa: E731
    R = state["random_rotations"]
    if name == "ETA":
        target, short, long, _ = eta_block(x, mask, R, kw["short_seq_len"], kw["topk"], kw["num_heads"],
                                           kw.get("use_scale", True), att("short_attention"), att("long_attention"))
        h = torch.cat(batch + [target, short, long], dim=-1)
    else:
        target, short, long = sdim_block(x, mask, R, kw["short_seq_len"], kw.get("l2_norm", False), kw["num_heads"],
                                         kw.get("use_scale", True), att("short_attention"))
        h = torch.cat(batch + [target, long, short], dim=-1)
    i = 0
    while "dnn.mlp.%d.weight" % i in state:
        h = torch.nn.functional.linear(h, state["dnn.mlp.%d.weight" % i], state["dnn.mlp.%d.bias" % i])
        if "dnn.mlp.%d.weight" % (i + 2) in state:
            h = torch.relu(h)
        i += 2
    return h

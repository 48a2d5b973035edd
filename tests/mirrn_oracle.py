"""Float64 restatement of MIRRN's interest block (model_zoo/LongCTR/MIRRN/MIRRN.py) for the MIRRN tests, written from
the model's math.  FilterLayer2 runs through torch.fft exactly as the reference writes it, so it checks the kernels'
closed form (a u + b H u) independently.  The retrievals follow the project's tie rule: the k smallest distances, ties
to the lower position, then in ascending position order.  A mean query is hashed from its masked sum: dividing by
count + 1e-9 keeps every sign.  Test infrastructure only: nothing under fuxictr_b200/ imports it."""
import torch

from longctr_oracle import mhta, short_window


def rotation_sets(R):
    """The (d, bits) rotations of the three retrievals (target, short, global) from (d, bits) or (3, d, bits)."""
    return [R] * 3 if R.dim() == 2 else [R[0], R[1], R[2]]


def query_sums(x, mask):
    """(B, 3, d): the target, the masked sum of the last min(16, L) history rows and the masked sum of all of them."""
    h = x[:, :-1] * (mask != 0).unsqueeze(-1).to(x.dtype)
    return torch.stack([x[:, -1], h[:, -16:].sum(1), h.sum(1)], dim=1)


def distances(x, mask, R):
    """(B, 3, L) Hamming distances of the history rows to the three queries, bits + 1 where masked."""
    xd = x.detach()
    qs = query_sums(xd, mask)
    out = []
    for q, Rq in enumerate(rotation_sets(R)):
        hist = (xd[:, :-1] @ Rq) > 0
        code = (qs[:, q] @ Rq) > 0
        dist = (hist ^ code.unsqueeze(1)).sum(-1)
        out.append(torch.where(mask != 0, dist, torch.full_like(dist, Rq.shape[-1] + 1)))
    return torch.stack(out, dim=1)


def select(dist, k):
    """(..., k) positions of the k smallest distances per row (ties to the lower position), ascending."""
    L = dist.shape[-1]
    key = dist.long() * (L + 1) + torch.arange(L, device=dist.device)
    return key.argsort(dim=-1)[..., :k].sort(dim=-1).values


def filter_layer(u, cw, gamma, beta, eps=1e-12):
    """FilterLayer2.forward without dropout: LN(irfft(rfft(u) W) + u), W the diagonal-block einsum of complex_weight."""
    B, k, d = u.shape
    n = cw.shape[0]
    A = torch.fft.rfft(u, dim=1, norm="ortho").view(B, k // 2 + 1, n, d // n)
    W = torch.view_as_complex(cw.contiguous())
    C = torch.einsum("blnd,ndd->blnd", A, W).reshape(B, k // 2 + 1, d)
    z = torch.fft.irfft(C, n=k, dim=1, norm="ortho") + u
    mu = z.mean(-1, keepdim=True)
    var = (z - mu).pow(2).mean(-1, keepdim=True)
    return gamma * (z - mu) / torch.sqrt(var + eps) + beta


def mirrn_block(x, mask, R, short_seq_len, topk, heads, use_scale, Ws, Wl, pos_table, cws, gammas, betas):
    """(target, short, long, positions (B, 3, k), interests (B, 3, d)) of MIRRN's interest block on x (B, L + 1, d)."""
    target = x[:, -1]
    hs, ms = short_window(x, mask, short_seq_len)
    short = mhta(target, hs, ms, heads, use_scale, Ws)
    L = mask.shape[1]
    k = min(topk, L)
    pos = select(distances(x, mask, R), k)
    hist = x[:, :-1]
    interests = []
    for q in range(3):
        idx = pos[:, q]
        u = torch.gather(hist, 1, idx.unsqueeze(-1).expand(-1, -1, x.shape[-1])) + pos_table[L - idx] * 0.02
        interests.append(filter_layer(u, cws[q], gammas[q], betas[q]).mean(1))
    interests = torch.stack(interests, dim=1)
    long = mhta(target, interests, torch.ones(x.shape[0], 3, dtype=x.dtype), heads, use_scale, Wl)
    return target, short, long, pos, interests


def block_params(state, prefix=""):
    """(Ws, Wl, pos_table, cws, gammas, betas) of a MIRRN state dict."""
    att = lambda p: tuple(state["%s%s.%s.weight" % (prefix, p, n)] for n in ("W_q", "W_k", "W_v", "W_o"))  # noqa
    blk = lambda q, n: state["%sMHFT_block.%d.%s" % (prefix, q, n)]                                   # noqa: E731
    return (att("short_attention"), att("long_attention"), state[prefix + "pos.weight"],
            [blk(q, "complex_weight") for q in range(3)], [blk(q, "LayerNorm.weight") for q in range(3)],
            [blk(q, "LayerNorm.bias") for q in range(3)])


def model_logit(state, fm, triple, kw):
    """MIRRN's pre-sigmoid logit (B, 1) on a LongCTR triple from a float64 state, with the shared rotations and no
    filter dropout: table lookups, the interest block, then the DNN (Linear / ReLU, no batch norm)."""
    batch_dict, item_dict, mask = triple

    def lookup(f, ids):
        table = state["embedding_layer.embedding_layer.embedding_layers.%s.weight" % f]
        return torch.nn.functional.embedding(ids.long(), table, padding_idx=fm.features[f].get("padding_idx"))
    feats = list(fm.features.keys())
    batch = [lookup(f, batch_dict[f]) for f in feats if f in batch_dict and f not in fm.labels]
    items = torch.cat([lookup(f, item_dict[f]) for f in feats if f in item_dict], dim=-1)
    B = mask.shape[0]
    x = items.view(B, mask.shape[1] + 1, -1)
    Ws, Wl, P, cws, gammas, betas = block_params(state)
    target, short, long = mirrn_block(x, mask, state["random_rotations"], kw["short_seq_len"], kw["topk"],
                                      kw["num_heads"], kw.get("use_scale", True), Ws, Wl, P, cws, gammas, betas)[:3]
    h = torch.cat(batch + [target, short, long], dim=-1)
    i = 0
    while "dnn.mlp.%d.weight" % i in state:
        h = torch.nn.functional.linear(h, state["dnn.mlp.%d.weight" % i], state["dnn.mlp.%d.bias" % i])
        if "dnn.mlp.%d.weight" % (i + 2) in state:
            h = torch.relu(h)
        i += 2
    return h

"""MIRRN on the GPU at two shapes: MIRRN_default (B 8192, D 16, three item fields so d 48, L 50, topk 4, 4 heads,
attention_dim 32, DNN [64, 32]) and a long shape (B 4096, L 1000, topk 50), each with one user field and pre-padded
histories of random length.

Times (CUDA events, median over the timed repeats after warm-up):
  - the interest block forward, and forward + backward, each captured into a CUDA graph and timed as replays: torch
    eager fp32 restating the reference's ops (three matmul hashes of the whole history, topk + sort + gather, rfft /
    einsum / irfft filters with LayerNorm, the two target attentions), and functional.mirrn_interest on the kernels
    in fp32, tf32x3, tf32 and bf16, training mode (filter dropout on in both);
  - the whole fused_train_step in samples/s, in the four modes (eager launches, as the model's users call it);
  - b2_mirrn_retrieve_fwd, b2_mirrn_filter_fwd and b2_mirrn_filter_bwd alone, with TB/s from the bytes they must move:
    retrieval the B (L + 1) d rows, the mask and the positions; the filter the gathered rows and their pos rows, u and
    y (forward) or dy, dres, u, du and the dpos rows (backward).
Prints one JSON object, with the card's name and power limit read in the same run.

    python tools/mirrn_times.py [--repeats 20]
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from longctr_times import card, timed  # noqa: E402
from transact_times import graphed  # noqa: E402
from sim_twin_times import eager_mhta  # noqa: E402

MODES = ("fp32", "tf32x3", "tf32", "bf16")
KW = dict(embedding_dim=16, dnn_hidden_units=[64, 32], attention_dim=32, num_heads=4, hash_bits=32,
          short_seq_len=50)
SHAPES = {"default": dict(batch=8192, L=50, topk=4), "long": dict(batch=4096, L=1000, topk=50)}


def fm_and_triple(B, L, gen):
    from fuxictr_b200.schema import FeatureMap
    specs = [("user_id", {"type": "categorical", "source": "user", "padding_idx": 0, "vocab_size": 500}),
             ("item_id", {"type": "categorical", "source": "item", "padding_idx": 0, "vocab_size": 3000}),
             ("cate_id", {"type": "categorical", "source": "item", "padding_idx": 0, "vocab_size": 60}),
             ("brand_id", {"type": "categorical", "source": "item", "padding_idx": 0, "vocab_size": 200})]
    fm = FeatureMap.from_specs(specs, embedding_dim=KW["embedding_dim"])
    lens = torch.randint(0, L + 1, (B,), generator=gen)
    hist = torch.randint(1, 3000, (B, L), generator=gen) * (torch.arange(L).view(1, -1) >= (L - lens).view(-1, 1))
    items = torch.cat([hist, torch.randint(1, 3000, (B, 1), generator=gen)], dim=1).flatten()
    idict = {"item_id": items, "cate_id": torch.where(items > 0, items % 59 + 1, torch.zeros_like(items)),
             "brand_id": torch.where(items > 0, items % 199 + 1, torch.zeros_like(items))}
    bd = {"user_id": torch.randint(1, 500, (B,), generator=gen), "label": (torch.rand(B, generator=gen) < 0.3).double()}
    return fm, ({k: v.cuda() for k, v in bd.items()}, {k: v.cuda() for k, v in idict.items()}, (hist > 0).float().cuda())


def eager_filter(u, blk):
    B, k, d = u.shape
    A = torch.fft.rfft(u, dim=1, norm="ortho").view(B, k // 2 + 1, 4, d // 4)
    C = torch.einsum("blnd,ndd->blnd", A, torch.view_as_complex(blk.complex_weight)).reshape(B, k // 2 + 1, d)
    h = torch.nn.functional.dropout(torch.fft.irfft(C, n=k, dim=1, norm="ortho"), 0.1, True) + u
    return blk.LayerNorm(h)


def eager_mirrn(x, mask, model, topk):
    """MIRRN.forward's interest block as the reference writes it, in eager fp32."""
    S, heads = KW["short_seq_len"], model.short_attention.num_heads
    mw = lambda a: (a.W_q.weight, a.W_k.weight, a.W_v.weight, a.W_o.weight)    # noqa: E731
    t, seq = x[:, -1], x[:, :-1]
    short = eager_mhta(t, x[:, -S:-1], mask[:, -S:-1], mw(model.short_attention), heads)
    R = model.random_rotations
    mm = lambda v, m: (v * m.unsqueeze(-1)).sum(1) / (m.unsqueeze(-1).sum(1) + 1e-9)     # noqa: E731
    ints = []
    for q, query in enumerate((t, mm(seq[:, -16:], mask[:, -16:]), mm(seq, mask))):
        qh = torch.relu(torch.sign(query.unsqueeze(1) @ R))
        sh = torch.relu(torch.sign(seq @ R))
        sim = -(sh - qh).abs().sum(-1)
        sim = sim.masked_fill(mask == 0, -(R.shape[1] + 1))
        idx = sim.topk(min(topk, sim.shape[1]), dim=1)[1].sort(-1)[0]
        emb = torch.gather(seq, 1, idx.unsqueeze(-1).expand(-1, -1, seq.shape[-1]))
        emb = emb + model.pos(seq.shape[1] - idx) * 0.02
        ints.append(eager_filter(emb, model.MHFT_block[q]).mean(1))
    interests = torch.stack(ints, 1)
    long = eager_mhta(t, interests, torch.ones(x.shape[0], 3, device=x.device), mw(model.long_attention), heads)
    return t, short, long


def block_times(x, mask, model, topk, repeats):
    from fuxictr_b200 import functional as F2
    xs = x.detach().requires_grad_(True)

    def fb(fn):
        def run():
            sum(o.sum() for o in fn()[:3]).backward()
        return run
    out = {}
    eager = lambda: eager_mirrn(xs, mask, model, topk)         # noqa: E731
    fused = lambda: model.interest(xs, mask)                   # noqa: E731
    F2.set_matmul_precision("fp32")
    with torch.no_grad():
        out["eager_fp32_fwd_us"] = timed(graphed(eager), repeats)
    out["eager_fp32_fwd_bwd_us"] = timed(graphed(fb(eager)), repeats)
    for mode in MODES:
        F2.set_matmul_precision(mode)
        with torch.no_grad():
            out["kernels_%s_fwd_us" % mode] = timed(graphed(fused), repeats)
        out["kernels_%s_fwd_bwd_us" % mode] = timed(graphed(fb(fused)), repeats)
    F2.set_matmul_precision("fp32")
    return out


def kernel_times(x, mask, model, topk, repeats):
    from fuxictr_b200 import _lib, functional as F2
    B, L1, d = x.shape
    L, bits, k = L1 - 1, model.hash_bits, min(topk, L1 - 1)
    m8 = torch.ne(mask, 0).view(torch.uint8)
    p, st = F2._ptr, F2._stream
    R = model.random_rotations.detach()
    pos = torch.empty(B, 3, k, dtype=torch.int32, device="cuda")
    res = {}
    fn = lambda: _lib.call("b2_mirrn_retrieve_fwd", p(x), p(m8), p(R), 0, B, L, d, bits, k, p(pos), st())  # noqa
    nbytes = 4 * B * L1 * d + B * L + 4 * B * 3 * k
    us = timed(fn, repeats)
    res["retrieve"] = {"us": us, "TB_per_s": nbytes / (us * 1e-6) / 1e12, "bytes": nbytes}
    htab = F2.mirrn_filter_table(k).float().cuda()
    P = model.pos.weight.detach()
    cws = [b.complex_weight.detach() for b in model.MHFT_block]
    u, y = torch.empty(3, B * k, d, device="cuda"), torch.empty(3, B * k, d, device="cuda")
    fn = lambda: _lib.call("b2_mirrn_filter_fwd", p(x), p(pos), p(P), P.shape[0], *map(p, cws), p(htab), B, L, d,  # noqa
                           k, p(u), p(y), st())
    nbytes = 3 * B * k * (4 * d * 2 + 4) + 2 * 4 * 3 * B * k * d
    us = timed(fn, repeats)
    res["filter_fwd"] = {"us": us, "TB_per_s": nbytes / (us * 1e-6) / 1e12, "bytes": nbytes}
    dy, du = torch.randn_like(u), torch.empty_like(u)
    dcw = [torch.zeros_like(w) for w in cws]
    dpos = torch.zeros_like(P)
    fn = lambda: _lib.call("b2_mirrn_filter_bwd", p(dy), p(dy), p(u), p(pos), P.shape[0], *map(p, cws), p(htab), B,  # noqa
                           L, d, k, p(du), *map(p, dcw), p(dpos), st())
    nbytes = 3 * 4 * 3 * B * k * d + 4 * 3 * B * k + 4 * 3 * B * k * d + 4 * 3 * B * k * d
    us = timed(fn, repeats)
    res["filter_bwd"] = {"us": us, "TB_per_s": nbytes / (us * 1e-6) / 1e12, "bytes": nbytes}
    return res


def step_rate(fm, triple, topk, L, mode, repeats):
    from fuxictr_b200 import zoo, functional as F2
    F2.set_matmul_precision(mode)
    torch.manual_seed(1)
    model = zoo.MIRRN(fm, gpu=0, topk=topk, max_len=L, **KW)
    model.use_fused_optimizer()
    us = timed(lambda: model.fused_train_step(triple), repeats)
    F2.set_matmul_precision("fp32")
    return triple[2].shape[0] / (us * 1e-6)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=20)
    args = ap.parse_args()
    import __graft_entry__
    __graft_entry__.build()
    from fuxictr_b200 import zoo
    res = {"card": card(), "shapes": {}}
    for sname, shp in SHAPES.items():
        fm, triple = fm_and_triple(shp["batch"], shp["L"], torch.Generator().manual_seed(3))
        torch.manual_seed(1)
        model = zoo.MIRRN(fm, gpu=0, topk=shp["topk"], max_len=shp["L"], **KW)
        model.train()
        with torch.no_grad():
            _, x, mask = model._item_inputs(triple)
        x = x.contiguous()
        res["shapes"][sname] = {
            "block": block_times(x, mask, model, shp["topk"], args.repeats),
            "kernel": kernel_times(x, mask, model, shp["topk"], args.repeats),
            "step_samples_per_s": {m: step_rate(fm, triple, shp["topk"], shp["L"], m, args.repeats) for m in MODES}}
        print(json.dumps(res["shapes"][sname]), flush=True)
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()

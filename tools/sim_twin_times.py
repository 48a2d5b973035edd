"""SIM and TWIN on the GPU at two shapes: SIM_default / TWIN_default (B 8192, D 4, three item fields so d 12, L 50,
topk 50, 2 heads, attention_dim 64, DNN [64, 32]) and a long shape (B 4096, L 1024, topk 50, mean history length about
L / 2), each with one user field.

Times (CUDA events, median over the timed repeats after warm-up):
  - the interest block forward, and forward + backward: torch eager fp32 restating the reference's ops (two Linears,
    bmm, topk, gather and the target attention for SIM; the four projections of the whole history, topk, gather and
    softmax for TWIN), and functional.sim_interest / twin_interest on the kernels in fp32;
  - the whole fused_train_step in samples/s, in fp32, tf32x3, tf32 and bf16;
  - b2_sim_retrieve_fwd and b2_twin_topk_fwd alone, with TB/s from the bytes they must move: the B (L + 1) d rows, the
    mask, u or q', and the outputs (SIM: qk, pooled, the compact rows, their mask and positions; TWIN: p, stats and
    positions).
Prints one JSON object, with the card's name and power limit read in the same run.

    python tools/sim_twin_times.py [--repeats 20]
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

MODES = ("fp32", "tf32x3", "tf32", "bf16")
SHAPES = {"default": dict(batch=8192, L=50), "long": dict(batch=4096, L=1024)}
KW = dict(embedding_dim=4, dnn_hidden_units=[64, 32], attention_dim=64, num_heads=2, topk=50, short_seq_len=50)


def fm_and_triple(B, L, gen):
    from fuxictr_b200.schema import FeatureMap
    specs = [("user_id", {"type": "categorical", "source": "user", "padding_idx": 0, "vocab_size": 500}),
             ("item_id", {"type": "categorical", "source": "item", "padding_idx": 0, "vocab_size": 3000}),
             ("cate_id", {"type": "categorical", "source": "item", "padding_idx": 0, "vocab_size": 60}),
             ("brand_id", {"type": "categorical", "source": "item", "padding_idx": 0, "vocab_size": 200})]
    fm = FeatureMap.from_specs(specs, embedding_dim=4)
    lens = torch.randint(0, L + 1, (B,), generator=gen)
    hist = torch.randint(1, 3000, (B, L), generator=gen) * (torch.arange(L).view(1, -1) >= (L - lens).view(-1, 1))
    items = torch.cat([hist, torch.randint(1, 3000, (B, 1), generator=gen)], dim=1).flatten()
    idict = {"item_id": items, "cate_id": torch.where(items > 0, items % 59 + 1, torch.zeros_like(items)),
             "brand_id": torch.where(items > 0, items % 199 + 1, torch.zeros_like(items))}
    bd = {"user_id": torch.randint(1, 500, (B,), generator=gen), "label": (torch.rand(B, generator=gen) < 0.3).double()}
    return fm, ({k: v.cuda() for k, v in bd.items()}, {k: v.cuda() for k, v in idict.items()}, (hist > 0).float().cuda())


def eager_mhta(t, h, mask, W, heads):
    B = t.shape[0]
    q, k, v = t @ W[0].t(), h @ W[1].t(), h @ W[2].t()
    hd = q.shape[-1] // heads
    q = q.view(B, 1, heads, hd).transpose(1, 2)
    k = k.view(B, -1, heads, hd).transpose(1, 2)
    v = v.view(B, -1, heads, hd).transpose(1, 2)
    s = (q @ k.transpose(-1, -2)) / hd ** 0.5
    s = s.masked_fill(mask.view(B, 1, 1, -1) == 0, -1e9)
    return (torch.softmax(s, -1) @ v).transpose(1, 2).reshape(B, -1) @ W[3].t()


def eager_sim(x, mask, S, topk, heads, Wa, Wb, Ws, Wl):
    t, hist = x[:, -1], x[:, :-1]
    short = eager_mhta(t, x[:, -S:-1], mask[:, -S:-1], Ws, heads)
    qk = torch.bmm((t @ Wa.t()).unsqueeze(1), (hist @ Wb.t()).transpose(-1, -2)).squeeze(1) * mask
    pooled = torch.bmm(qk.unsqueeze(1), hist).squeeze(1)
    idx = qk.topk(min(topk, qk.shape[1]), dim=1)[1]
    emb = torch.gather(hist, 1, idx.unsqueeze(-1).expand(-1, -1, hist.shape[-1]))
    return t, short, eager_mhta(t, emb, torch.gather(mask, 1, idx), Wl, heads), pooled


def eager_twin(x, mask, S, topk, heads, Ws, Wt):
    t, hist = x[:, -1], x[:, :-1]
    B, L, _ = hist.shape
    short = eager_mhta(t, x[:, -S:-1], mask[:, -S:-1], Ws, heads)
    q, kh, v = t @ Wt[0].t(), hist @ Wt[1].t(), hist @ Wt[2].t()
    hd = q.shape[-1] // heads
    q = q.view(B, 1, heads, hd).transpose(1, 2)
    kh = kh.view(B, L, heads, hd).transpose(1, 2)
    v = v.view(B, L, heads, hd).transpose(1, 2)
    s = (q @ kh.transpose(-1, -2)) / hd ** 0.5
    s = s.masked_fill(mask.view(B, 1, 1, L) == 0, -1e9)
    ts, ti = s.topk(min(topk, L), dim=-1)
    tv = torch.gather(v, 2, ti.transpose(-1, -2).expand(-1, -1, -1, hd))
    out = (ts.softmax(-1) @ tv).transpose(1, 2).reshape(B, -1) @ Wt[3].t()
    return t, short, out


def block_times(name, x, mask, model, repeats):
    from fuxictr_b200 import functional as F2
    S, k, H = KW["short_seq_len"], KW["topk"], KW["num_heads"]
    xs = x.detach().requires_grad_(True)
    sa, la = model.short_attention, model.long_attention
    mw = lambda a: (a.W_q.weight, a.W_k.weight, a.W_v.weight, a.W_o.weight)    # noqa: E731
    if name == "SIM":
        fused = lambda: F2.sim_interest(xs, mask, S, k, H, model.W_a.weight, model.W_b.weight, mw(sa), mw(la))[:4]  # noqa
        eager = lambda: eager_sim(xs, mask, S, k, H, model.W_a.weight, model.W_b.weight, mw(sa), mw(la))  # noqa
    else:
        fused = lambda: F2.twin_interest(xs, mask, S, k, H, mw(sa), la.weights())[:3]      # noqa: E731
        eager = lambda: eager_twin(xs, mask, S, k, H, mw(sa), la.weights())                 # noqa: E731

    def fb(fn):
        def run():
            sum(o.sum() for o in fn()).backward()
        return run
    out = {}
    F2.set_matmul_precision("fp32")
    for tag, fn in (("eager", eager), ("kernels", fused)):
        with torch.no_grad():
            out[tag + "_fwd_us"] = timed(fn, repeats)
        out[tag + "_fwd_bwd_us"] = timed(fb(fn), repeats)
    return out


def kernel_times(name, x, mask, repeats):
    from fuxictr_b200 import _lib, functional as F2
    B, L1, d = x.shape
    L, k, H = L1 - 1, KW["topk"], KW["num_heads"]
    m8 = torch.ne(mask, 0).view(torch.uint8)
    p = F2._ptr
    if name == "SIM":
        u = torch.randn(B, d, device="cuda")
        qk, pooled = torch.empty(B, L, device="cuda"), torch.empty(B, d, device="cuda")
        emb = torch.empty(B, k, d, device="cuda")
        tm, pos = torch.empty(B, k, dtype=torch.uint8, device="cuda"), torch.empty(B, k, dtype=torch.int32, device="cuda")
        fn = lambda: _lib.call("b2_sim_retrieve_fwd", p(x), p(m8), p(u), B, L, d, k, p(qk), p(pooled), p(emb),  # noqa
                               p(tm), p(pos), F2._stream())
        nbytes = 4 * B * L1 * d + B * L + 4 * B * d + 4 * B * L + 4 * B * d + 4 * B * k * d + 5 * B * k
    else:
        q = torch.randn(B, H * d, device="cuda")
        pp, st = torch.empty(B, H * d, device="cuda"), torch.empty(B, H, 2, device="cuda")
        pos = torch.empty(B, H, k, dtype=torch.int32, device="cuda")
        fn = lambda: _lib.call("b2_twin_topk_fwd", p(q), p(x), p(m8), B, L, d, H, k, p(pp), p(st), p(pos),  # noqa
                               F2._stream())
        nbytes = 4 * B * L1 * d + B * L + 4 * B * H * d + 4 * B * H * d + 8 * B * H + 4 * B * H * k
    us = timed(fn, repeats)
    return {"us": us, "TB_per_s": nbytes / (us * 1e-6) / 1e12, "bytes": nbytes}


def step_rate(name, fm, triple, mode, repeats):
    from fuxictr_b200 import zoo, functional as F2
    F2.set_matmul_precision(mode)
    torch.manual_seed(1)
    model = getattr(zoo, name)(fm, gpu=0, **KW)
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
        for name in ("SIM", "TWIN"):
            torch.manual_seed(1)
            model = getattr(zoo, name)(fm, gpu=0, **KW)
            with torch.no_grad():
                _, x, mask = model._item_inputs(triple)
            x = x.contiguous()
            r = {"block": block_times(name, x, mask, model, args.repeats),
                 "kernel_fwd": kernel_times(name, x, mask, args.repeats),
                 "step_samples_per_s": {m: step_rate(name, fm, triple, m, args.repeats) for m in MODES}}
            res["shapes"]["%s_%s" % (name, sname)] = r
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()

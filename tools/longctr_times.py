"""ETA and SDIM on the GPU at three shapes: ETA_default (B 8192, D 4, L 50, topk 50, so the top-k keeps every
position), SDIM_default (B 10000, D 32, L 50, 2 hashes of 4 bits) and a long shape (ETA and SDIM at B 4096, L 1024,
topk 50, D 4), each with three item fields (item_info_dim 3 D) and one user field.

Times (CUDA events, median over the timed repeats after warm-up):
  - the interest block (short attention, retrieval or pooling, long attention for ETA) forward, and forward + backward:
    torch eager fp32 restating the reference's ops (einsum / argmax / topk / gather / target attention for ETA,
    einsum / argmax / nonzero / embedding_bag for SDIM; each call synchronised, since SDIM's nonzero waits for the
    host), and functional.eta_interest / sdim_interest on the kernels in fp32, tf32x3, tf32 and bf16;
  - the whole fused_train_step in samples/s, per mode;
  - b2_eta_retrieve_fwd and b2_sdim_pool_fwd alone, with bytes/s from the bytes they must move: the B L d history and
    the target, the mask, the rotations, and the compact output (ETA: topk rows, mask and positions; SDIM: the pooled
    row, the per-hash sums and the collision words);
  - at the long shape, the share of the fp32 step taken by the embedding gather and its backward scatter (torch.profiler
    kernel time of those kernels over the step's kernel time), and the step's heaviest kernels.
Prints one JSON object, with the card's name and power limit read in the same run.

    python tools/longctr_times.py [--repeats 20]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

MODES = ("fp32", "tf32x3", "tf32", "bf16")
SHAPES = {
    "ETA_default": dict(model="ETA", batch=8192, dim=4, L=50, kw=dict(attention_dim=64, num_heads=2, hash_bits=32,
                                                                        topk=50, short_seq_len=50)),
    "SDIM_default": dict(model="SDIM", batch=10000, dim=32, L=50, kw=dict(attention_dim=64, num_heads=2, num_hashes=2,
                                                                           hash_bits=4, short_seq_len=50)),
    "ETA_long": dict(model="ETA", batch=4096, dim=4, L=1024, kw=dict(attention_dim=64, num_heads=2, hash_bits=32,
                                                                       topk=50, short_seq_len=50)),
    "SDIM_long": dict(model="SDIM", batch=4096, dim=4, L=1024, kw=dict(attention_dim=64, num_heads=2, num_hashes=2,
                                                                        hash_bits=4, short_seq_len=50)),
}


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in out.split(",")]
        return {"name": name, "power_limit": power}
    except Exception as e:      # noqa: BLE001  the numbers stay; the card is reported unknown
        return {"name": "unknown (%s)" % e}


def timed(fn, repeats, warmup=3):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(repeats):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b) * 1000.0)
    ts.sort()
    return ts[len(ts) // 2]


def feature_map(dim):
    from fuxictr_b200.schema import FeatureMap
    specs = [("user_id", {"type": "categorical", "source": "user", "padding_idx": 0, "vocab_size": 100000}),
             ("item_id", {"type": "categorical", "source": "item", "padding_idx": 0, "vocab_size": 500000}),
             ("cate_id", {"type": "categorical", "source": "item", "padding_idx": 0, "vocab_size": 5000}),
             ("brand_id", {"type": "categorical", "source": "item", "padding_idx": 0, "vocab_size": 50000})]
    return FeatureMap.from_specs(specs, embedding_dim=dim)


def triple(B, L, gen):
    lens = torch.randint(0, L + 1, (B, 1), generator=gen)
    hist = torch.randint(1, 500000, (B, L), generator=gen) * (torch.arange(L).view(1, -1) >= L - lens)
    items = torch.cat([hist, torch.randint(1, 500000, (B, 1), generator=gen)], dim=1).flatten()
    idict = {"item_id": items, "cate_id": torch.where(items > 0, items % 4999 + 1, torch.zeros_like(items)),
             "brand_id": torch.where(items > 0, items % 49999 + 1, torch.zeros_like(items))}
    bd = {"user_id": torch.randint(1, 100000, (B,), generator=gen),
          "label": (torch.rand(B, generator=gen) < 0.3).double()}
    return ({k: v.cuda() for k, v in bd.items()}, {k: v.cuda() for k, v in idict.items()}, (hist > 0).float().cuda())


def eager_mhta(att, t, h, mask):
    """MultiHeadTargetAttention.forward with ScaledDotProductAttention, in torch eager."""
    B = t.shape[0]
    q = (t @ att.W_q.weight.t()).view(B, 1, att.num_heads, att.head_dim).transpose(1, 2)
    k = (h @ att.W_k.weight.t()).view(B, -1, att.num_heads, att.head_dim).transpose(1, 2)
    v = (h @ att.W_v.weight.t()).view(B, -1, att.num_heads, att.head_dim).transpose(1, 2)
    s = (q @ k.transpose(-1, -2)) / att.scale
    s = s.masked_fill(mask.view(B, 1, 1, -1).float() == 0, -1e9)
    out = (s.softmax(dim=-1) @ v).transpose(1, 2).reshape(B, -1)
    return out @ att.W_o.weight.t()


def eager_block(name, model, x, mask):
    """The reference's interest block restated in torch eager fp32 (ETA.py topk_retrieval / lsh_hash, SDIM.py
    lsh_attentioin / lsh_hash, target_attention.py MultiHeadTargetAttention)."""
    s = model.short_seq_len
    target = x[:, -1]
    short = eager_mhta(model.short_attention, target, x[:, -s:-1], mask[:, -s:-1])
    hist = x[:, :-1]
    R = model.random_rotations.repeat(x.size(0), *([1] * (model.random_rotations.dim() - 1)))
    if name == "ETA":
        def lsh(v):
            r = torch.einsum("bld,bdh->blh", v, R).unsqueeze(-1)
            return torch.argmax(torch.cat([-r, r], dim=-1), dim=-1).float()
        dis = torch.abs(lsh(hist) - lsh(target.unsqueeze(1))).sum(dim=-1)
        dis = dis.masked_fill_(mask.float() == 0, 1 + model.hash_bits)
        idx = dis.topk(min(model.topk, dis.shape[1]), dim=1, largest=False, sorted=True)[1]
        emb = torch.gather(hist, 1, idx.unsqueeze(-1).expand(-1, -1, hist.shape[-1]))
        long = eager_mhta(model.long_attention, target, emb, torch.gather(mask, 1, idx))
    else:
        def lsh(v):
            r = torch.einsum("bld,bdht->blht", v, R).unsqueeze(-1)
            code = torch.argmax(torch.cat([-r, r], dim=-1), dim=-1).float()
            return torch.matmul(code, model.powers_of_two.unsqueeze(-1)).squeeze(-1)
        sb = lsh(hist)
        tb = lsh(target.unsqueeze(1)).repeat(1, sb.shape[1], 1)
        cm = ((sb == tb) * mask.unsqueeze(-1)).float().permute(2, 0, 1)
        _, ci = torch.nonzero(cm.flatten(start_dim=1), as_tuple=True)
        off = cm.sum(dim=-1).flatten().cumsum(dim=0)
        off = torch.cat([torch.zeros(1, device=off.device), off]).long()
        out = torch.nn.functional.embedding_bag(ci, hist.reshape(-1, x.size(-1)), off, mode="sum",
                                                include_last_offset=True)
        long = out.view(model.num_hashes, -1, x.size(-1)).mean(dim=0)
    return target, short, long


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("longctr_times.py measures on the GPU; no CUDA device found")
    import __graft_entry__
    __graft_entry__.build()
    from fuxictr_b200 import zoo, functional as F2, _lib
    res = {"card": card()}
    for shape, cfg in SHAPES.items():
        name, B, D, L = cfg["model"], cfg["batch"], cfg["dim"], cfg["L"]
        fm = feature_map(D)
        gen = torch.Generator().manual_seed(1)
        batch = triple(B, L, gen)

        def build():
            torch.manual_seed(0)
            m = getattr(zoo, name)(fm, gpu=0, embedding_dim=D, dnn_hidden_units=[64, 32], **cfg["kw"])
            with torch.no_grad():
                for mod in m.modules():
                    if isinstance(mod, torch.nn.Embedding):
                        mod.weight[1:].normal_(0, 0.1)
            m.train()
            return m

        model = build()
        d = model.item_info_dim
        mask = batch[2]
        x = (torch.randn(B, L + 1, d, device="cuda") * 0.3)
        x[:, :L] *= mask.unsqueeze(-1)
        x.requires_grad_(True)
        gout = [torch.randn(B, d, device="cuda") for _ in range(3)]
        out = {"batch": B, "L": L, "item_info_dim": d, "mean_history_length": float(mask.sum(1).mean())}

        def eager_fwd():
            with torch.no_grad():
                eager_block(name, model, x, mask)
            torch.cuda.synchronize()

        def eager_fb():
            o = eager_block(name, model, x, mask)
            sum((a * g).sum() for a, g in zip(o, gout)).backward()
            torch.cuda.synchronize()

        out["block_fwd_us"] = {"torch_eager_fp32": timed(eager_fwd, args.repeats)}
        out["block_fwd_bwd_us"] = {"torch_eager_fp32": timed(eager_fb, args.repeats)}
        for mode in MODES:
            F2.set_matmul_precision(mode)

            def fwd():
                with torch.no_grad():
                    model.interest(x, mask)

            def fb():
                o = model.interest(x, mask)
                sum((a * g).sum() for a, g in zip(o, gout)).backward()
            out["block_fwd_us"][mode] = timed(fwd, args.repeats)
            out["block_fwd_bwd_us"][mode] = timed(fb, args.repeats)
        F2.set_matmul_precision("fp32")
        for key in ("block_fwd_us", "block_fwd_bwd_us"):
            base = out[key]["torch_eager_fp32"]
            out[key.replace("_us", "_speedup_vs_eager")] = {k: base / v for k, v in out[key].items()
                                                             if k != "torch_eager_fp32"}

        out["fused_train_step_samples_per_s"] = {}
        for mode in MODES:
            F2.set_matmul_precision(mode)
            m = build()
            m.use_fused_optimizer()
            us = timed(lambda: m.fused_train_step(batch), args.repeats)
            out["fused_train_step_samples_per_s"][mode] = B / (us * 1e-6)
        F2.set_matmul_precision("fp32")

        xs = x.detach().contiguous()
        m8 = torch.ne(mask, 0).view(torch.uint8)
        p = F2._ptr
        R = model.random_rotations.detach()
        if name == "ETA":
            k = min(model.topk, L)
            te = torch.empty(B, k, d, device="cuda")
            tm = torch.empty(B, k, dtype=torch.uint8, device="cuda")
            tp = torch.empty(B, k, dtype=torch.int32, device="cuda")

            def kern():
                _lib.call("b2_eta_retrieve_fwd", p(xs), p(m8), p(R), 0, B, L, d, model.hash_bits, k, p(te), p(tm),
                          p(tp), F2._stream())
            nbytes = B * (L + 1) * d * 4 + B * L + R.numel() * 4 + B * k * (d * 4 + 1 + 4)
        else:
            nh = model.num_hashes
            o1 = torch.empty(B, d, device="cuda")
            sm = torch.empty(B, nh, d, device="cuda")
            cw = torch.empty(B, L, dtype=torch.int32, device="cuda")

            def kern():
                _lib.call("b2_sdim_pool_fwd", p(xs), p(m8), p(R), 0, B, L, d, nh, model.hash_bits, 0, p(o1), p(sm),
                          p(cw), F2._stream())
            nbytes = B * (L + 1) * d * 4 + B * L + R.numel() * 4 + B * d * 4 + B * nh * d * 4 + B * L * 4
        t = timed(kern, args.repeats * 5)
        out["kernel"] = {"us": t, "bytes": nbytes, "TBps": nbytes / (t * 1e-6) / 1e12}

        if L > 50:      # the item gather's share of the step, for a later fused gather-and-retrieve
            from torch.profiler import profile, ProfilerActivity
            m = build()
            m.use_fused_optimizer()
            for _ in range(3):
                m.fused_train_step(batch)
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(5):
                    m.fused_train_step(batch)
                torch.cuda.synchronize()
            total, gather, names = 0.0, 0.0, {}
            for ev in prof.key_averages():
                t_dev = getattr(ev, "device_time_total", getattr(ev, "cuda_time_total", 0.0))
                if ev.key.startswith(("cuda", "Memcpy", "Memset")) and "Kernel" not in ev.key:
                    continue
                total += t_dev
                names[ev.key] = t_dev
                if any(w in ev.key.lower() for w in ("embed", "gather", "scatter", "front")):
                    gather += t_dev
            out["step_kernel_share"] = {"embedding_gather_and_backward": gather / total if total else None,
                                        "top_kernels_us_per_step": dict(sorted(((k, v / 5) for k, v in names.items()),
                                                                               key=lambda kv: -kv[1])[:8])}
        res[shape] = out
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()

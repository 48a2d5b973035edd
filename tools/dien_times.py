"""DIEN at DIEN_default's shape on the GPU: B 10000, D 16, adgroup_id / click_sequence with max_len 50 (H 16), three
categorical fields, AUGRU with bilinear attention and softmax, DNN [1024, 512, 256] with Dice and batch norm.

Times (CUDA events, median over the timed repeats after warm-up):
  - the interest stack (extractor GRU, attention, evolution AUGRU) forward, and forward + backward: torch eager fp32
    restating the reference's arithmetic (pack_padded_sequence + nn.GRU for the extractor, the per-step AUGRU loop
    for the evolution, with its host-side lengths; each call synchronised, since that path cannot be captured), and
    zoo.DIEN.interest on the kernels in fp32, tf32x3, tf32 and bf16;
  - the whole fused_train_step (embedding lookup, forward, backward, clip + Adam) in samples/s, per mode;
  - the recurrence kernels alone (b2_gru_fwd / _bwd, AUGRU) and their achieved bytes/s from the bytes they must move:
    forward reads x (B L H), the mask and the attention and writes h_seq and h_last; backward reads x, h_seq, dh_seq,
    the mask and the attention and writes dx and da.
Prints one JSON object, with the card's name and power limit read in the same run.

    python tools/dien_times.py [--batch 10000] [--repeats 20]
"""
import argparse
import json
import os
import subprocess
import sys

import torch
from torch.nn.utils.rnn import pack_padded_sequence, pad_packed_sequence

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


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


def feature_map(max_len, dim, n_cat):
    from fuxictr_b200.schema import FeatureMap
    specs = [("C%d" % i, {"type": "categorical", "source": "", "padding_idx": 0, "vocab_size": 1000 + i})
             for i in range(n_cat)]
    specs += [("adgroup_id", {"type": "categorical", "source": "", "padding_idx": 0, "vocab_size": 100000}),
              ("click_sequence", {"type": "sequence", "source": "", "padding_idx": 0, "vocab_size": 100000,
                                  "max_len": max_len, "share_embedding": "adgroup_id", "feature_encoder": None})]
    return FeatureMap.from_specs(specs, embedding_dim=dim)


def eager_stack(model, seq, tgt, mask):
    """The reference's interest_extraction, AttentionLayer and interest_evolution (DynamicGRU's loop over the packed
    time steps) in torch eager fp32, rows with an empty history dropped and put back."""
    ext, att = model.extraction_modules[0], model.attention_modules[0]
    cell = model.evolving_modules[0].gru_cell
    nz = mask.sum(dim=1) > 0
    seq, tgt, mask = seq[nz], tgt[nz], mask[nz]
    lens = mask.sum(dim=1).cpu()
    packed, _ = ext(pack_padded_sequence(seq, lens, batch_first=True, enforce_sorted=False))
    interest, _ = pad_packed_sequence(packed, batch_first=True, padding_value=0.0, total_length=mask.size(1))
    m = mask.float()
    s = ((interest @ att.W_kernel) @ tgt.unsqueeze(-1)).view(-1, mask.size(1)) * m
    s = (s + -1.e9 * (1 - m)).softmax(dim=-1)
    ps = pack_padded_sequence(s, lens, batch_first=True, enforce_sorted=False)
    x, batch_sizes, _, unsorted = packed
    a = ps.data
    h = torch.zeros(int(batch_sizes[0]), cell.h2h.in_features, device=seq.device)
    out_h = torch.zeros_like(h)
    start = 0
    for bs in batch_sizes.tolist():
        gx, gh = cell.x2h(x[start:start + bs]), cell.h2h(h[:bs])
        i_u, i_r, i_n = gx.chunk(3, 1)
        h_u, h_r, h_n = gh.chunk(3, 1)
        u = torch.sigmoid(i_u + h_u) * a[start:start + bs].unsqueeze(-1)
        r = torch.sigmoid(i_r + h_r)
        n = torch.tanh(i_n + r * h_n)
        h = h[:bs] + u * (n - h[:bs])
        out_h[:bs] = h
        start += bs
    full = torch.zeros(nz.shape[0], h.shape[1], device=seq.device)
    full[nz] = out_h[unsorted]
    return full


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=10000)
    ap.add_argument("--repeats", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("dien_times.py measures on the GPU; no CUDA device found")
    import __graft_entry__
    __graft_entry__.build()
    from fuxictr_b200 import zoo, functional as F2, _lib
    B, D, max_len = args.batch, 16, 50
    fm = feature_map(max_len, D, 3)
    res = {"card": card(), "batch": B, "embedding_dim": D, "max_len": max_len}

    def build():
        torch.manual_seed(0)
        m = zoo.DIEN(fm, gpu=0, embedding_dim=D, dnn_hidden_units=[1024, 512, 256], dnn_activations="Dice",
                     batch_norm=True, dien_target_field="adgroup_id", dien_sequence_field="click_sequence",
                     dien_neg_seq_field=[], gru_type="AUGRU", attention_type="bilinear_attention")
        with torch.no_grad():
            for mod in m.modules():
                if isinstance(mod, torch.nn.Embedding):
                    mod.weight[1:].normal_(0, 0.1)
        m.train()
        return m

    gen = torch.Generator().manual_seed(1)
    cols = [torch.randint(0, fm.features["C%d" % i]["vocab_size"], (B, 1), generator=gen).double() for i in range(3)]
    cols.append(torch.randint(1, 100000, (B, 1), generator=gen).double())
    ids = torch.randint(1, 100000, (B, max_len), generator=gen)
    lens = torch.randint(0, max_len + 1, (B, 1), generator=gen)
    ids = ids * (torch.arange(max_len).view(1, -1) < lens)
    mat = torch.cat(cols + [ids.double(), (torch.rand(B, 1, generator=gen) < 0.3).double()], dim=1).cuda()
    batch = fm.batch_dict(mat)
    res["mean_history_length"] = float(lens.float().mean())

    model = build()
    H = D
    seq = (torch.randn(B, max_len, H, device="cuda") * 0.3 * (ids != 0).unsqueeze(-1).cuda()).requires_grad_(True)
    tgt = (torch.randn(B, H, device="cuda") * 0.3).requires_grad_(True)
    mask_b = (ids != 0).cuda()
    mask = mask_b.to(torch.uint8).contiguous()
    gout = torch.randn(B, H, device="cuda")

    def eager_fwd():
        with torch.no_grad():
            eager_stack(model, seq, tgt, mask_b)

    def eager_fb():
        (eager_stack(model, seq, tgt, mask_b) * gout).sum().backward()

    res["stack_fwd_us"] = {"torch_eager_fp32": timed(eager_fwd, args.repeats)}
    res["stack_fwd_bwd_us"] = {"torch_eager_fp32": timed(eager_fb, args.repeats)}
    for mode in ("fp32", "tf32x3", "tf32", "bf16"):
        F2.set_matmul_precision(mode)

        def fwd():
            with torch.no_grad():
                model.interest(0, seq, tgt, mask)

        def fb():
            (model.interest(0, seq, tgt, mask) * gout).sum().backward()
        res["stack_fwd_us"][mode] = timed(fwd, args.repeats)
        res["stack_fwd_bwd_us"][mode] = timed(fb, args.repeats)
    F2.set_matmul_precision("fp32")
    for key in ("stack_fwd_us", "stack_fwd_bwd_us"):
        base = res[key]["torch_eager_fp32"]
        res[key.replace("_us", "_speedup_vs_eager")] = {k: base / v for k, v in res[key].items()
                                                          if k != "torch_eager_fp32"}

    res["fused_train_step_samples_per_s"] = {}
    for mode in ("fp32", "tf32x3", "tf32", "bf16"):
        F2.set_matmul_precision(mode)
        m = build()
        m.use_fused_optimizer()
        us = timed(lambda: m.fused_train_step(batch), args.repeats)
        res["fused_train_step_samples_per_s"][mode] = B / (us * 1e-6)
    F2.set_matmul_precision("fp32")

    L = max_len
    cellm = model.evolving_modules[0].gru_cell
    x = seq.detach().contiguous()
    a = torch.rand(B, L, device="cuda")
    hs = torch.empty(B, L, H, device="cuda")
    hl = torch.empty(B, H, device="cuda")
    dhs = torch.randn_like(hs)
    dx = torch.empty_like(hs)
    da = torch.empty_like(a)
    gW = [torch.zeros_like(p) for p in (cellm.x2h.weight, cellm.x2h.bias, cellm.h2h.weight, cellm.h2h.bias)]
    p = F2._ptr
    w = (p(cellm.x2h.weight), p(cellm.x2h.bias), p(cellm.h2h.weight), p(cellm.h2h.bias))

    def kfwd():
        _lib.call("b2_gru_fwd", p(x), L * H, p(mask), *w, p(a), _lib.B2_DIEN_AUGRU, B, L, H, p(hs), p(hl),
                  F2._stream())

    def kbwd():
        _lib.call("b2_gru_bwd", p(x), L * H, p(mask), *w, p(a), _lib.B2_DIEN_AUGRU, B, L, H, p(hs), p(dhs), None,
                  p(dx), 0, p(da), p(gW[0]), p(gW[1]), p(gW[2]), p(gW[3]), F2._stream())
    kfwd()
    t_f, t_b = timed(kfwd, args.repeats * 5), timed(kbwd, args.repeats * 5)
    bytes_f = B * L * H * 4 * 2 + B * L * (1 + 4) + B * H * 4
    bytes_b = B * L * H * 4 * 4 + B * L * (1 + 4 + 4)
    res["recurrence_kernels"] = {"fwd_us": t_f, "fwd_TBps": bytes_f / (t_f * 1e-6) / 1e12,
                                 "bwd_us": t_b, "bwd_TBps": bytes_b / (t_b * 1e-6) / 1e12,
                                 "fwd_bytes": bytes_f, "bwd_bytes": bytes_b}
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()

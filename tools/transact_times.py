"""TransAct at TransAct_default's shape on the GPU: B 10000, D 64, one head, one layer, FFN 512, three cross layers,
DCN [1024, 512, 256], target adgroup_id, sequence click_sequence (model_dim 128, head width 128), six categorical
fields, left-padded histories of random length; at max_len 50 and at max_len 100.

Times (CUDA events around CUDA-graph replays, median over the timed repeats after warm-up):
  - the sequence block (tokens, encoder, zeroing, last slot and out_linear(max over L)) forward and forward + backward:
    torch eager fp32 with the reference's own modules (the block's nn.TransformerEncoder and out_linear, called as
    TransActTransformer.forward calls them), and TransActTransformer.run on the kernels in fp32, tf32x3, tf32 and bf16;
  - the whole fused_train_step (embedding lookup, forward, backward, clip + Adam) per mode, in samples/s;
  - the attention kernels alone (b2_transact_attn_fwd / _bwd) and their FLOP/s from the shapes: 4 L^2 md per sample
    forward (q k^T and p v), 10 L^2 md backward (the scores recomputed, dp, dq, dk, dv), padded rows counted.
Prints one JSON object, with the card's name and power limit read in the same run.

    python tools/transact_times.py [--batch 10000] [--repeats 20]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

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


def graphed(fn, warmup=3):
    """fn captured into a CUDA graph after warm-up on a side stream; returns the replay."""
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(warmup):
            fn()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fn()
    return g.replay


def feature_map(max_len, dim, n_cat):
    from fuxictr_b200.schema import FeatureMap
    specs = [("C%d" % i, {"type": "categorical", "source": "", "padding_idx": 0, "vocab_size": 1000 + i})
             for i in range(n_cat)]
    specs += [("adgroup_id", {"type": "categorical", "source": "", "padding_idx": 0, "vocab_size": 100000}),
              ("click_sequence", {"type": "sequence", "source": "", "padding_idx": 0, "vocab_size": 100000,
                                  "max_len": max_len, "share_embedding": "adgroup_id", "feature_encoder": None})]
    return FeatureMap.from_specs(specs, embedding_dim=dim)


def matrix(fm, B, gen):
    cols = []
    for _, spec in fm.features.items():
        if spec["type"] == "sequence":
            L_ = spec["max_len"]
            ids = torch.randint(1, spec["vocab_size"], (B, L_), generator=gen)
            lens = torch.randint(0, L_ + 1, (B, 1), generator=gen)
            cols.append((ids * (torch.arange(L_).view(1, -1) >= L_ - lens)).double())
        else:
            cols.append(torch.randint(0, spec["vocab_size"], (B, 1), generator=gen).double())
    cols.append((torch.rand(B, 1, generator=gen) < 0.3).double())
    return torch.cat(cols, dim=1)


def eager_block(enc, seq, tgt, ids):
    """TransActTransformer.forward's arithmetic with the block's own torch modules, eager fp32."""
    L = seq.shape[1]
    x = torch.cat([seq, tgt.unsqueeze(1).expand(-1, L, -1)], dim=-1)
    mask = ids == 0
    mask = mask.clone()
    mask[:, -1] &= ~mask.all(dim=-1)
    y = enc.transformer_encoder(src=x, src_key_padding_mask=mask)
    y = y.masked_fill(mask.unsqueeze(-1), 0.0)
    last = y[:, -enc.first_k_cols:].flatten(start_dim=1)
    pooled = enc.out_linear(y.masked_fill(mask.unsqueeze(-1), -1e9).max(dim=1).values)
    return torch.cat([last, pooled], dim=-1)


def one_shape(args, max_len):
    from fuxictr_b200 import zoo, functional as F2, _lib
    from fuxictr_b200.pipeline import TrainPipeline
    B, D, H = args.batch, 64, 1
    fm = feature_map(max_len, D, 6)
    mat = matrix(fm, B, torch.Generator().manual_seed(1)).cuda()
    batch = fm.batch_dict(mat)
    res = {"shape": {"batch": B, "max_len": max_len, "embedding_dim": D, "num_heads": H, "model_dim": 2 * D,
                     "dim_feedforward": 512, "dcn_cross_layers": 3, "dcn": [1024, 512, 256],
                     "valid_slot_fraction": float((batch["click_sequence"] != 0).float().mean())}}

    def build():
        torch.manual_seed(0)
        return zoo.TransAct(fm, gpu=0, embedding_dim=D, num_heads=H, dcn_hidden_units=[1024, 512, 256],
                            mlp_hidden_units=[], dim_feedforward=512, dcn_cross_layers=3,
                            target_item_field="adgroup_id", sequence_item_field="click_sequence")
    model = build()
    model.train()
    enc = model.transformer_encoders[0]
    X = model.get_inputs(batch)
    ids = X["click_sequence"]
    emb = model.embedding_layer(X)
    seq = emb["click_sequence"].detach().clone().requires_grad_(True)
    tgt = emb["adgroup_id"].detach().clone().requires_grad_(True)
    gout = torch.randn(B, 2 * 2 * D, device="cuda")
    ids_long = ids.long()

    fwd_us, fb_us = {}, {}
    F2.set_matmul_precision("fp32")
    with torch.no_grad():
        fwd_us["torch_eager_fp32"] = timed(graphed(lambda: eager_block(enc, seq, tgt, ids_long)), args.repeats)
    fb_us["torch_eager_fp32"] = timed(graphed(lambda: eager_block(enc, seq, tgt, ids_long).backward(gout)),
                                      args.repeats)
    for mode in ("fp32", "tf32x3", "tf32", "bf16"):
        F2.set_matmul_precision(mode)
        with torch.no_grad():
            fwd_us["kernels_" + mode] = timed(graphed(lambda: enc.run([seq], [tgt], ids)), args.repeats)
        fb_us["kernels_" + mode] = timed(graphed(lambda: enc.run([seq], [tgt], ids).backward(gout)), args.repeats)
    F2.set_matmul_precision("fp32")
    res["block_fwd_us"], res["block_fwd_bwd_us"] = fwd_us, fb_us
    res["block_speedup_vs_eager"] = {
        "fwd": {k: fwd_us["torch_eager_fp32"] / v for k, v in fwd_us.items() if k != "torch_eager_fp32"},
        "fwd_bwd": {k: fb_us["torch_eager_fp32"] / v for k, v in fb_us.items() if k != "torch_eager_fp32"}}

    res["fused_train_step_samples_per_s"] = {}
    for mode in ("fp32", "tf32x3", "tf32", "bf16"):
        F2.set_matmul_precision(mode)
        m = build()
        m.train()
        m.use_fused_optimizer()
        pipe = TrainPipeline(m, mat.shape[0], mat.shape[1], graph=True)
        pipe.prime(mat)
        pipe.capture(warmup=3)
        us = timed(lambda: pipe.step_device(mat), args.repeats)
        res["fused_train_step_samples_per_s"][mode] = B / (us * 1e-6)
        del pipe, m
    F2.set_matmul_precision("fp32")

    L, md = max_len, 2 * D
    gen = torch.Generator(device="cuda").manual_seed(2)
    qkv = torch.randn(B * L, 3 * md, device="cuda", generator=gen)
    _, valid = F2.transact_tokens([seq.detach()], [tgt.detach()], ids)
    ctx = torch.empty(B * L, md, device="cuda")
    smax = torch.empty(B, H, L, device="cuda")
    ssum = torch.empty_like(smax)
    delta = torch.empty_like(smax)
    dctx = torch.randn(B * L, md, device="cuda", generator=gen)
    dqkv = torch.empty_like(qkv)
    scale = (md // H) ** -0.5
    p = F2._ptr

    def fwd():
        _lib.call("b2_transact_attn_fwd", p(qkv), p(valid), B, L, md, H, scale, None, 0, 0, 0.0, p(ctx), None, 0, 0,
                  p(smax), p(ssum), F2._stream())

    def bwd():
        _lib.call("b2_transact_attn_bwd", p(qkv), p(valid), p(ctx), p(dctx), p(smax), p(ssum), B, L, md, H, scale,
                  None, 0, 0, 0.0, p(delta), p(dqkv), None, 0, 0, F2._stream())
    fwd()
    t_f, t_b = timed(graphed(fwd), args.repeats * 5), timed(graphed(bwd), args.repeats * 5)
    flop_f, flop_b = 4.0 * B * L * L * md, 10.0 * B * L * L * md
    res["attention_kernels"] = {"fwd_us": t_f, "fwd_TFLOPs": flop_f / (t_f * 1e-6) / 1e12,
                                "bwd_us": t_b, "bwd_TFLOPs": flop_b / (t_b * 1e-6) / 1e12}
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=10000)
    ap.add_argument("--repeats", type=int, default=20)
    ap.add_argument("--max-lens", default="50,100")
    args = ap.parse_args()
    import __graft_entry__
    __graft_entry__.build()
    assert torch.cuda.is_available(), "needs a GPU"
    res = {"card": card()}
    for max_len in [int(v) for v in args.max_lens.split(",")]:
        res["max_len_%d" % max_len] = one_shape(args, max_len)
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()

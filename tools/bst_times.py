"""BST at BST_default's shape on the GPU: B 10000, D 16, 4 heads, one block, max_len 50 (L 51, model_dim 32), six
categorical fields, DNN [1024, 512, 256].

Times (CUDA events, median over the timed repeats after warm-up):
  - dense forward + backward from the embeddings to the loss: torch eager fp32 (the reference's arithmetic restated
    with nn.MultiheadAttention, LayerNorm and the MLP), and zoo.BST's dnn_input + DNN + BCE on the kernels in fp32,
    tf32x3, tf32 and bf16;
  - the whole fused_train_step (embedding lookup, forward, backward, clip + Adam) in samples/s, per mode;
  - the attention row kernels alone (b2_bst_attn_fwd / _bwd) and their achieved bytes/s from the bytes they must move:
    forward reads QKV (B L 3 md) and writes ctx and the statistics; backward reads QKV, ctx, dctx and the statistics
    and writes dQKV.
Prints one JSON object, with the card's name and power limit read in the same run.

    python tools/bst_times.py [--batch 10000] [--repeats 20]
"""
import argparse
import json
import os
import subprocess
import sys

import torch
import torch.nn.functional as TF

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


def matrix(fm, B, gen):
    cols = []
    for _, spec in fm.features.items():
        if spec["type"] == "sequence":
            L_ = spec["max_len"]
            ids = torch.randint(1, spec["vocab_size"], (B, L_), generator=gen)
            lens = torch.randint(0, L_ + 1, (B, 1), generator=gen)
            cols.append((ids * (torch.arange(L_).view(1, -1) < lens)).double())
        else:
            cols.append(torch.randint(0, spec["vocab_size"], (B, 1), generator=gen).double())
    cols.append((torch.rand(B, 1, generator=gen) < 0.3).double())
    return torch.cat(cols, dim=1)


def eager_dense(model, emb, ids, y):
    """The reference's dense arithmetic from the embedding dict to the loss, in torch eager fp32."""
    enc = model.transformer_encoders[0]
    blk = enc.transformer_blocks[0]
    seq, tgt = emb["click_sequence"], emb["adgroup_id"]
    x = torch.cat([seq, tgt.unsqueeze(1)], dim=1)
    B = x.shape[0]
    x = torch.cat([x, enc.position_emb.unsqueeze(0).expand(B, -1, -1)], dim=-1)
    pad = torch.cat([ids == 0, torch.zeros(B, 1, dtype=torch.bool, device=ids.device)], dim=1)
    L = pad.shape[1]
    mask = pad.unsqueeze(1).expand(B, L, L) & ~torch.eye(L, dtype=torch.bool, device=ids.device)
    mask = mask.repeat_interleave(blk.attention.num_heads, dim=0)
    attn, _ = blk.attention(x, x, x, attn_mask=mask)
    s = blk.layer_norm1(attn + x)
    out = blk.layer_norm2(blk.ffn(s) + s)
    w = torch.cat([(~pad).float()], dim=1).unsqueeze(-1)
    pooled = (out * w).sum(1) / (w.sum(1) + 1e-12)
    x = torch.cat([v for k, v in emb.items() if k != "click_sequence"] + [pooled], dim=-1)
    for m in list(model.dnn.mlp)[:-1]:        # nn.Linear / nn.ReLU modules, eager; the Sigmoid is in the loss
        x = m(x)
    logit = x
    return TF.binary_cross_entropy_with_logits(logit, y)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=10000)
    ap.add_argument("--repeats", type=int, default=20)
    args = ap.parse_args()
    import __graft_entry__
    __graft_entry__.build()
    from fuxictr_b200 import zoo, functional as F2, _lib
    assert torch.cuda.is_available(), "needs a GPU"
    B, max_len, D, H = args.batch, 50, 16, 4
    fm = feature_map(max_len, D, 6)
    torch.manual_seed(0)
    mat = matrix(fm, B, torch.Generator().manual_seed(1)).cuda()
    batch = fm.batch_dict(mat)
    res = {"card": card(), "shape": {"batch": B, "max_len": max_len, "embedding_dim": D, "num_heads": H,
                                     "model_dim": 32, "dnn": [1024, 512, 256]}}

    def build():
        torch.manual_seed(0)
        return zoo.BST(fm, gpu=0, embedding_dim=D, num_heads=H, dnn_hidden_units=[1024, 512, 256],
                       bst_target_field="adgroup_id", bst_sequence_field="click_sequence")
    model = build()
    model.train()
    X = model.get_inputs(batch)
    y = model.get_labels(batch)
    ids = X["click_sequence"].long()
    emb = {k: v.detach().requires_grad_(True) for k, v in model.embedding_layer(X).items()}

    def eager():
        eager_dense(model, emb, ids, y).backward()
    F2.set_matmul_precision("fp32")
    res["dense_fwd_bwd_us"] = {"torch_eager_fp32": timed(eager, args.repeats)}

    class _Emb(torch.nn.Module):      # the kernels' dense path on the same fixed embeddings
        def forward(self, inputs):
            return dict(emb)
    orig = model.embedding_layer
    for mode in ("fp32", "tf32x3", "tf32", "bf16"):
        F2.set_matmul_precision(mode)
        model.embedding_layer = _Emb()

        def kernels():
            loss, _ = F2.logit_bce(y, model.forward_logits(batch)[0])
            loss.backward()
        res["dense_fwd_bwd_us"]["kernels_" + mode] = timed(kernels, args.repeats)
        model.embedding_layer = orig
    F2.set_matmul_precision("fp32")
    base = res["dense_fwd_bwd_us"]["torch_eager_fp32"]
    res["dense_speedup_vs_eager"] = {k: base / v for k, v in res["dense_fwd_bwd_us"].items() if k != "torch_eager_fp32"}

    res["fused_train_step_samples_per_s"] = {}
    for mode in ("fp32", "tf32x3", "tf32", "bf16"):
        F2.set_matmul_precision(mode)
        m = build()
        m.use_fused_optimizer()
        us = timed(lambda: m.fused_train_step(batch), args.repeats)
        res["fused_train_step_samples_per_s"][mode] = B / (us * 1e-6)
    F2.set_matmul_precision("fp32")

    L, md = max_len + 1, 32
    qkv = torch.randn(B * L, 3 * md, device="cuda")
    valid = (ids != 0).to(torch.uint8).contiguous()
    ctx = torch.empty(B * L, md, device="cuda")
    smax = torch.empty(B, H, L, device="cuda")
    ssum = torch.empty_like(smax)
    dctx = torch.randn_like(ctx)
    dqkv = torch.empty_like(qkv)
    scale = (md // H) ** -0.5
    p = F2._ptr

    def fwd():
        _lib.call("b2_bst_attn_fwd", p(qkv), p(valid), B, L, md, H, 0, scale, None, 0, 0, 0.0, p(ctx), None, 0, 0,
                  p(smax), p(ssum), F2._stream())

    def bwd():
        _lib.call("b2_bst_attn_bwd", p(qkv), p(valid), p(ctx), p(dctx), p(smax), p(ssum), B, L, md, H, 0, scale, None,
                  0, 0, 0.0, p(dqkv), None, 0, 0, F2._stream())
    fwd()
    t_f, t_b = timed(fwd, args.repeats * 5), timed(bwd, args.repeats * 5)
    stats = 2 * B * H * L * 4
    bytes_f = B * L * 3 * md * 4 + B * L * md * 4 + stats + B * (L - 1)
    bytes_b = 2 * B * L * 3 * md * 4 + 2 * B * L * md * 4 + stats + B * (L - 1)
    res["attention_kernels"] = {"fwd_us": t_f, "fwd_GBps": bytes_f / (t_f * 1e-6) / 1e9,
                                "bwd_us": t_b, "bwd_GBps": bytes_b / (t_b * 1e-6) / 1e9}
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()

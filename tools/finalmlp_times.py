"""Time of FinalMLP on the kernels: its training step, its dense forward + backward against stock torch eager, and
the interaction aggregation alone:

    python tools/finalmlp_times.py [--reps 20] [--rounds 5] [--out FILE]

Shape: FinalMLP_default (model_zoo/FinalMLP/config/model_config.yaml) at a Criteo-like size: 39 categorical fields of
25,641 rows, embedding 16 (d = 624), B 10000, mlp1 [1024, 512], mlp2 [1024, 512, 256], fs [1024, 512], 2 heads, no
context features.

- step: zoo.FinalMLP's whole fused_train_step (embedding, gates, towers, fusion, fused logit + BCE, clip + Adam),
  captured (pipeline.TrainPipeline) and replayed, per matmul mode; the same for zoo.DualMLP (FinalMLP's towers, each
  with a logit head) and for a FinalMLP with one context field per gate (fs1_context C0, fs2_context C1).
- dense: one forward + backward from the flattened embedding to the loss (gates, towers, fusion, sigmoid + BCE) of the
  same model, per mode, against the reference's ops restated in torch eager fp32: each gate MLP over the context row
  repeated B times, the towers' nn.Sequential, the fusion's view / matmul.  Both sides are captured in a CUDA graph.
- fusion: layers.InteractionAggregation alone, forward + backward, at the model's shape (H 2, dx 512, dy 256) and at
  a many-head shape (H 16, dx = dy = 512), against the reference's ops in eager fp32.

Every number is the median over `--rounds` rounds of `--reps` graph replays between CUDA events, after a warm-up:
the device's time, no host work.  The card's name and power limit are read in the same run and printed with them.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

MODES = ["fp32", "tf32x3", "tf32", "bf16"]
MODEL = dict(fields=39, vocab=25641, dim=16, B=10000, mlp1=[1024, 512], mlp2=[1024, 512, 256], fs=[1024, 512],
             heads=2)
FUSION_SHAPES = {"model_h2": dict(dx=512, dy=256, heads=2), "many_heads_h16": dict(dx=512, dy=512, heads=16)}


def gpu_name():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def graph_replay(fn):
    """fn captured in a CUDA graph after two warm-up calls on a side stream."""
    import torch
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            fn()
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        fn()
    return graph.replay


def timed(fn, reps, rounds):
    import torch
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    runs = []
    for _ in range(rounds):
        e0.record()
        for _ in range(reps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        runs.append(e0.elapsed_time(e1) * 1e3 / reps)
    return round(statistics.median(runs), 1), [round(x, 1) for x in runs]


def eager_fusion(agg, x, y):
    """InteractionAggregation.forward op for op (the reference's view / matmul), stock torch."""
    import torch
    out = agg.w_x(x) + agg.w_y(y)
    hx = x.view(-1, agg.num_heads, agg.head_x_dim)
    hy = y.view(-1, agg.num_heads, agg.head_y_dim)
    xy = torch.matmul(torch.matmul(hx.unsqueeze(2), agg.w_xy.view(agg.num_heads, agg.head_x_dim, -1))
                      .view(-1, agg.num_heads, agg.output_dim, agg.head_y_dim), hy.unsqueeze(-1)).squeeze(-1)
    return out + xy.sum(dim=1)


def eager_dense_loss(model, emb, label):
    """FinalMLP.forward after the embedding, as the reference runs it, in stock torch: the gates over the context
    row repeated B times, the towers' Sequentials, the fusion, sigmoid and BCE."""
    import torch
    fs, B = model.fs_module, emb.shape[0]
    g1 = fs.fs1_gate.mlp(fs.fs1_ctx_bias.repeat(B, 1)) * 2
    f1 = emb * g1
    g2 = fs.fs2_gate.mlp(fs.fs2_ctx_bias.repeat(B, 1)) * 2
    f2 = emb * g2
    logit = eager_fusion(model.fusion_module, model.mlp1.mlp(f1), model.mlp2.mlp(f2))
    return torch.nn.functional.binary_cross_entropy(torch.sigmoid(logit), label)


def kernel_dense_loss(model, emb, label):
    from fuxictr_b200 import functional as F2
    f1, f2 = model.fs_module({}, emb)
    return F2.logit_bce(label, model.fusion_module(model.mlp1(f1), model.mlp2(f2)))[0]


def criteo_like(m):
    import torch
    from fuxictr_b200.schema import FeatureMap
    specs = [("C%d" % i, {"type": "categorical", "source": "", "padding_idx": 0, "vocab_size": m["vocab"]})
             for i in range(m["fields"])]
    fm = FeatureMap.from_specs(specs, embedding_dim=m["dim"])
    gen = torch.Generator().manual_seed(11)
    ids = torch.randint(0, m["vocab"], (m["B"], m["fields"]), generator=gen).double()
    mat = torch.cat([ids, (torch.rand(m["B"], 1, generator=gen) < 0.25).double()], 1).cuda()
    return fm, mat


def make_model(name, fm, **extra):
    import torch
    from fuxictr_b200 import zoo
    m = MODEL
    torch.manual_seed(5)
    kw = dict(embedding_dim=m["dim"], mlp1_hidden_units=m["mlp1"], mlp2_hidden_units=m["mlp2"])
    if name == "FinalMLP":
        kw.update(fs_hidden_units=m["fs"], num_heads=m["heads"])
    kw.update(extra)
    return getattr(zoo, name)(fm, gpu=0, **kw)


def run_steps(args, fm, mat):
    import torch
    from fuxictr_b200 import functional as F2
    from fuxictr_b200.pipeline import TrainPipeline
    out = {}
    for tag, name, extra in (("FinalMLP", "FinalMLP", {}), ("DualMLP", "DualMLP", {}),
                             ("FinalMLP_ctx1", "FinalMLP", dict(fs1_context=["C0"], fs2_context=["C1"]))):
        out[tag] = {}
        for mode in MODES:
            F2.set_matmul_precision(mode)
            model = make_model(name, fm, **extra)
            model.use_fused_optimizer()
            pipe = TrainPipeline(model, MODEL["B"], mat.shape[1], graph=False)
            pipe.prime(mat)
            pipe.capture(warmup=3)
            us, runs = timed(lambda: pipe.step_device(mat), args.reps, args.rounds)
            out[tag][mode] = {"step_us": us, "step_runs": runs, "samples_per_s": round(MODEL["B"] / (us * 1e-6))}
            del pipe, model
            torch.cuda.empty_cache()
    F2.set_matmul_precision("fp32")
    return out


def run_dense(args, fm):
    import torch
    from fuxictr_b200 import functional as F2
    B, d = MODEL["B"], MODEL["fields"] * MODEL["dim"]
    model = make_model("FinalMLP", fm)
    gen = torch.Generator(device="cuda").manual_seed(8)
    emb = (torch.randn(B, d, device="cuda", generator=gen) * 0.1).requires_grad_(True)
    label = (torch.rand(B, 1, device="cuda", generator=gen) < 0.25).float()

    def step(loss_fn):
        def run():
            model.zero_grad(set_to_none=True)
            emb.grad = None
            loss_fn(model, emb, label).backward()
        return run

    def measure(loss_fn):
        us, runs = timed(graph_replay(step(loss_fn)), args.reps, args.rounds)
        with torch.no_grad():
            loss = float(loss_fn(model, emb, label))
        return {"fwd_bwd_us": us, "fwd_bwd_runs": runs, "loss": loss}

    F2.set_matmul_precision("fp32")
    res = {"torch_eager_fp32": measure(eager_dense_loss)}
    for mode in MODES:
        F2.set_matmul_precision(mode)
        res[mode] = measure(kernel_dense_loss)
        res[mode]["speedup"] = round(res["torch_eager_fp32"]["fwd_bwd_us"] / res[mode]["fwd_bwd_us"], 2)
    F2.set_matmul_precision("fp32")
    fs_row_macs = sum(a * b for a, b in zip([MODEL["dim"]] + MODEL["fs"], MODEL["fs"] + [d]))
    tower_macs = sum(a * b for a, b in zip([d] + MODEL["mlp1"][:-1], MODEL["mlp1"])) + \
        sum(a * b for a, b in zip([d] + MODEL["mlp2"][:-1], MODEL["mlp2"]))
    return {"macs_per_row": {"one_gate_mlp": fs_row_macs, "towers": tower_macs}, "results": res}


def run_fusion(args):
    import torch
    from fuxictr_b200 import functional as F2, layers
    B = MODEL["B"]
    out = {}
    for tag, s in FUSION_SHAPES.items():
        torch.manual_seed(7)
        agg = layers.InteractionAggregation(s["dx"], s["dy"], num_heads=s["heads"]).cuda()
        gen = torch.Generator(device="cuda").manual_seed(9)
        x = torch.rand(B, s["dx"], device="cuda", generator=gen).requires_grad_(True)
        y = torch.rand(B, s["dy"], device="cuda", generator=gen).requires_grad_(True)
        gout = torch.randn(B, 1, device="cuda", generator=gen)

        def step(f):
            def run():
                agg.zero_grad(set_to_none=True)
                x.grad = y.grad = None
                f(agg, x, y).backward(gout)
            return run
        F2.set_matmul_precision("fp32")
        res = {"torch_eager_fp32": {"fwd_bwd_us": timed(graph_replay(step(eager_fusion)), args.reps, args.rounds)[0]}}
        for mode in MODES:
            F2.set_matmul_precision(mode)
            us = timed(graph_replay(step(lambda m, a, b: m(a, b))), args.reps, args.rounds)[0]
            res[mode] = {"fwd_bwd_us": us, "speedup": round(res["torch_eager_fp32"]["fwd_bwd_us"] / us, 2)}
        F2.set_matmul_precision("fp32")
        hx, hy = s["dx"] // s["heads"], s["dy"] // s["heads"]
        out[tag] = {"shape": dict(s, B=B), "bilinear_macs_per_row": s["heads"] * hx * hy,
                    "block_diagonal_gemm_macs_per_row": (s["dy"] + 4) * s["dx"], "results": res}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None, help="also write the JSON here")
    args = ap.parse_args()
    import torch
    import __graft_entry__
    __graft_entry__.build()
    if not torch.cuda.is_available():
        raise SystemExit("finalmlp_times.py measures on a CUDA device; none is visible")
    torch.backends.cuda.matmul.allow_tf32 = False
    fm, mat = criteo_like(MODEL)
    out = {"gpu": gpu_name(), "shape": MODEL, "fusion": run_fusion(args), "dense": run_dense(args, fm),
           "step": run_steps(args, fm, mat)}
    text = json.dumps(out, indent=1)
    print(text)
    if args.out:
        with open(args.out, "w") as fd:
            fd.write(text)


if __name__ == "__main__":
    main()

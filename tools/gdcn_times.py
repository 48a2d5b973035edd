"""Time of GDCN's gated cross layer on the kernels against stock torch eager, and of a zoo.GDCN training step:

    python tools/gdcn_times.py [--reps 30] [--rounds 5] [--out FILE]

Layer shapes: "criteo16", B 8192, d 624 (39 fields x 16), and "default32", B 10000, d 1248 (39 x 32, GDCN_default's
embedding width), each a 3-layer layers.GateCorssLayer.  For each matmul mode (fp32, tf32x3, tf32, bf16) the layer's
forward, and forward + backward, are captured in a CUDA graph and replayed `--reps` times per round for `--rounds`
rounds between CUDA events, after a warm-up; the median per call is printed (the device's time: no host work).  The
baseline is the reference layer's own ops (two Linears, sigmoid, mul, add per layer) in torch eager fp32 on the same
GPU, captured and timed the same way.  Each mode's output is compared with those ops evaluated in float64 on a
float64 copy of the layer (relative Frobenius error).

Model: zoo.GDCN at the Criteo shape (39 fields of 25,641 rows, embedding 16, DNN [1024, 512, 256], B 8192) with the
fused optimizer; its whole fused_train_step is captured (pipeline.TrainPipeline) and replayed, per mode, and the
samples per second of the median round are printed.

The card's name and power limit are read in the same run and printed with the numbers.
"""
import argparse
import copy
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

LAYER_SHAPES = {"criteo16": dict(B=8192, d=624), "default32": dict(B=10000, d=1248)}
LAYERS = 3
MODES = ["fp32", "tf32x3", "tf32", "bf16"]
MODEL = dict(fields=39, vocab=25641, dim=16, dnn=[1024, 512, 256], B=8192)


def gpu_name():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def eager_forward(layer, x):
    """GateCorssLayer.forward op for op in stock torch: the reference's arithmetic."""
    import torch
    x0 = x
    for i in range(layer.cn_layers):
        xw = torch.nn.functional.linear(x, layer.w[i].weight)
        xg = torch.sigmoid(torch.nn.functional.linear(x, layer.wg[i].weight))
        x = x0 * (xw + layer.b[i]) * xg + x
    return x


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


def run_layer(s, args):
    import torch
    from fuxictr_b200 import functional as F2, layers
    B, d = s["B"], s["d"]
    torch.manual_seed(7)
    layer = layers.GateCorssLayer(d, LAYERS).cuda()
    gen = torch.Generator(device="cuda").manual_seed(8)
    x = torch.randn(B, d, device="cuda", generator=gen) * 0.5
    xg = x.clone().requires_grad_(True)
    gout = torch.randn(B, d, device="cuda", generator=gen)
    with torch.no_grad():
        y64 = eager_forward(copy.deepcopy(layer).double(), x.double())

    def fwd(f):
        def run():
            with torch.no_grad():
                f(layer, x)
        return run

    def fwd_bwd(f):
        def run():
            layer.zero_grad(set_to_none=True)
            xg.grad = None
            f(layer, xg).backward(gout)
        return run

    def mirror(m, a):
        return m(a)

    def measure(f):
        r = {}
        for key, make in (("fwd", fwd), ("fwd_bwd", fwd_bwd)):
            r[key + "_us"], r[key + "_runs"] = timed(graph_replay(make(f)), args.reps, args.rounds)
        with torch.no_grad():
            r["fwd_rel_fro_vs_fp64"] = float("%.3g" % float((f(layer, x).double() - y64).norm() / y64.norm()))
        return r

    F2.set_matmul_precision("fp32")
    results = {"torch_eager_fp32": measure(eager_forward)}
    for mode in MODES:
        F2.set_matmul_precision(mode)
        results[mode] = measure(mirror)
        for key in ("fwd_us", "fwd_bwd_us"):
            results[mode][key.replace("_us", "_speedup")] = round(results["torch_eager_fp32"][key] / results[mode][key], 2)
    F2.set_matmul_precision("fp32")
    gemm_gflop = 2.0 * B * (2 * d) * d / 1e9
    return {"shape": dict(s, layers=LAYERS), "fwd_gemm_gflop_per_layer": round(gemm_gflop, 2), "results": results}


def run_model(args):
    import torch
    from fuxictr_b200 import functional as F2, zoo
    from fuxictr_b200.pipeline import TrainPipeline
    from fuxictr_b200.schema import FeatureMap
    m = MODEL
    specs = [("C%d" % i, {"type": "categorical", "source": "", "padding_idx": 0, "vocab_size": m["vocab"]})
             for i in range(m["fields"])]
    fm = FeatureMap.from_specs(specs, embedding_dim=m["dim"])
    gen = torch.Generator().manual_seed(11)
    ids = torch.randint(0, m["vocab"], (m["B"], m["fields"]), generator=gen).double()
    mat = torch.cat([ids, (torch.rand(m["B"], 1, generator=gen) < 0.25).double()], 1).cuda()
    out = {}
    for mode in MODES:
        F2.set_matmul_precision(mode)
        torch.manual_seed(5)
        model = zoo.GDCN(fm, gpu=0, embedding_dim=m["dim"], dnn_hidden_units=m["dnn"], num_cross_layers=LAYERS)
        model.use_fused_optimizer()
        pipe = TrainPipeline(model, m["B"], mat.shape[1], graph=False)
        pipe.prime(mat)
        pipe.capture(warmup=3)
        us, runs = timed(lambda: pipe.step_device(mat), args.reps, args.rounds)
        out[mode] = {"step_us": us, "step_runs": runs, "samples_per_s": round(m["B"] / (us * 1e-6))}
        del pipe, model
        torch.cuda.empty_cache()
    F2.set_matmul_precision("fp32")
    return {"shape": m, "results": out}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None, help="also write the JSON here")
    args = ap.parse_args()
    import torch
    import __graft_entry__
    __graft_entry__.build()
    if not torch.cuda.is_available():
        raise SystemExit("gdcn_times.py measures on a CUDA device; none is visible")
    torch.backends.cuda.matmul.allow_tf32 = False
    out = {"gpu": gpu_name(),
           "layer": {name: run_layer(s, args) for name, s in LAYER_SHAPES.items()},
           "model_GDCN": run_model(args)}
    text = json.dumps(out, indent=1)
    print(text)
    if args.out:
        with open(args.out, "w") as fd:
            fd.write(text)


if __name__ == "__main__":
    main()

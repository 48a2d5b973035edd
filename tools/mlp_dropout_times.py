"""Step time of MLP dropout on the fused chain, against a build whose dropout stacks take the per-layer path:

    python tools/mlp_dropout_times.py [--reps 50] [--rounds 3] [--compare-root OTHER_TREE]

DeepFM C2 (B = 4096) and DCNv2 C3 (B = 8192) at bench.py's shapes, fused_train_step captured in a CUDA graph
(TrainPipeline) in 3xTF32, with net_dropout = 0.2 and with net_dropout = 0 (the ceiling).  One process times one
tree: it builds each model once, replays its graph `--reps` times per round for `--rounds` rounds (CUDA events),
and counts the kernels of one replay with torch.profiler.  --compare-root alternates subprocesses of this tree and
of another checkout (its library built), `--rounds` of each, and prints the medians with the card name and its
power limit.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

HERE = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CASES = [("deepfm", 0.2), ("deepfm", 0.0), ("dcnv2", 0.2), ("dcnv2", 0.0)]


def gpu_name():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def build(workload, p):
    import torch
    import bench
    from fuxictr_b200 import zoo
    from fuxictr_b200.schema import FeatureMap
    ns = argparse.Namespace(workload=workload, vocab_scale=1.0)
    specs = bench.make_specs(ns)
    fm = FeatureMap.from_specs(specs, embedding_dim=bench.DIM)
    torch.manual_seed(2019)
    with torch.device("cuda:0"):
        if workload == "deepfm":
            m = zoo.DeepFM(fm, gpu=0, embedding_dim=bench.DIM, hidden_units=bench.HIDDEN, net_dropout=p)
        else:
            m = zoo.DCNv2(fm, gpu=0, embedding_dim=bench.DIM, model_structure="parallel", num_cross_layers=3,
                          parallel_dnn_hidden_units=bench.DCN_HIDDEN, net_dropout=p)
    m.use_fused_optimizer()
    m.train()
    return m, fm, specs


def run_local(args):
    import torch
    from fuxictr_b200 import functional as F2
    from fuxictr_b200.pipeline import TrainPipeline
    import bench
    F2.set_matmul_precision("tf32x3")
    out = {}
    for workload, p in CASES:
        m, fm, specs = build(workload, p)
        B = bench.DEFAULT_BATCH[workload]
        batches = [b.cuda() for b in bench.make_batches(4, B, seed=1000, specs=specs)]
        pipe = TrainPipeline(m, B, batches[0].shape[1], torch.float64, graph=False)
        pipe.prime(batches[0])
        pipe.capture(warmup=3)
        for i in range(10):
            pipe.step_device(batches[i % 4])
        torch.cuda.synchronize()
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            pipe.step_device(batches[0])
            torch.cuda.synchronize()
        kernels = sum(1 for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA
                      and not e.name.lower().startswith(("memcpy", "memset")))
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        runs = []
        for _ in range(args.rounds):
            e0.record()
            for i in range(args.reps):
                pipe.step_device(batches[i % 4])
            e1.record()
            torch.cuda.synchronize()
            runs.append(e0.elapsed_time(e1) * 1e3 / args.reps)
        out["%s_p%s" % (workload, p)] = {"batch": B, "us_per_step_median": round(statistics.median(runs), 1),
                                         "us_per_step_runs": [round(x, 1) for x in runs], "kernels_per_step": kernels}
        del pipe, m
        torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--root", default=HERE, help="checkout whose fuxictr_b200 is imported")
    ap.add_argument("--compare-root", default="", help="another checkout: alternate runs of both trees")
    args = ap.parse_args()
    if args.compare_root:
        runs = {"this": [], "other": []}
        base = [sys.executable, os.path.abspath(__file__), "--reps", str(args.reps), "--rounds", "1"]
        for _ in range(args.rounds):
            for tag, root in (("other", args.compare_root), ("this", args.root)):
                r = subprocess.run(base + ["--root", os.path.abspath(root)], capture_output=True, text=True,
                                   timeout=1800)
                if r.returncode != 0:
                    raise SystemExit(r.stdout[-2000:] + r.stderr[-2000:])
                runs[tag].append(json.loads(r.stdout.strip().splitlines()[-1])["results"])
        summary = {}
        for case in runs["this"][0]:
            this = [x[case]["us_per_step_median"] for x in runs["this"]]
            other = [x[case]["us_per_step_median"] for x in runs["other"]]
            summary[case] = {"us_this": this, "us_other": other, "median_this": statistics.median(this),
                             "median_other": statistics.median(other),
                             "speedup_this_over_other": round(statistics.median(other) / statistics.median(this), 4),
                             "kernels_this": runs["this"][0][case]["kernels_per_step"],
                             "kernels_other": runs["other"][0][case]["kernels_per_step"]}
        print(json.dumps({"gpu": gpu_name(), "precision": "tf32x3", "compare": summary}))
        return
    sys.path.insert(0, os.path.abspath(args.root))
    print(json.dumps({"gpu": gpu_name(), "precision": "tf32x3", "root": os.path.abspath(args.root),
                      "results": run_local(args)}))


if __name__ == "__main__":
    main()

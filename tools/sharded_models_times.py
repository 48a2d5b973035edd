"""Step time of row-sharded tables at world 1 against the unsharded model, per workload (bench.py shapes):

    python tools/sharded_models_times.py [--workloads dcnv2,din,xdeepfm,deepfm] [--reps 30] [--rounds 3]
    python tools/sharded_models_times.py --workloads deepfm --sharded-only --compare-root OTHER_TREE

One real rank (SymmPeerGroup over a world-1 NCCL group: torch symmetric memory works at world 1), so the
sharded step runs the real push / pull kernels and barriers, with nothing to exchange.  Each workload builds
both models once; eager fused_train_steps alternate between them for `--rounds` rounds of `--reps` steps
(CUDA events), and the median us/step of each is printed with the card name and power limit.
--compare-root: the sharded step of this tree against the one of another checkout (its library built), in
alternating subprocesses, `--rounds` of each.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

HERE = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def gpu_name():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def build(ns, sharded):
    import torch
    import bench
    from fuxictr_b200 import zoo
    from fuxictr_b200.schema import FeatureMap
    fm = FeatureMap.from_specs(bench.make_specs(ns), embedding_dim=bench.DIM)
    torch.manual_seed(2019)
    D = bench.DIM
    with torch.device("cuda:0"):
        w = ns.workload
        if w == "deepfm":
            m = zoo.DeepFM(fm, gpu=0, embedding_dim=D, hidden_units=bench.HIDDEN)
        elif w == "dcnv2":
            m = zoo.DCNv2(fm, gpu=0, embedding_dim=D, model_structure="parallel", num_cross_layers=3,
                          parallel_dnn_hidden_units=bench.DCN_HIDDEN)
        elif w == "din":
            m = zoo.DIN(fm, gpu=0, embedding_dim=D, dnn_hidden_units=bench.DIN_HIDDEN, attention_hidden_units=[64],
                        attention_hidden_activations="Dice")
        else:
            m = zoo.xDeepFM(fm, gpu=0, embedding_dim=D, dnn_hidden_units=bench.XDFM_HIDDEN,
                            cin_hidden_units=bench.XDFM_CIN)
    if sharded:
        from fuxictr_b200.sharded import SymmPeerGroup
        m.enable_sharding(SymmPeerGroup(), ns.batch, fm.input_length + 1, torch.float64, want_fm=(w == "deepfm"))
    m.use_fused_optimizer()
    m.train()
    return m, fm


def time_steps(m, fm, batches, reps):
    import torch
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(reps):
        m.fused_train_step(fm.batch_dict(batches[i % len(batches)]))
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / reps


def run_local(args):
    import torch
    import torch.distributed as dist
    import bench
    from fuxictr_b200 import functional as F2
    torch.cuda.set_device(0)
    os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
    os.environ.setdefault("MASTER_PORT", "29631")
    dist.init_process_group("nccl", rank=0, world_size=1, device_id=torch.device("cuda", 0))
    F2.set_matmul_precision(args.precision)
    out = {}
    for w in args.workloads.split(","):
        ns = argparse.Namespace(workload=w, vocab_scale=1.0, batch=bench.DEFAULT_BATCH[w], dp_only=False, gpus=1)
        arms = [("sharded", True)] + ([] if args.sharded_only else [("unsharded", False)])
        models = {name: build(ns, sh) for name, sh in arms}
        batches = [b.cuda() for b in bench.make_batches(4, ns.batch, seed=1000, specs=bench.make_specs(ns))]
        for name, (m, fm) in models.items():           # warm-up (first-call plans, allocator)
            time_steps(m, fm, batches, 5)
        times = {name: [] for name in models}
        for _ in range(args.rounds):
            for name, (m, fm) in models.items():
                times[name].append(time_steps(m, fm, batches, args.reps))
        med = {k: round(statistics.median(v), 1) for k, v in times.items()}
        res = {"batch": ns.batch, "us_per_step_median": med,
               "us_per_step_runs": {k: [round(x, 1) for x in v] for k, v in times.items()}}
        if "unsharded" in med:
            res["sharded_over_unsharded"] = round(med["sharded"] / med["unsharded"], 4)
        out[w] = res
        del models
        torch.cuda.empty_cache()
    dist.destroy_process_group()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="dcnv2,din,xdeepfm,deepfm")
    ap.add_argument("--precision", default="tf32x3", choices=["tf32x3", "fp32"])
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--sharded-only", action="store_true")
    ap.add_argument("--root", default=HERE, help="checkout whose fuxictr_b200 is imported")
    ap.add_argument("--compare-root", default="", help="another checkout: alternate sharded runs of both trees")
    args = ap.parse_args()
    if args.compare_root:
        runs = {"this": [], "other": []}
        base = [sys.executable, os.path.abspath(__file__), "--workloads", args.workloads, "--precision", args.precision,
                "--reps", str(args.reps), "--rounds", "1", "--sharded-only"]
        for _ in range(args.rounds):
            for tag, root in (("other", args.compare_root), ("this", args.root)):
                r = subprocess.run(base + ["--root", os.path.abspath(root)], capture_output=True, text=True,
                                   timeout=1800)
                if r.returncode != 0:
                    raise SystemExit(r.stdout[-2000:] + r.stderr[-2000:])
                res = json.loads(r.stdout.strip().splitlines()[-1])
                runs[tag].append({w: v["us_per_step_median"]["sharded"] for w, v in res["results"].items()})
        summary = {}
        for w in args.workloads.split(","):
            this = [x[w] for x in runs["this"]]
            other = [x[w] for x in runs["other"]]
            summary[w] = {"sharded_us_this": this, "sharded_us_other": other,
                          "median_this": statistics.median(this), "median_other": statistics.median(other),
                          "this_over_other": round(statistics.median(this) / statistics.median(other), 4)}
        print(json.dumps({"gpu": gpu_name(), "precision": args.precision, "world": 1, "compare": summary}))
        return
    sys.path.insert(0, os.path.abspath(args.root))
    print(json.dumps({"gpu": gpu_name(), "precision": args.precision, "world": 1, "root": os.path.abspath(args.root),
                      "results": run_local(args)}))


if __name__ == "__main__":
    main()

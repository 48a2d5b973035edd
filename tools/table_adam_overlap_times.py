"""Step time with the table Adam split (FusedAdam.start_early_tables) against the serial table pass, and the sweep of
the untouched-granule pass's CTA cap (FusedAdam.EARLY_CTAS, one 1024-thread CTA per SM).  Every configuration is
one CUDA graph of the full training step (TrainPipeline, as bench.py replays it), captured once; the replays
alternate for `--rounds` rounds of `--reps` steps each and the median per step is printed.  `--profile` adds one
eager profiled step of each schedule and lists the Adam kernels in it (the table pass that remains after the norm).

    python tools/table_adam_overlap_times.py [--caps 16,24,32,48,66] [--profile]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--precision", default="tf32x3", choices=["tf32x3", "tf32", "bf16"])
    ap.add_argument("--caps", default="16,24,32,48,66")
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=9)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--out", default="", help="write the trace of the profiled steps here")
    args = ap.parse_args()
    import torch
    import bench
    from fuxictr_b200 import arena, functional as F2
    from fuxictr_b200.pipeline import TrainPipeline
    F2.set_matmul_precision(args.precision)
    ns = argparse.Namespace(workload="deepfm", vocab_scale=1.0, batch=bench.BATCH, dp_only=False, lazy_adam=0, gpus=1)
    model, fm, _ = bench.build_model(ns, 0, 1)
    opt = model._fused_optimizer
    width = fm.input_length + 1
    batches = [m.cuda() for m in bench.make_batches(4, ns.batch, seed=1000, specs=bench.make_specs(ns))]

    configs = [("serial", None)] + [("early_%d" % c, c) for c in (int(x) for x in args.caps.split(","))]
    pipes = {}
    for name, cap in configs:
        arena.set_early_table_adam(cap is not None)
        if cap is not None:
            opt.EARLY_CTAS = cap
        p = TrainPipeline(model, ns.batch, width, torch.float64, graph=False)
        p.prime(batches[0])
        p.capture(3)
        pipes[name] = p
    times = {k: [] for k in pipes}
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(args.rounds):
        for name, p in pipes.items():
            e0.record()
            for i in range(args.reps):
                p.step_device(batches[i % len(batches)])
            e1.record()
            torch.cuda.synchronize()
            times[name].append(e0.elapsed_time(e1) * 1e3 / args.reps)
    try:
        gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        gpu = torch.cuda.get_device_name()
    med = {k: round(statistics.median(v), 2) for k, v in times.items()}
    res = {"gpu": gpu, "workload": "deepfm", "precision": args.precision, "batch": ns.batch,
           "us_per_step_median": med, "us_range": {k: [round(min(v), 2), round(max(v), 2)] for k, v in times.items()},
           "speedup_vs_serial": {k: round(med["serial"] / v, 4) for k, v in med.items()}}
    if args.profile:
        from torch.profiler import profile, ProfilerActivity
        res["profiled_adam_kernels_us"] = {}
        for name, on in (("serial", False), ("early_%d" % opt.EARLY_CTAS, True)):
            arena.set_early_table_adam(on)
            for _ in range(3):
                model.fused_train_step(fm.batch_dict(batches[0]))
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                model.fused_train_step(fm.batch_dict(batches[1]))
                torch.cuda.synchronize()
            ks = [(e.name, round(e.device_time, 1)) for e in prof.events()
                  if e.device_time > 0 and ("adam" in e.name or "sumsq" in e.name or "table_mark" in e.name)]
            res["profiled_adam_kernels_us"][name] = ks
            if args.out:
                os.makedirs(args.out, exist_ok=True)
                prof.export_chrome_trace(os.path.join(args.out, "step_deepfm_%s.json" % name))
    print(json.dumps(res))


if __name__ == "__main__":
    main()

"""Device time of DeepFM C2's backward and optimizer step (batch 4096, 39 fields x 25,641 rows, D = 16, MLP
624-300-300-300-1), as fused_train_step runs them: the head backward, per MLP layer the dgrad and the wgrad, the
fused front's backward, then the fused clip + Adam.  Two schedules are captured, each as one CUDA graph of `--reps`
backward + optimizer passes over one forward: serial (every launch on one stream) and forked (the wgrads on a side
stream beside the dgrad chain, joined by the optimizer before it reads the dense gradients; functional._WgradFork).
The replays alternate for `--rounds` rounds; the median of each is printed.

    python tools/mlp_bwd_times.py [--precision tf32x3|tf32|bf16] [--reps 20] [--rounds 15]
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
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=15)
    args = ap.parse_args()
    import torch
    import bench
    from fuxictr_b200 import functional as F2, zoo
    from fuxictr_b200.schema import FeatureMap
    F2.set_matmul_precision(args.precision)
    F2.set_x3_inline(True)
    specs = bench.make_specs()
    fm = FeatureMap.from_specs(specs, embedding_dim=bench.DIM)
    torch.manual_seed(2019)
    model = zoo.DeepFM(fm, gpu=0, embedding_dim=bench.DIM, hidden_units=bench.HIDDEN)
    opt = model.use_fused_optimizer()
    model.train()
    batch = fm.batch_dict(bench.make_batches(1, bench.BATCH, specs=specs)[0].cuda())
    # autograd runs a node's backward on the stream its forward ran on: the forward runs on the capture stream
    stream = torch.cuda.Stream()
    stream.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(stream):
        loss, _ = F2.logit_bce(model.get_labels(batch), *model.forward_logits(batch))

    def backward_and_step():       # fused_train_step after its forward
        opt.zero_grad()
        opt.arena.defer_join = True
        loss.backward(retain_graph=True)
        opt.arena.defer_join = False
        opt.step()

    def capture(fork):
        F2.set_backward_fork(fork)
        with torch.cuda.stream(stream):
            for _ in range(3):
                backward_and_step()
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=stream):
            for _ in range(args.reps):
                backward_and_step()
        g.replay()
        torch.cuda.synchronize()
        return g

    graphs = {"serial": capture(False), "forked": capture(True)}
    times = {k: [] for k in graphs}
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(args.rounds):
        for name, g in graphs.items():
            e0.record()
            g.replay()
            e1.record()
            torch.cuda.synchronize()
            times[name].append(e0.elapsed_time(e1) * 1e3 / args.reps)
    try:
        gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        gpu = torch.cuda.get_device_name()
    med = {k: round(statistics.median(v), 2) for k, v in times.items()}
    print(json.dumps({"gpu": gpu, "precision": args.precision, "us_per_backward_and_step_median": med,
                      "us_range": {k: [round(min(v), 2), round(max(v), 2)] for k, v in times.items()},
                      "speedup": round(med["serial"] / med["forked"], 4)}))


if __name__ == "__main__":
    main()

"""Time of CrossNetMix (DCNv2's low-rank mixture of experts) on the kernels against stock torch eager:

    python tools/crossnet_mix_times.py [--reps 30] [--rounds 5] [--profile]

Shape C3: B = 8192, d = 624 (DCNv2's bench width), 3 layers, low_rank 32, 4 experts.  For each matmul mode
(fp32, tf32x3, tf32, bf16) the mirror layers.CrossNetMix runs forward, and forward + backward, `--reps` times per
round for `--rounds` rounds between CUDA events, after a warm-up; the median per call is printed.  The baseline
is the same computation written with the reference layer's own ops (per-sample (B, d, 1) matmuls per expert, a
stack and a batched matmul for the gate), in torch eager fp32 on the same GPU.  The card's name and power limit
are printed with the numbers.  --profile adds a separate torch.profiler run of one forward + backward per mode,
listing the kernels it launched.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

B, D, LAYERS, RANK, EXPERTS = 8192, 624, 3, 32, 4
MODES = ["fp32", "tf32x3", "tf32", "bf16"]


def gpu_name():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def eager_forward(layer, inputs):
    """CrossNetMix.forward (cross_net.py:167-201) op for op in stock torch: the reference's arithmetic."""
    import torch
    x_0 = inputs.unsqueeze(2)
    x_l = x_0
    for i in range(layer.layer_num):
        experts, gates = [], []
        for e in range(layer.num_experts):
            gates.append(layer.gating[e](x_l.squeeze(2)))
            v = torch.tanh(torch.matmul(layer.V_list[i][e].t(), x_l))
            v = torch.tanh(torch.matmul(layer.C_list[i][e], v))
            experts.append((x_0 * (torch.matmul(layer.U_list[i][e], v) + layer.bias[i])).squeeze(2))
        moe = torch.matmul(torch.stack(experts, 2), torch.stack(gates, 1).softmax(1))
        x_l = moe + x_l
    return x_l.squeeze()


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


def kernels_of(fn):
    import torch
    fn()
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    rows = {}
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            n, us = rows.get(e.name, (0, 0.0))
            rows[e.name] = (n + 1, us + e.device_time)
    return [{"kernel": k[:120], "launches": n, "us": round(us, 1)} for k, (n, us) in
            sorted(rows.items(), key=lambda kv: -kv[1][1])]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--profile", action="store_true")
    args = ap.parse_args()
    import torch
    import __graft_entry__
    __graft_entry__.build()
    from fuxictr_b200 import functional as F2, layers
    if not torch.cuda.is_available():
        raise SystemExit("crossnet_mix_times.py measures on a CUDA device; none is visible")
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.manual_seed(7)
    layer = layers.CrossNetMix(D, LAYERS, RANK, EXPERTS).cuda()
    with torch.no_grad():
        for b in layer.bias:
            b.normal_(0, 0.1)
    x = torch.randn(B, D, device="cuda") * 0.5
    xg = x.clone().requires_grad_(True)
    gout = torch.randn(B, D, device="cuda")

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

    def mirror(m, inp):
        return m(inp)

    results = {}
    us, runs = timed(fwd(eager_forward), args.reps, args.rounds)
    us2, runs2 = timed(fwd_bwd(eager_forward), args.reps, args.rounds)
    results["torch_eager_fp32"] = {"fwd_us": us, "fwd_runs": runs, "fwd_bwd_us": us2, "fwd_bwd_runs": runs2}
    with torch.no_grad():
        y_ref = eager_forward(layer, x)
    for mode in MODES:
        F2.set_matmul_precision(mode)
        with torch.no_grad():
            err = float((layer(x) - y_ref).norm() / y_ref.norm())
        us, runs = timed(fwd(mirror), args.reps, args.rounds)
        us2, runs2 = timed(fwd_bwd(mirror), args.reps, args.rounds)
        results[mode] = {"fwd_us": us, "fwd_runs": runs, "fwd_bwd_us": us2, "fwd_bwd_runs": runs2,
                         "fwd_rel_fro_vs_eager": float("%.3g" % err)}
    F2.set_matmul_precision("fp32")
    base = results["torch_eager_fp32"]
    for mode in MODES:
        results[mode]["fwd_speedup_vs_eager"] = round(base["fwd_us"] / results[mode]["fwd_us"], 2)
        results[mode]["fwd_bwd_speedup_vs_eager"] = round(base["fwd_bwd_us"] / results[mode]["fwd_bwd_us"], 2)
    out = {"gpu": gpu_name(), "shape": {"B": B, "d": D, "layers": LAYERS, "low_rank": RANK, "num_experts": EXPERTS},
           "results": results}
    if args.profile:
        prof = {"torch_eager_fp32": kernels_of(fwd_bwd(eager_forward))}
        for mode in MODES:
            F2.set_matmul_precision(mode)
            prof[mode] = kernels_of(fwd_bwd(mirror))
        F2.set_matmul_precision("fp32")
        out["profile_fwd_bwd"] = prof
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()

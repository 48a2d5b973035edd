"""Device time of each of the nine tensor-core GEMM launches of DeepFM C2's MLP (624-300-300-300-1, batch 4096)
in one training step, launched with the descriptors the fused MLP chain uses: three forwards (bias + ReLU), and
per layer, last first, the dgrad dX = dZ W (W MN-major; the ReLU backward of the layer below and its bias
gradient fused) and the wgrad dW = dZ^T X (both operands MN-major).

Each launch is timed by bench.time_kernel: back-to-back launches captured in one CUDA graph, CUDA events
around the replay.  Prints one JSON line: the GPU name and power limit, then microseconds per launch.

    python tools/gemm_c2_times.py [--precision tf32x3|tf32|bf16] [--reps 200]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--precision", default="tf32x3", choices=["tf32x3", "tf32", "bf16"])
    ap.add_argument("--reps", type=int, default=200)
    args = ap.parse_args()
    import torch
    from bench import time_kernel
    from fuxictr_b200 import functional as F2
    from fuxictr_b200._lib import B2_ACT_RELU
    F2.set_matmul_precision(args.precision)
    F2.set_x3_inline(True)
    B, dims = 4096, [624, 300, 300, 300]
    gen = torch.Generator(device="cuda").manual_seed(0)
    rnd = lambda *s: torch.randn(*s, device="cuda", generator=gen)  # noqa: E731
    xs = [rnd(B, d) for d in dims]                       # layer inputs (activations)
    ws = [rnd(dims[i + 1], dims[i]) * 0.05 for i in range(3)]
    bs = [rnd(dims[i + 1]) for i in range(3)]
    dzs = [rnd(B, dims[i + 1]) for i in range(3)]         # gradients at the pre-activations
    made = {id(t): F2.make_aux(t) for t in xs + ws + dzs}   # bf16 copies are made once, outside the timing
    aux = lambda t: made[id(t)]  # noqa: E731
    launches = []
    for i in range(3):
        y = torch.empty(B, dims[i + 1], device="cuda")
        launches.append(("fwd%d %dx%dx%d" % (i + 1, B, dims[i + 1], dims[i]),
                         lambda i=i, y=y: F2.gemm_ex(xs[i], ws[i], y, a_small=aux(xs[i]), b_small=aux(ws[i]),
                                                     bias=bs[i], act=B2_ACT_RELU)))
    for i in (2, 1, 0):
        dx = torch.empty(B, dims[i], device="cuda")
        if i > 0:       # dZ of the layer below: its ReLU backward against its output, and its bias gradient
            colsum = torch.empty(dims[i], device="cuda")
            launches.append(("dgrad%d %dx%dx%d" % (i + 1, B, dims[i], dims[i + 1]),
                             lambda i=i, dx=dx, cs=colsum: F2.gemm_ex(
                                 dzs[i], ws[i], dx, b_mn=True, a_small=aux(dzs[i]), b_small=aux(ws[i]),
                                 ybwd=xs[i], act_bwd=B2_ACT_RELU, colsum=cs)))
        else:
            launches.append(("dgrad%d %dx%dx%d" % (i + 1, B, dims[i], dims[i + 1]),
                             lambda i=i, dx=dx: F2.gemm_ex(dzs[i], ws[i], dx, b_mn=True, a_small=aux(dzs[i]),
                                                           b_small=aux(ws[i]))))
        dw = torch.zeros(dims[i + 1], dims[i], device="cuda")
        launches.append(("wgrad%d %dx%dx%d" % (i + 1, dims[i + 1], dims[i], B),
                         lambda i=i, dw=dw: F2.gemm_ex(dzs[i], xs[i], dw, a_mn=True, b_mn=True, a_small=aux(dzs[i]),
                                                       b_small=aux(xs[i]), out_is_zero=True)))
    us = {name: round(time_kernel(fn, args.reps) * 1e3, 2) for name, fn in launches}
    try:
        gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        gpu = torch.cuda.get_device_name()
    print(json.dumps({"gpu": gpu, "precision": args.precision, "us_per_launch": us,
                      "total_us": round(sum(us.values()), 2)}))


if __name__ == "__main__":
    main()

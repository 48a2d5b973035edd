"""Time of MultiHeadTargetAttention on the kernels against stock torch eager:

    python tools/target_attention_times.py [--reps 30] [--rounds 5]

Shapes: "sim", the SIM / ETA configs of the reference's LongCTR zoo (B 8192, history length 50, item width 12,
attention_dim 64, 2 heads), and "wide" (B 4096, L 200, d 64, attention_dim 64, 4 heads); histories are padded
to random lengths (a tenth of them padding only).  For each matmul mode (fp32, tf32x3, tf32, bf16) the mirror
layers.MultiHeadTargetAttention runs forward, and forward + backward, `--reps` times per round for `--rounds`
rounds between CUDA events, after a warm-up, first as eager calls (host work included) and then as replays of
the call captured in a CUDA graph (the device's time); the median per call is printed.  The baseline is the
reference layer's own ops (three projections, head split, matmul, scale, masked_fill, softmax, matmul, W_o) in
torch eager fp32 on the same GPU, timed the same two ways.  Also printed: the CUDA kernels one call launches and
their summed device time (torch.profiler, in a run of its own), the bytes each path moves by the algorithm's
count from the shapes (not measured), the relative Frobenius error of the output against eager fp32, and the
card's name and power limit.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SHAPES = {"sim": dict(B=8192, L=50, d=12, A=64, H=2), "wide": dict(B=4096, L=200, d=64, A=64, H=4)}
MODES = ["fp32", "tf32x3", "tf32", "bf16"]


def gpu_name():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def eager_forward(layer, t, x, mask):
    """MultiHeadTargetAttention.forward + ScaledDotProductAttention (target_attention.py:150-172,
    dot_product_attention.py:48-58) op for op in stock torch: the reference's arithmetic."""
    import torch
    B, H, hd = t.shape[0], layer.num_heads, layer.head_dim
    q = layer.W_q(t).view(B, 1, H, hd).transpose(1, 2)
    k = layer.W_k(x).view(B, -1, H, hd).transpose(1, 2)
    v = layer.W_v(x).view(B, -1, H, hd).transpose(1, 2)
    scores = torch.matmul(q, k.transpose(-1, -2)) / layer.scale
    scores = scores.masked_fill_(mask.view(B, 1, 1, -1).expand(-1, H, -1, -1).float() == 0, -1.e9)
    out = torch.matmul(scores.softmax(dim=-1), v)
    return layer.W_o(out.transpose(1, 2).contiguous().view(-1, H * hd))


def algorithmic_bytes(B, L, d, A, H):
    """Bytes each path reads and writes in HBM, counted from the shapes (fp32, byte mask), weights left out."""
    f = 4
    hist, hd_rows, rows = B * L * d * f, B * H * d * f, B * d * f
    ours_fwd = rows + hd_rows + (hd_rows + hist + B * L + hd_rows + 2 * B * H * f) + (hd_rows + rows)
    ours_bwd = (rows + hd_rows) + (rows + hd_rows) + (4 * hd_rows + 2 * B * H * f + 2 * hist + B * L) + \
        (hd_rows + rows) + (hd_rows + rows)
    kv, sc, qa = B * L * A * f, B * H * L * f, B * A * f
    eager_fwd = (rows + qa) + 2 * (hist + kv) + (qa + kv + sc) + 2 * sc + B * L + (2 * sc) + (sc + kv + qa) + \
        2 * qa + (qa + rows)
    return {"kernels_fwd_MB": round(ours_fwd / 1e6, 1), "kernels_bwd_MB": round(ours_bwd / 1e6, 1),
            "eager_fwd_MB": round(eager_fwd / 1e6, 1)}


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


def graph_replay(fn):
    """fn captured in a CUDA graph (after two warm-up calls on a side stream): its replay runs the same kernels
    without the host's Python and launch work, so its time is the device's."""
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


def kernel_launches(fn):
    """(kernels one call launches, their summed device time in us, their names) from torch.profiler."""
    import torch
    fn()
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    ev = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA
          and "Memcpy" not in e.name and "Memset" not in e.name]
    return len(ev), round(sum(e.device_time for e in ev), 1), sorted(set(e.name[:80] for e in ev))


def run_shape(name, s, args):
    import torch
    from fuxictr_b200 import functional as F2, layers
    B, L, d, A, H = s["B"], s["L"], s["d"], s["A"], s["H"]
    torch.manual_seed(7)
    layer = layers.MultiHeadTargetAttention(input_dim=d, attention_dim=A, num_heads=H).cuda()
    gen = torch.Generator(device="cuda").manual_seed(8)
    t = torch.randn(B, d, device="cuda", generator=gen) * 0.5
    x = torch.randn(B, L, d, device="cuda", generator=gen) * 0.5
    lens = torch.randint(1, L + 1, (B,), device="cuda", generator=gen)
    lens[torch.rand(B, device="cuda", generator=gen) < 0.1] = 0
    mask = (torch.arange(L, device="cuda")[None, :] < lens[:, None]).float()
    tg, xg = t.clone().requires_grad_(True), x.clone().requires_grad_(True)
    gout = torch.randn(B, d, device="cuda", generator=gen)

    def fwd(f):
        def run():
            with torch.no_grad():
                f(layer, t, x, mask)
        return run

    def fwd_bwd(f):
        def run():
            layer.zero_grad(set_to_none=True)
            tg.grad = xg.grad = None
            f(layer, tg, xg, mask).backward(gout)
        return run

    def mirror(m, a, b, c):
        return m(a, b, c)

    def measure(f):
        """Per call: host-clocked eager calls, then CUDA graph replays of the same call (device time)."""
        r = {}
        for key, make in (("fwd", fwd), ("fwd_bwd", fwd_bwd)):
            r[key + "_eager_us"], r[key + "_eager_runs"] = timed(make(f), args.reps, args.rounds)
            r[key + "_graph_us"], r[key + "_graph_runs"] = timed(graph_replay(make(f)), args.reps, args.rounds)
        return r

    results = {"torch_eager_fp32": measure(eager_forward)}
    with torch.no_grad():
        y_ref = eager_forward(layer, t, x, mask)
    for mode in MODES:
        F2.set_matmul_precision(mode)
        with torch.no_grad():
            err = float((layer(t, x, mask) - y_ref).norm() / y_ref.norm())
        results[mode] = measure(mirror)
        results[mode]["fwd_rel_fro_vs_eager"] = float("%.3g" % err)
    base = results["torch_eager_fp32"]
    for mode in MODES:
        for key in ("fwd_graph_us", "fwd_bwd_graph_us", "fwd_eager_us", "fwd_bwd_eager_us"):
            results[mode][key.replace("_us", "_speedup")] = round(base[key] / results[mode][key], 2)
    launches = {}
    F2.set_matmul_precision("fp32")
    for mode, f in [("torch_eager_fp32", eager_forward)] + [(m, mirror) for m in MODES]:
        if f is mirror:
            F2.set_matmul_precision(mode)
        n_f, us_f, k_f = kernel_launches(fwd(f))
        n_fb, us_fb, _ = kernel_launches(fwd_bwd(f))
        launches[mode] = {"fwd": n_f, "fwd_kernel_us": us_f, "fwd_bwd": n_fb, "fwd_bwd_kernel_us": us_fb,
                          "fwd_kernels": k_f}
    F2.set_matmul_precision("fp32")
    return {"shape": s, "bytes_from_shapes": algorithmic_bytes(B, L, d, A, H), "launches_per_call": launches,
            "results": results}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    import torch
    import __graft_entry__
    __graft_entry__.build()
    if not torch.cuda.is_available():
        raise SystemExit("target_attention_times.py measures on a CUDA device; none is visible")
    torch.backends.cuda.matmul.allow_tf32 = False
    out = {"gpu": gpu_name(), "shapes": {name: run_shape(name, s, args) for name, s in SHAPES.items()}}
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()

"""Time of AutoInt's self-attention stack on the kernels against stock torch eager, of its row kernels alone, and of a
zoo.AutoInt training step:

    python tools/autoint_times.py [--reps 30] [--rounds 5] [--out FILE]

Stack: AutoInt_default's interaction on the Criteo-like map, B 10000, F 39 fields, embedding 40, attention_dim 40,
2 heads, 3 layers (identity residual), as layers.MultiHeadSelfAttention.  For each matmul mode (fp32, tf32x3, tf32,
bf16) the stack's forward, and forward + backward, are captured in a CUDA graph and replayed `--reps` times per round
for `--rounds` rounds between CUDA events, after a warm-up; the median per call is printed (the device's time: no
host work).  The baseline is the reference's ops (three Linears, view/transpose, matmul, softmax, matmul, residual
add, ReLU per layer) restated in torch eager fp32 on the same GPU, captured and timed the same way.  Each mode's
output is compared with those ops evaluated in float64 (relative Frobenius error).

Row kernels: b2_autoint_fwd and b2_autoint_bwd alone at that shape, timed the same way, with the bytes they must
move and the FLOPs of the attention computed from the shapes, and the achieved rates.

Model: zoo.AutoInt at AutoInt_default on the Criteo-like map (39 fields of 25,641 rows, embedding 40, DNN
[400, 400], B 10000) with the fused optimizer; its whole fused_train_step is captured (pipeline.TrainPipeline) and
replayed, per mode, and the samples per second of the median round are printed.

The card's name and power limit are read in the same run and printed with the numbers.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

STACK = dict(B=10000, F=39, D=40, A=40, H=2, layers=3)
MODES = ["fp32", "tf32x3", "tf32", "bf16"]
MODEL = dict(fields=39, vocab=25641, dim=40, attention_dim=40, heads=2, layers=3, dnn=[400, 400], B=10000)


def gpu_name():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def eager_layer(m, X):
    """MultiHeadSelfAttention.forward op for op in stock torch: the reference's arithmetic."""
    import torch
    B = X.shape[0]
    q = torch.nn.functional.linear(X, m.W_q.weight).view(B, -1, m.num_heads, m.head_dim).transpose(1, 2)
    k = torch.nn.functional.linear(X, m.W_k.weight).view(B, -1, m.num_heads, m.head_dim).transpose(1, 2)
    v = torch.nn.functional.linear(X, m.W_v.weight).view(B, -1, m.num_heads, m.head_dim).transpose(1, 2)
    scores = torch.matmul(q, k.transpose(-1, -2))
    if m.scale:
        scores = scores / m.scale
    out = torch.matmul(scores.softmax(dim=-1), v).transpose(1, 2).contiguous().view(B, -1, m.num_heads * m.head_dim)
    res = torch.nn.functional.linear(X, m.W_res.weight) if m.W_res is not None else X
    if m.use_residual:
        out = out + res
    if m.layer_norm is not None:
        out = m.layer_norm(out)
    return out.relu()


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


def make_stack():
    import torch
    from fuxictr_b200 import layers
    s = STACK
    torch.manual_seed(7)
    return torch.nn.Sequential(*[layers.MultiHeadSelfAttention(s["D"] if i == 0 else s["A"], s["A"], s["H"])
                                 for i in range(s["layers"])]).cuda()


def run_stack(args):
    import copy
    import torch
    from fuxictr_b200 import functional as F2
    s = STACK
    stack = make_stack()
    gen = torch.Generator(device="cuda").manual_seed(8)
    x = torch.randn(s["B"], s["F"], s["D"], device="cuda", generator=gen) * 0.5
    xg = x.clone().requires_grad_(True)
    gout = torch.randn(s["B"], s["F"], s["A"], device="cuda", generator=gen)
    ref64 = copy.deepcopy(stack).double()
    with torch.no_grad():
        y64 = x.double()
        for m in ref64:
            y64 = eager_layer(m, y64)

    def kernels(a):
        n = len(stack)
        for i, m in enumerate(stack):
            a = m(a, want_aux=i + 1 < n)
        return a

    def eager(a):
        for m in stack:
            a = eager_layer(m, a)
        return a

    def fwd(f):
        def run():
            with torch.no_grad():
                f(x)
        return run

    def fwd_bwd(f):
        def run():
            stack.zero_grad(set_to_none=True)
            xg.grad = None
            f(xg).backward(gout)
        return run

    def measure(f):
        r = {}
        for key, make in (("fwd", fwd), ("fwd_bwd", fwd_bwd)):
            r[key + "_us"], r[key + "_runs"] = timed(graph_replay(make(f)), args.reps, args.rounds)
        with torch.no_grad():
            r["fwd_rel_fro_vs_fp64"] = float("%.3g" % float((f(x).double() - y64).norm() / y64.norm()))
        return r

    F2.set_matmul_precision("fp32")
    results = {"torch_eager_fp32": measure(eager)}
    for mode in MODES:
        F2.set_matmul_precision(mode)
        results[mode] = measure(kernels)
        for key in ("fwd_us", "fwd_bwd_us"):
            results[mode][key.replace("_us", "_speedup")] = round(results["torch_eager_fp32"][key] /
                                                                  results[mode][key], 2)
    F2.set_matmul_precision("fp32")
    rows = s["B"] * s["F"]
    return {"shape": s, "fwd_gemm_gflop_per_layer": round(2.0 * rows * 3 * s["A"] * s["D"] / 1e9, 2),
            "results": results}


def run_row_kernels(args):
    """b2_autoint_fwd / _bwd alone on one layer's P (identity residual, no LayerNorm, no dropout)."""
    import torch
    from fuxictr_b200 import _lib, functional as F2
    s = STACK
    B, F, A, H = s["B"], s["F"], s["A"], s["H"]
    rows, NP = B * F, 3 * A
    gen = torch.Generator(device="cuda").manual_seed(9)
    P = torch.randn(rows, NP, device="cuda", generator=gen) * 0.5
    X = torch.randn(rows, A, device="cuda", generator=gen)
    g = torch.randn(rows, A, device="cuda", generator=gen)
    out = torch.empty(rows, A, device="cuda")
    smax = torch.empty(B, H, F, device="cuda")
    ssum = torch.empty_like(smax)
    dP = torch.empty(rows, NP, device="cuda")
    gres = torch.empty(rows, A, device="cuda")
    p = F2._ptr
    z = p(None)

    def fwd():
        _lib.call("b2_autoint_fwd", p(P), p(X), B, F, A, A, H, 1, 0.0, z, z, 1e-5, z, 0, 0, 0.0, p(out), z, 0, 0,
                  p(smax), p(ssum), z, z, F2._stream())

    def bwd():
        _lib.call("b2_autoint_bwd", p(P), p(X), p(out), p(g), p(smax), p(ssum), z, z, B, F, A, A, H, 1, 0.0, z, z, 0,
                  0, 0.0, p(dP), z, 0, 0, p(gres), z, z, F2._stream())
    fwd()
    fwd_us, fwd_runs = timed(graph_replay(fwd), args.reps, args.rounds)
    bwd_us, bwd_runs = timed(graph_replay(bwd), args.reps, args.rounds)
    f4 = 4
    stats = 2 * B * H * F * f4
    fwd_bytes = rows * NP * f4 + rows * A * f4 * 2 + stats                   # P, X (residual); out; statistics
    bwd_bytes = rows * NP * f4 + rows * A * f4 * 3 + stats + rows * NP * f4 + rows * A * f4   # + out, g; dP, gres
    dh = A // H
    fwd_flop = 2.0 * B * H * F * F * dh * 2                                  # scores and A V
    bwd_flop = 2.0 * B * H * F * F * dh * 5            # recomputed scores; dA, dV, dQ, dK (no LayerNorm: O not rebuilt)
    return {"fwd_us": fwd_us, "fwd_runs": fwd_runs, "bwd_us": bwd_us, "bwd_runs": bwd_runs,
            "fwd_mbytes": round(fwd_bytes / 1e6, 1), "bwd_mbytes": round(bwd_bytes / 1e6, 1),
            "fwd_gflop": round(fwd_flop / 1e9, 2), "bwd_gflop": round(bwd_flop / 1e9, 2),
            "fwd_tb_per_s": round(fwd_bytes / (fwd_us * 1e-6) / 1e12, 2),
            "bwd_tb_per_s": round(bwd_bytes / (bwd_us * 1e-6) / 1e12, 2),
            "fwd_tflop_per_s": round(fwd_flop / (fwd_us * 1e-6) / 1e12, 2),
            "bwd_tflop_per_s": round(bwd_flop / (bwd_us * 1e-6) / 1e12, 2)}


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
        model = zoo.AutoInt(fm, gpu=0, embedding_dim=m["dim"], attention_dim=m["attention_dim"],
                            num_heads=m["heads"], attention_layers=m["layers"], dnn_hidden_units=m["dnn"])
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
        raise SystemExit("autoint_times.py measures on a CUDA device; none is visible")
    torch.backends.cuda.matmul.allow_tf32 = False
    out = {"gpu": gpu_name(), "stack": run_stack(args), "row_kernels": run_row_kernels(args),
           "model_AutoInt": run_model(args)}
    text = json.dumps(out, indent=1)
    print(text)
    if args.out:
        with open(args.out, "w") as fd:
            fd.write(text)


if __name__ == "__main__":
    main()

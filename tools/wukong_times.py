"""Time of WuKong's layer stack on the kernels against stock torch eager, of its row kernels alone, and of a
zoo.WuKong training step:

    python tools/wukong_times.py [--reps 20] [--rounds 5] [--out FILE]

Stack: WuKong_default's interaction on the Criteo-like map, B 10000, F 39 fields, embedding 64, 3 layers of
lcb = fmb = 40 (layer 0 with the residual projection 39 -> 80), rank 8, FMB MLP [512, 256], as layers.WuKongLayer.
For each matmul mode (fp32, tf32x3, tf32, bf16) the stack's forward, and forward + backward, are captured in a CUDA
graph and replayed `--reps` times per round for `--rounds` rounds between CUDA events, after a warm-up; the median per
call is printed.  The baseline is the reference's ops (x^T Y, bmm, LayerNorm, the MLP, the transposed Linears, cat,
residual add, LayerNorm per layer) restated in torch eager fp32 on the same GPU, captured and timed the same way.
Each mode's output is compared with those ops evaluated in float64 (relative Frobenius error).

Row kernels: b2_wukong_fm_fwd (layer 0: reads X, writes X'_0 and the MLP input; layer 1: reads X') and
b2_wukong_out_fwd (layer 1: identity residual, writes X'), and their backward passes, alone at that shape, timed the
same way, with the bytes they must move counted from the shapes and the achieved rate.

Model: zoo.WuKong at WuKong_default on the Criteo-like map (39 fields of 25,641 rows, fc [512, 256], B 10000) with the
fused optimizer, mlp_batch_norm on and off; its whole fused_train_step is captured (pipeline.TrainPipeline) and
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

STACK = dict(B=10000, F=39, D=64, lcb=40, fmb=40, k=8, fmb_mlp=[512, 256], layers=3)
MODES = ["fp32", "tf32x3", "tf32", "bf16"]
MODEL = dict(fields=39, vocab=25641, B=10000, kw=dict(embedding_dim=64, num_wukong_layers=3, lcb_features=40,
                                                       fmb_features=40, fmb_mlp_units=[512, 256], fmp_rank_k=8,
                                                       mlp_hidden_units=[512, 256]))


def gpu_name():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def eager_layer(m, x):
    """WuKongLayer.forward op for op in stock torch: the reference's arithmetic."""
    import torch
    import torch.nn.functional as F
    fmb = m.fmb
    fm = torch.bmm(x, x.transpose(1, 2) @ fmb.proj_Y).flatten(start_dim=1)
    h = F.layer_norm(fm, fm.shape[1:], fmb.layer_norm.weight, fmb.layer_norm.bias, fmb.layer_norm.eps)
    for mod in fmb.mlp.mlp:
        h = F.linear(h, mod.weight, mod.bias) if isinstance(mod, torch.nn.Linear) else torch.relu(h)
    out = torch.cat([h.view(x.shape[0], -1, x.shape[2]), F.linear(x.transpose(1, 2), m.lcb.linear.weight).transpose(1, 2)], 1)
    res = getattr(m, "residual_proj", None)
    out = out + (F.linear(x.transpose(1, 2), res.weight, res.bias).transpose(1, 2) if res is not None else x)
    return F.layer_norm(out, out.shape[-1:], m.layer_norm.weight, m.layer_norm.bias, m.layer_norm.eps)


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
    net = torch.nn.Sequential(*[layers.WuKongLayer(s["F"] if i == 0 else s["lcb"] + s["fmb"], s["lcb"], s["fmb"],
                                                   s["D"], s["k"], s["fmb_mlp"], "relu", 0.0, True)
                                for i in range(s["layers"])])
    with torch.no_grad():
        for m in net:
            m.fmb.proj_Y.mul_(0.3)
    return net.cuda()


def run_stack(args):
    import copy
    import torch
    from fuxictr_b200 import functional as F2, layers
    s = STACK
    stack = make_stack()
    gen = torch.Generator(device="cuda").manual_seed(8)
    x = torch.randn(s["B"], s["F"], s["D"], device="cuda", generator=gen) * 0.5
    xg = x.clone().requires_grad_(True)
    gout = torch.randn(s["B"], (s["lcb"] + s["fmb"]) * s["D"], device="cuda", generator=gen)
    ref64 = copy.deepcopy(stack).double()
    with torch.no_grad():
        y64 = x.double()
        for m in ref64:
            y64 = eager_layer(m, y64)
        y64 = y64.flatten(start_dim=1)

    def kernels(a):
        return layers.wukong_stack(list(stack), a)

    def eager(a):
        for m in stack:
            a = eager_layer(m, a)
        return a.flatten(start_dim=1)

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
    return {"shape": s, "results": results}


def run_row_kernels(args):
    """The four row kernels alone at the default shape, fp32 operands (no operand copies)."""
    import torch
    from fuxictr_b200 import _lib, functional as F2
    s = STACK
    B, F, D, k, lcb, fmb = s["B"], s["F"], s["D"], s["k"], s["lcb"], s["fmb"]
    Fo = lcb + fmb
    fp0, fpo = F2.wukong_pitch(F), F2.wukong_pitch(Fo)
    gen = torch.Generator(device="cuda").manual_seed(9)

    def rnd(*shape):
        return torch.randn(*shape, device="cuda", generator=gen) * 0.5
    X, Xp = rnd(B, F, D), rnd(B * D, fpo)
    Y0, Y1 = rnd(F, k), rnd(Fo, k)
    g0, b0, g1, b1 = rnd(F * k) + 1, rnd(F * k), rnd(Fo * k) + 1, rnd(Fo * k)
    fm0, fm1 = torch.empty(B, F * k, device="cuda"), torch.empty(B, Fo * k, device="cuda")
    xp0 = torch.empty(B * D, fp0, device="cuda")
    mean, rstd = torch.empty(B * Fo, device="cuda"), torch.empty(B * Fo, device="cuda")
    mlp, C = rnd(B, fmb * D), rnd(B * D, lcb)
    gam, bet = rnd(D) + 1, rnd(D)
    out, gout = torch.empty(B * D, fpo, device="cuda"), rnd(B * D, fpo)
    gfm = rnd(B, Fo * k)
    gx = torch.empty(B * D, fpo, device="cuda")
    gY, dg, db = torch.zeros(Fo * k, device="cuda"), torch.zeros(Fo * k, device="cuda"), torch.zeros(Fo * k, device="cuda")
    gmlp, dC = torch.empty(B, fmb * D, device="cuda"), torch.empty(B * D, lcb, device="cuda")
    dgam, dbet = torch.zeros(D, device="cuda"), torch.zeros(D, device="cuda")
    p, z, st = F2._ptr, F2._ptr(None), F2._stream
    m1, r1 = torch.empty(B, device="cuda"), torch.empty(B, device="cuda")

    def fm_fwd0():
        _lib.call("b2_wukong_fm_fwd", p(X), 0, B, F, D, k, p(Y0), p(g0), p(b0), 1e-5, p(fm0), z, 0, 0, p(xp0), z, 0,
                  p(m1), p(r1), st())

    def fm_fwd1():
        _lib.call("b2_wukong_fm_fwd", p(Xp), 1, B, Fo, D, k, p(Y1), p(g1), p(b1), 1e-5, p(fm1), z, 0, 0, z, z, 0,
                  p(m1), p(r1), st())

    def fm_bwd1():
        _lib.call("b2_wukong_fm_bwd", p(Xp), 1, B, Fo, D, k, p(Y1), p(g1), p(m1), p(r1), p(gfm), z, p(gx), 1, p(gY),
                  p(dg), p(db), st())

    def out_fwd1():
        _lib.call("b2_wukong_out_fwd", p(mlp), p(C), p(Xp), B, Fo, D, lcb, fmb, 1, p(gam), p(bet), 1e-5, 1, p(out), z,
                  0, 0, p(mean), p(rstd), st())

    def out_bwd1():
        _lib.call("b2_wukong_out_bwd", p(mlp), p(C), p(Xp), B, Fo, D, lcb, fmb, 1, p(gam), p(mean), p(rstd), 1,
                  p(gout), p(gmlp), p(dC), z, 0, 0, p(gx), 0, z, p(dgam), p(dbet), st())
    f4 = 4
    nbytes = {   # counted from the shapes: every tensor the kernel must read or write once
        "fm_fwd_layer0": f4 * (B * F * D + B * D * fp0 + B * F * k + 2 * B),
        "fm_fwd_layer1": f4 * (B * D * fpo + B * Fo * k + 2 * B),
        "fm_bwd_layer1": f4 * (B * D * fpo + B * Fo * k + 2 * B + 2 * B * D * fpo),      # X', g, stats; gx read + write
        "out_fwd_layer1": f4 * (B * fmb * D + B * D * lcb + 2 * B * D * fpo + 2 * B * Fo),
        "out_bwd_layer1": f4 * (B * fmb * D + B * D * lcb + B * D * fpo + 2 * B * Fo + B * D * fpo   # z's inputs, g
                                + B * fmb * D + B * D * lcb + B * D * fpo),                      # g_mlp, dC, gx
    }
    fm_fwd1()
    out_fwd1()
    res = {}
    for name, fn in (("fm_fwd_layer0", fm_fwd0), ("fm_fwd_layer1", fm_fwd1), ("fm_bwd_layer1", fm_bwd1),
                     ("out_fwd_layer1", out_fwd1), ("out_bwd_layer1", out_bwd1)):
        us, runs = timed(graph_replay(fn), args.reps, args.rounds)
        res[name] = {"us": us, "runs": runs, "mbytes": round(nbytes[name] / 1e6, 1),
                     "tb_per_s": round(nbytes[name] / (us * 1e-6) / 1e12, 2)}
    return res


def run_model(args):
    import torch
    from fuxictr_b200 import functional as F2, zoo
    from fuxictr_b200.pipeline import TrainPipeline
    from fuxictr_b200.schema import FeatureMap
    m = MODEL
    specs = [("C%d" % i, {"type": "categorical", "source": "", "padding_idx": 0, "vocab_size": m["vocab"]})
             for i in range(m["fields"])]
    fm = FeatureMap.from_specs(specs, embedding_dim=m["kw"]["embedding_dim"])
    gen = torch.Generator().manual_seed(11)
    ids = torch.randint(0, m["vocab"], (m["B"], m["fields"]), generator=gen).double()
    mat = torch.cat([ids, (torch.rand(m["B"], 1, generator=gen) < 0.25).double()], 1).cuda()
    out = {}
    for bn in (True, False):
        for mode in MODES:
            F2.set_matmul_precision(mode)
            torch.manual_seed(5)
            model = zoo.WuKong(fm, gpu=0, mlp_batch_norm=bn, **m["kw"])
            model.use_fused_optimizer()
            pipe = TrainPipeline(model, m["B"], mat.shape[1], graph=False)
            pipe.prime(mat)
            pipe.capture(warmup=3)
            us, runs = timed(lambda: pipe.step_device(mat), args.reps, args.rounds)
            out["%s_bn%d" % (mode, bn)] = {"step_us": us, "step_runs": runs,
                                           "samples_per_s": round(m["B"] / (us * 1e-6))}
            del pipe, model
            torch.cuda.empty_cache()
    F2.set_matmul_precision("fp32")
    return {"shape": m, "results": out}


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
        raise SystemExit("wukong_times.py measures on a CUDA device; none is visible")
    torch.backends.cuda.matmul.allow_tf32 = False
    out = {"gpu": gpu_name(), "stack": run_stack(args), "row_kernels": run_row_kernels(args),
           "model_WuKong": run_model(args)}
    text = json.dumps(out, indent=1)
    print(text)
    if args.out:
        with open(args.out, "w") as fd:
            fd.write(text)


if __name__ == "__main__":
    main()

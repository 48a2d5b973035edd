"""Time of FinalNet's dense part on the kernels against stock torch eager, of its row kernels alone, and of a
zoo.FinalNet training step:

    python tools/finalnet_times.py [--reps 20] [--rounds 5] [--out FILE]

Dense part: FinalNet_default (2B, feature gating, batch norm, concat, blocks [64, 64, 64]) from the field embeddings
(B 10000, F 39, D 40) to the loss: the gating, both blocks, fc1 / fc2 and the 2B loss, forward and backward.  For each
matmul mode (fp32, tf32x3, tf32, bf16) that is captured in a CUDA graph and replayed `--reps` times per round for
`--rounds` rounds between CUDA events, after a warm-up; the median per call is printed.  The baseline is the
reference's ops (the gating Linear over the field axis, cat, each FactorizedInteraction's Linear, chunk, cat,
BatchNorm1d in training, fc1 / fc2 and add_loss's three BCE terms) in torch eager fp32 on the same GPU, captured and
timed the same way.  Each mode's loss is compared with those ops evaluated in float64 (relative error).

Row kernels: b2_finalnet_gate_fwd / _bwd at (10000, 39, 40), and b2_finalnet_fi_fwd / _bwd of block 1's first layer
(h of width 2 x 32, batch norm in training), alone, timed the same way, with the bytes they must move counted from the
shapes and the achieved rate.

Model: zoo.FinalNet at FinalNet_default on the Criteo-like map (39 fields of 25,641 rows, D 40, B 10000) with the
fused optimizer; its whole fused_train_step is captured (pipeline.TrainPipeline) and replayed, per mode, and the
samples per second of the median round are printed.

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

MODES = ["fp32", "tf32x3", "tf32", "bf16"]
SHAPE = dict(B=10000, F=39, D=40, vocab=25641)
DEFAULT = dict(embedding_dim=40, block_type="2B", batch_norm=True, use_feature_gating=True,
               block1_hidden_units=[64, 64, 64], block2_hidden_units=[64, 64, 64], residual_type="concat")


def gpu_name():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return "unknown"


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


def feature_map():
    from fuxictr_b200.schema import FeatureMap
    specs = [("C%d" % i, {"type": "categorical", "source": "", "padding_idx": 0, "vocab_size": SHAPE["vocab"]})
             for i in range(SHAPE["F"])]
    return FeatureMap.from_specs(specs, embedding_dim=SHAPE["D"])


def eager_block(block, x):
    """FinalBlock.forward op for op in stock torch (no dropout, activations None): the reference's arithmetic."""
    import torch
    import torch.nn.functional as F
    for lin, norm in zip(block.layer, block.norm):
        h = F.linear(x, lin.linear.weight, lin.linear.bias)
        h2, h1 = torch.chunk(h, 2, dim=-1)
        x = F.batch_norm(torch.cat([h2, h1 * h2], dim=-1), norm.running_mean, norm.running_var, norm.weight,
                         norm.bias, True, norm.momentum, norm.eps)
    return x


def eager_dense(model, e, y):
    """FinalNet.forward + add_loss from the embedding e (B, F, D), in stock torch."""
    import torch
    import torch.nn.functional as F
    gates = F.linear(e.transpose(1, 2), model.feature_gating.linear.weight,
                     model.feature_gating.linear.bias).transpose(1, 2)
    x1 = torch.cat([e, e * gates], dim=1).flatten(start_dim=1)
    y1 = F.linear(eager_block(model.block1, x1), model.fc1.weight, model.fc1.bias)
    y2 = F.linear(eager_block(model.block2, e.flatten(start_dim=1)), model.fc2.weight, model.fc2.bias)
    p = torch.sigmoid(0.5 * (y1 + y2))
    return (F.binary_cross_entropy(p, y) + F.binary_cross_entropy(torch.sigmoid(y1), p.detach())
            + F.binary_cross_entropy(torch.sigmoid(y2), p.detach()))


def kernel_dense(model, e, y):
    """The same on the kernels: zoo.FinalNet.forward_logits from e, then functional.finalnet_loss."""
    from fuxictr_b200 import functional as F2
    flat, sink = F2.shared_grad(e.flatten(start_dim=1))
    x1 = model.feature_gating.run(flat, sink=sink, want_aux=F2._tc_layer_ok(model.block1.layer[0].linear.weight))
    y1 = F2.linear_act(model.block1.run(x1), model.fc1.weight, model.fc1.bias)
    y2 = F2.linear_act(model.block2.run(flat, sink=sink), model.fc2.weight, model.fc2.bias)
    return F2.finalnet_loss(y, y1, y2)[0]


def make_model():
    import torch
    from fuxictr_b200 import zoo
    torch.manual_seed(5)
    model = zoo.FinalNet(feature_map(), gpu=0, **DEFAULT)
    with torch.no_grad():
        model.feature_gating.linear.weight.normal_(0, 0.1)
    return model.train()


def run_dense(args):
    import copy
    import torch
    from fuxictr_b200 import functional as F2
    s = SHAPE
    model = make_model()
    gen = torch.Generator(device="cuda").manual_seed(8)
    e = torch.randn(s["B"], s["F"], s["D"], device="cuda", generator=gen) * 0.3
    y = (torch.rand(s["B"], 1, device="cuda", generator=gen) < 0.25).float()
    eg = e.clone().requires_grad_(True)
    ref64 = copy.deepcopy(model).double()
    with torch.no_grad():
        l64 = float(eager_dense(ref64, e.double(), y.double()))

    def fwd_bwd(f):
        def run():
            model.zero_grad(set_to_none=True)
            eg.grad = None
            f(model, eg, y).backward()
        return run

    def measure(f):
        r = {}
        r["fwd_bwd_us"], r["fwd_bwd_runs"] = timed(graph_replay(fwd_bwd(f)), args.reps, args.rounds)
        with torch.no_grad():
            r["loss_rel_err_vs_fp64"] = float("%.3g" % (abs(float(f(model, e, y)) - l64) / abs(l64)))
        return r

    F2.set_matmul_precision("fp32")
    results = {"torch_eager_fp32": measure(eager_dense)}
    for mode in MODES:
        F2.set_matmul_precision(mode)
        results[mode] = measure(kernel_dense)
        results[mode]["fwd_bwd_speedup"] = round(results["torch_eager_fp32"]["fwd_bwd_us"] /
                                                 results[mode]["fwd_bwd_us"], 2)
    F2.set_matmul_precision("fp32")
    return {"shape": dict(s, model=DEFAULT), "results": results}


def run_row_kernels(args):
    """The gating and block 1's first FI layer alone at the default shape, fp32 operands (no operand copies)."""
    import torch
    from fuxictr_b200 import _lib, functional as F2
    s = SHAPE
    B, F, D = s["B"], s["F"], s["D"]
    half, n = 32, 64
    gen = torch.Generator(device="cuda").manual_seed(9)

    def rnd(*shape):
        return torch.randn(*shape, device="cuda", generator=gen) * 0.5
    e, W, b = rnd(B, F, D), rnd(F, F) * 0.2, rnd(F) + 1
    gout_gate, out_gate, de = rnd(B, 2 * F * D), torch.empty(B, 2 * F * D, device="cuda"), torch.empty(B, F, D,
                                                                                                        device="cuda")
    dW, db = torch.zeros(F, F, device="cuda"), torch.zeros(F, device="cuda")
    h, out, g, dh = rnd(B, 2 * half), torch.empty(B, n, device="cuda"), rnd(B, n), torch.empty(B, 2 * half,
                                                                                              device="cuda")
    gamma, beta = rnd(n) + 1, rnd(n)
    rm, rv, nbt = torch.zeros(n, device="cuda"), torch.ones(n, device="cuda"), torch.zeros(1, dtype=torch.int64,
                                                                                         device="cuda")
    ws = torch.empty(4 * n, dtype=torch.float64, device="cuda")
    mean, rstd = torch.empty(n, device="cuda"), torch.empty(n, device="cuda")
    dbias, dgamma, dbeta = torch.zeros(2 * half, device="cuda"), torch.empty(n, device="cuda"), torch.empty(
        n, device="cuda")
    p, z, st = F2._ptr, F2._ptr(None), F2._stream

    def gate_fwd():
        _lib.call("b2_finalnet_gate_fwd", p(e), B, F, D, p(W), p(b), p(out_gate), z, 0, 0, st())

    def gate_bwd():
        _lib.call("b2_finalnet_gate_bwd", p(e), B, F, D, p(W), p(b), p(gout_gate), p(de), 0, p(dW), p(db), st())

    def fi_fwd():
        _lib.call("b2_finalnet_fi_fwd", p(h), B, half, _lib.B2_FINALNET_CONCAT, p(gamma), p(beta), 1e-5, 0.1, 1, p(rm),
                  p(rv), p(nbt), p(ws), 0, z, 0, 0, 0.0, p(out), z, 0, 0, p(mean), p(rstd), st())

    def fi_bwd():
        _lib.call("b2_finalnet_fi_bwd", p(h), B, half, _lib.B2_FINALNET_CONCAT, p(gamma), p(beta), p(mean), p(rstd), 1,
                  ctypes_offset(ws, 2 * n), 1, 0, z, 0, 0, 0.0, p(g), p(dh), z, 0, 0, p(dbias), p(dgamma), p(dbeta),
                  st())
    f4 = 4
    nbytes = {   # counted from the shapes: every tensor the entry point's passes must read or write
        "gate_fwd": f4 * (B * F * D + 2 * B * F * D),                       # e; out
        "gate_bwd": f4 * (B * F * D + 2 * B * F * D + B * F * D),           # e, g; de
        "fi_fwd_train_bn": f4 * (2 * B * 2 * half + B * n),                 # h twice (statistics, apply); out
        "fi_bwd_train_bn": f4 * (2 * (B * 2 * half + B * n) + B * 2 * half),   # h and g twice; dh
    }
    fi_fwd()
    res = {}
    for name, fn in (("gate_fwd", gate_fwd), ("gate_bwd", gate_bwd), ("fi_fwd_train_bn", fi_fwd),
                     ("fi_bwd_train_bn", fi_bwd)):
        us, runs = timed(graph_replay(fn), args.reps, args.rounds)
        res[name] = {"us": us, "runs": runs, "mbytes": round(nbytes[name] / 1e6, 1),
                     "tb_per_s": round(nbytes[name] / (us * 1e-6) / 1e12, 2)}
    return res


def ctypes_offset(t, elems):
    import ctypes
    return ctypes.c_void_p(t.data_ptr() + elems * t.element_size())


def run_model(args):
    import torch
    from fuxictr_b200 import functional as F2
    from fuxictr_b200.pipeline import TrainPipeline
    s = SHAPE
    fm = feature_map()
    gen = torch.Generator().manual_seed(11)
    ids = torch.randint(0, s["vocab"], (s["B"], s["F"]), generator=gen).double()
    mat = torch.cat([ids, (torch.rand(s["B"], 1, generator=gen) < 0.25).double()], 1).cuda()
    out = {}
    for mode in MODES:
        F2.set_matmul_precision(mode)
        model = make_model()
        model.use_fused_optimizer()
        pipe = TrainPipeline(model, s["B"], mat.shape[1], graph=False)
        pipe.prime(mat)
        pipe.capture(warmup=3)
        us, runs = timed(lambda: pipe.step_device(mat), args.reps, args.rounds)
        out[mode] = {"step_us": us, "step_runs": runs, "samples_per_s": round(s["B"] / (us * 1e-6))}
        del pipe, model
        torch.cuda.empty_cache()
    F2.set_matmul_precision("fp32")
    return {"shape": dict(s, model=DEFAULT), "results": out}


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
        raise SystemExit("finalnet_times.py measures on a CUDA device; none is visible")
    torch.backends.cuda.matmul.allow_tf32 = False
    out = {"gpu": gpu_name(), "dense": run_dense(args), "row_kernels": run_row_kernels(args),
           "model_FinalNet": run_model(args)}
    text = json.dumps(out, indent=1)
    print(text)
    if args.out:
        with open(args.out, "w") as fd:
            fd.write(text)


if __name__ == "__main__":
    main()

"""Time of MaskNet on the kernels against the reference's ops in stock torch eager, and of a zoo.MaskNet training step:

    python tools/masknet_times.py [--reps 20] [--rounds 5] [--out FILE]

Shapes (B 4096, the Criteo-like map of 39 fields x 25,641 rows):
  "serial":   SerialMaskNet at MaskNet_default, embedding 40 (d 1560), dnn_hidden_units [400, 400, 400];
  "parallel": ParallelMaskNet, embedding 16 (d 624), 4 blocks of 64, MLP [400, 400, 400].
Both with the embedding LayerNorm and the blocks' LayerNorm, reduction_ratio 1, no dropout.

For each matmul mode (fp32, tf32x3, tf32, bf16): the dense forward + backward (embedding LayerNorm, mask blocks and
head, from the flattened embedding to the logit: zoo.MaskNet.dense_logit) captured in a CUDA graph and replayed
`--reps` times per round for `--rounds` rounds between CUDA events; the median per call is printed.  The baseline is
the reference's ops (per-field nn.LayerNorm and cat, the blocks' Linears, mul, LayerNorm, ReLU, the head) in torch
eager fp32 on the same GPU, captured and timed the same way.  Each mode's forward output is compared with those ops in
float64 (relative Frobenius error).  The whole fused_train_step is captured (pipeline.TrainPipeline) and replayed.

The block row kernel (b2_mask_row_fwd / _bwd at the serial shape's first block: B 4096, n 400) is timed alone in the
same way; its bytes are counted from the shapes (forward: z read, out written, mean and rstd written, gamma and beta
read; backward: z, g read, dz written, mean, rstd, gamma, beta read) over the measured time.

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
B, FIELDS, VOCAB = 4096, 39, 25641
SHAPES = {
    "serial": dict(embedding_dim=40, dnn_hidden_units=[400, 400, 400], model_type="SerialMaskNet"),
    "parallel": dict(embedding_dim=16, dnn_hidden_units=[400, 400, 400], model_type="ParallelMaskNet",
                     parallel_num_blocks=4, parallel_block_dim=64),
}


def gpu_name():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def graph_replay(fn):
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


def eager_logit(model, emb):
    """MaskNet.forward's dense part op for op in stock torch (the reference's arithmetic), pre-sigmoid."""
    import torch
    import torch.nn.functional as F
    nf = model.num_fields
    feats = emb.view(emb.shape[0], nf, -1)
    hid = torch.cat([model.emb_norm[i](feats[:, i]) for i in range(nf)], dim=1)

    def block(blk, v_in):
        vm = blk.mask_layer(emb)
        z = F.linear(vm * v_in, blk.hidden_layer[0].weight)
        return torch.relu(blk.hidden_layer[1](z))
    net = model.mask_net
    if type(net).__name__ == "SerialMaskNet":
        v = hid
        for blk in net.mask_blocks:
            v = block(blk, v)
        return net.fc[0](v)
    cat = torch.cat([block(blk, hid) for blk in net.mask_blocks], dim=1)
    return torch.nn.Sequential(*list(net.dnn.mlp)[:-1])(cat)


def build(name, mode):
    import torch
    from fuxictr_b200 import functional as F2, zoo
    from fuxictr_b200.schema import FeatureMap
    kw = SHAPES[name]
    specs = [("C%d" % i, {"type": "categorical", "source": "", "padding_idx": 0, "vocab_size": VOCAB})
             for i in range(FIELDS)]
    fm = FeatureMap.from_specs(specs, embedding_dim=kw["embedding_dim"])
    F2.set_matmul_precision(mode)
    torch.manual_seed(5)
    model = zoo.MaskNet(fm, gpu=0, **kw)
    return fm, model


def run_dense(name, args):
    import copy
    import torch
    from fuxictr_b200 import functional as F2
    _, model = build(name, "fp32")
    d = FIELDS * SHAPES[name]["embedding_dim"]
    gen = torch.Generator(device="cuda").manual_seed(8)
    emb = torch.randn(B, d, device="cuda", generator=gen) * 0.1
    eg = emb.clone().requires_grad_(True)
    gout = torch.randn(B, 1, device="cuda", generator=gen)
    m64 = copy.deepcopy(model).double()
    with torch.no_grad():
        y64 = eager_logit(m64, emb.double())

    def fwd_bwd(f):
        def run():
            model.zero_grad(set_to_none=True)
            eg.grad = None
            f(model, eg).backward(gout)
        return run

    def measure(f):
        r = {}
        r["fwd_bwd_us"], r["fwd_bwd_runs"] = timed(graph_replay(fwd_bwd(f)), args.reps, args.rounds)
        with torch.no_grad():
            r["fwd_rel_fro_vs_fp64"] = float("%.3g" % float((f(model, emb).double() - y64).norm() / y64.norm()))
        return r
    results = {"torch_eager_fp32": measure(eager_logit)}
    for mode in MODES:
        F2.set_matmul_precision(mode)
        results[mode] = measure(lambda m, x: m.dense_logit(x))
        results[mode]["speedup"] = round(results["torch_eager_fp32"]["fwd_bwd_us"] / results[mode]["fwd_bwd_us"], 2)
    F2.set_matmul_precision("fp32")
    return results


def run_step(name, args):
    import torch
    from fuxictr_b200 import functional as F2
    from fuxictr_b200.pipeline import TrainPipeline
    gen = torch.Generator().manual_seed(11)
    ids = torch.randint(0, VOCAB, (B, FIELDS), generator=gen).double()
    mat = torch.cat([ids, (torch.rand(B, 1, generator=gen) < 0.25).double()], 1).cuda()
    out = {}
    for mode in MODES:
        _, model = build(name, mode)
        model.use_fused_optimizer()
        pipe = TrainPipeline(model, B, mat.shape[1], graph=False)
        pipe.prime(mat)
        pipe.capture(warmup=3)
        us, runs = timed(lambda: pipe.step_device(mat), args.reps, args.rounds)
        out[mode] = {"step_us": us, "step_runs": runs, "samples_per_s": round(B / (us * 1e-6))}
        del pipe, model
        torch.cuda.empty_cache()
    F2.set_matmul_precision("fp32")
    return out


def run_row_kernel(args):
    import ctypes
    import torch
    from fuxictr_b200 import _lib
    from fuxictr_b200.functional import _ptr, _stream
    n = 400
    gen = torch.Generator(device="cuda").manual_seed(3)
    z = torch.randn(B, n, device="cuda", generator=gen)
    g = torch.randn(B, n, device="cuda", generator=gen)
    gamma, beta = torch.ones(n, device="cuda"), torch.zeros(n, device="cuda")
    out, dz = torch.empty_like(z), torch.empty_like(z)
    mean, rstd = torch.empty(B, device="cuda"), torch.empty(B, device="cuda")
    dgamma, dbeta = torch.zeros(n, device="cuda"), torch.zeros(n, device="cuda")
    null = ctypes.c_void_p(0)

    def fwd():
        _lib.call("b2_mask_row_fwd", _ptr(z), B, n, _ptr(gamma), _ptr(beta), 1e-5, _lib.B2_ACT_RELU, null, 0, 0, 0.0,
                  _ptr(out), n, null, 0, 0, _ptr(mean), _ptr(rstd), _stream())

    def bwd():
        _lib.call("b2_mask_row_bwd", _ptr(z), _ptr(mean), _ptr(rstd), _ptr(gamma), _ptr(beta), _lib.B2_ACT_RELU, null,
                  0, 0, 0.0, _ptr(g), n, B, n, _ptr(dz), null, 0, 0, _ptr(dgamma), _ptr(dbeta), _stream())
    fwd_bytes = 4 * (2 * B * n + 2 * B + 2 * n)
    bwd_bytes = 4 * (3 * B * n + 2 * B + 4 * n)
    res = {}
    for key, fn, nbytes in (("fwd", fwd, fwd_bytes), ("bwd", bwd, bwd_bytes)):
        us, runs = timed(graph_replay(fn), args.reps * 10, args.rounds)
        res[key] = {"us": us, "runs": runs, "bytes": nbytes, "GB_per_s": round(nbytes / (us * 1e-6) / 1e9)}
    return {"shape": {"B": B, "n": n, "act": "relu", "layer_norm": True}, "results": res}


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
        raise SystemExit("masknet_times.py measures on a CUDA device; none is visible")
    torch.backends.cuda.matmul.allow_tf32 = False
    out = {"gpu": gpu_name(), "batch": B}
    for name in SHAPES:
        out[name] = {"config": SHAPES[name], "dense_fwd_bwd": run_dense(name, args),
                     "fused_train_step": run_step(name, args)}
    out["row_kernel"] = run_row_kernel(args)
    text = json.dumps(out, indent=1)
    print(text)
    if args.out:
        with open(args.out, "w") as fd:
            fd.write(text)


if __name__ == "__main__":
    main()

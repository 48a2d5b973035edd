"""Evaluation throughput of row-sharded DLRM at the C5 field layout (bench.py: 26 categorical fields, emb_dim 16,
top MLP [64, 64, 64]), and the evaluation lookup beside the training push at the same shape:

    python tools/sharded_eval_times.py [--world 8] [--batch-local 8192] [--rounds 4] [--vocab-scale 0.1] [--reps 5]
    python -m torch.distributed.run --nproc-per-node N tools/sharded_eval_times.py      # real ranks

Without torchrun, `--world` virtual ranks share one GPU (sharded.VirtualPeerGroup, driven by
sharded.lockstep_evaluate), so the rate is that of one GPU doing every rank's work.  Under torchrun each process is
a real rank on its own GPU (SymmPeerGroup, RankModel.evaluate).  The validation split has
rounds * batch_local * world + 3 rows (a ragged last round).  Times come from CUDA events around whole
evaluate() calls (which end in a device-to-host copy) after one warm-up call; the kernel times are CUDA events
over `--kernel-reps` launches of every rank's lookup / push.  One JSON line, with the card's name and power limit.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

HERE = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, HERE)


def gpu_name():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        return "unknown"


def make_model(fm, device_index):
    import torch
    import bench
    from fuxictr_b200 import zoo
    torch.manual_seed(2019)
    return zoo.DLRM(fm, gpu=device_index, embedding_dim=bench.DIM, top_mlp_units=bench.DLRM_TOP,
                    interaction_op="dot")


def events_ms(fn, reps):
    import torch
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--world", type=int, default=8, help="virtual ranks (ignored under torchrun)")
    ap.add_argument("--batch-local", type=int, default=8192)
    ap.add_argument("--rounds", type=int, default=4, help="full rounds of the validation split (+ a 3-row tail)")
    ap.add_argument("--vocab-scale", type=float, default=0.1, help="scale of the C5 cardinalities (1.0: ~200 M rows)")
    ap.add_argument("--reps", type=int, default=5, help="timed evaluate() calls")
    ap.add_argument("--kernel-reps", type=int, default=20)
    ap.add_argument("--precision", default="tf32x3", choices=["tf32x3", "fp32"])
    args = ap.parse_args()

    import torch
    import bench
    from fuxictr_b200 import sharded as SH, functional as F2
    from fuxictr_b200.dataloader import MatrixDataLoader
    from fuxictr_b200.schema import FeatureMap
    import __graft_entry__
    real = "WORLD_SIZE" in os.environ
    if real:
        import torch.distributed as dist
        rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
        torch.cuda.set_device(local)
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
        if rank == 0:
            __graft_entry__.build()
        dist.barrier()
    else:
        rank, world, local = 0, args.world, 0
        torch.cuda.set_device(0)
        __graft_entry__.build()
    card = gpu_name()
    F2.set_matmul_precision(args.precision)
    ns = argparse.Namespace(workload="dlrm", vocab_scale=args.vocab_scale)
    specs = bench.make_specs(ns)
    fm = FeatureMap.from_specs(specs, embedding_dim=bench.DIM)
    B = args.batch_local
    n = args.rounds * B * world + 3
    data = bench.make_batches(1, n, seed=1000, specs=specs)[0].numpy()
    W = fm.input_length + 1

    if real:
        groups = [SH.SymmPeerGroup()]
    else:
        registry = {}
        groups = [SH.VirtualPeerGroup(r, world, registry) for r in range(world)]
    models = []
    for g in groups:
        m = make_model(fm, local)
        m.enable_sharding(g, B, W, torch.float64, want_fm=False)
        with torch.no_grad():         # rows of a trained scale, so that the predictions are not all one value
            for t in m._sharded_front.distinct_tables():
                t.normal_(0, 0.1)
        models.append(m)
    ranks = [rank] if real else list(range(world))
    loaders = [MatrixDataLoader(fm, data, batch_size=B, shard=(r, world), drop_last=False) for r in ranks]

    if real:
        def evaluate():
            return models[0].evaluate(loaders[0], ["logloss", "AUC"])
    else:
        def evaluate():
            return SH.lockstep_evaluate(models, loaders, ["logloss", "AUC"])[0]
    metrics = evaluate()                                   # warm-up: plans, allocator, first launches
    times = []
    for _ in range(args.reps):
        times.append(events_ms(evaluate, 1))
    ms = statistics.median(times)

    # the lookup beside the training push, full batches on every rank (the same candidates); all ranks' launches
    fronts = [m._sharded_front for m in models]
    mats = [torch.from_numpy(data[r * B:(r + 1) * B]).cuda() for r in ranks]
    barrier = (lambda: groups[0].barrier()) if real else (lambda: None)
    for fr, mat in zip(fronts, mats):
        fr.phase_ids(mat)
    barrier()
    push_ms = events_ms(lambda: [fr.phase_push() for fr in fronts], args.kernel_reps) / len(fronts)
    barrier()
    for fr, mat in zip(fronts, mats):
        fr.eval_phase_ids(mat)
    barrier()
    lookup_ms = events_ms(lambda: [fr.eval_phase_lookup() for fr in fronts], args.kernel_reps) / len(fronts)
    barrier()

    out = {"gpu": card, "precision": args.precision, "mode": "real ranks" if real else "virtual ranks on one GPU",
           "world": world, "batch_local": B, "fields": len(specs), "emb_dim": bench.DIM,
           "vocab_scale": args.vocab_scale, "table_rows": sum(sp["vocab_size"] for _, sp in specs),
           "validation_rows": n, "evaluate_ms_median": round(ms, 2), "evaluate_ms_runs": [round(t, 2) for t in times],
           "eval_samples_per_s": round(n / (ms / 1e3)), "logloss": metrics["logloss"], "AUC": metrics["AUC"],
           "lookup_us_per_rank_launch": round(lookup_ms * 1e3, 1),
           "train_push_us_per_rank_launch": round(push_ms * 1e3, 1)}
    if real:
        out["rank"] = rank
        if rank == 0:
            print(json.dumps(out), flush=True)
        dist.barrier()
        dist.destroy_process_group()
    else:
        out["real_ranks"] = "not measured (launch under torchrun on a machine with several GPUs)"
        print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()

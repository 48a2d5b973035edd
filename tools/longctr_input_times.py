"""The LongCTR input path on the GPU: the reference's collator against the HBM store, at ETA_default's shape (B 8192,
L 50) and a long shape (B 4096, L 1024), with three item columns and one user field.

A seeded synthetic dataset is written to a temporary directory per shape: 20 000 users with histories of 0 to 2 L
items, a 500 000-row item_info, and batches_per_epoch full batches of samples whose seq_len runs past L for most rows
(so nearly every batch is padded to L = max_len, as on real data).

Times:
  - b2_longctr_collate alone (CUDA events around graph replays of 20 launches, median of the repeats), with TB/s
    from the bytes it must move: the mask and the C int64 item columns written, the kept history ids, the C int32
    item_info values per slot and the three batch values read;
  - the reference's collator alone (model_zoo/LongCTR/longctr_dataloader.py, which oracle/install_longctr_ref.py
    copies to oracle/_ref during build(); num_workers as given; keras pad_sequences replaced by the keras-semantics
    stand-in of tests/golden/make_longctr_loader_golden.py): host seconds per batch, and the per-feature pageable
    `.to(device)` of one of its triples;
  - whole epochs of fused_train_step in samples/s for ETA and TWIN, three ways: (1) the reference's collator with the
    model's per-feature `.to(device)`, (2) LongCTRDataLoader eager, (3) LongCTRPipeline with the captured step.  Each
    epoch is run twice and the second is timed (host clock around the epoch, ending in a synchronise).
Without oracle/_ref's longctr_dataloader.py the reference arms are skipped with a message.  Prints one JSON object,
with the card's name and power limit read in the same run.

    python tools/longctr_input_times.py [--batches-per-epoch 6] [--repeats 50] [--num-workers 3]
"""
import argparse
import importlib.util
import json
import os
import shutil
import sys
import tempfile
import time
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from longctr_times import card, timed  # noqa: E402

REF_LOADER = os.path.join(ROOT, "oracle", "_ref", "extras", "model_zoo", "LongCTR", "longctr_dataloader.py")
SHAPES = {"ETA_default": dict(batch=8192, L=50), "long": dict(batch=4096, L=1024)}
MODELS = {"ETA": dict(embedding_dim=4, dnn_hidden_units=[64, 32], attention_dim=64, num_heads=2, hash_bits=32,
                      topk=50, reuse_hash=True, short_seq_len=50),
          "TWIN": dict(embedding_dim=4, dnn_hidden_units=[64, 32], attention_dim=64, num_heads=2, topk=50,
                       short_seq_len=50)}
N_USERS, N_ITEMS = 20000, 500000
FEATURES = [("user_index", {"type": "meta"}), ("item_index", {"type": "meta"}), ("seq_len", {"type": "meta"}),
            ("user_id", {"type": "categorical", "source": "user", "padding_idx": 0, "vocab_size": N_USERS + 1}),
            ("item_id", {"type": "categorical", "source": "item", "padding_idx": 0, "vocab_size": N_ITEMS}),
            ("cate_id", {"type": "categorical", "source": "item", "padding_idx": 0, "vocab_size": 5000}),
            ("brand_id", {"type": "categorical", "source": "item", "padding_idx": 0, "vocab_size": 50000})]


def write_dataset(out, B, L, batches, seed=0):
    import pandas as pd
    rng = np.random.default_rng(seed)
    lens = rng.integers(0, 2 * L + 1, N_USERS)
    flat = rng.integers(1, N_ITEMS, int(lens.sum()))
    bounds = np.concatenate([[0], np.cumsum(lens)])
    pd.DataFrame({"full_item_seq": [flat[bounds[u]:bounds[u + 1]] for u in range(N_USERS)]}).to_parquet(
        os.path.join(out, "user_info.parquet"))
    ids = np.arange(N_ITEMS, dtype=np.int64)
    pd.DataFrame({"item_index": ids, "item_id": ids, "cate_id": ids % 4999 + 1,
                  "brand_id": ids % 49999 + 1}).to_parquet(os.path.join(out, "item_info.parquet"))
    n = B * batches
    users = rng.integers(0, N_USERS, n)
    pd.DataFrame({"user_index": users, "item_index": rng.integers(1, N_ITEMS, n), "seq_len": rng.integers(0, 2 * L, n),
                  "user_id": users + 1, "label": (rng.random(n) < 0.3).astype(np.int64)}).to_parquet(
        os.path.join(out, "train.parquet"))
    return os.path.join(out, "train.parquet"), os.path.join(out, "user_info.parquet"), os.path.join(out,
                                                                                                   "item_info.parquet")


def reference_loader_class():
    if not os.path.exists(REF_LOADER):
        return None
    sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
    from make_longctr_loader_golden import pad_sequences
    for name in ("keras_preprocessing", "keras_preprocessing.sequence"):
        sys.modules.setdefault(name, types.ModuleType(name))
    sys.modules["keras_preprocessing.sequence"].pad_sequences = pad_sequences
    sys.modules["keras_preprocessing"].sequence = sys.modules["keras_preprocessing.sequence"]
    spec = importlib.util.spec_from_file_location("ref_longctr_dataloader", REF_LOADER)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod.LongCTRDataLoader


def collate_bytes(loader, mat, L):
    """Bytes b2_longctr_collate must move for one batch."""
    B, C = mat.shape[0], len(loader.item_columns)
    users, seq = mat[:, loader.cols[0]].numpy(), mat[:, loader.cols[2]].numpy()
    kept = np.minimum(np.minimum(seq, np.diff(loader.store.offsets)[users]), L).sum()
    return 4 * B * L + 8 * C * B * (L + 1) + 4 * int(kept) + 4 * C * B * (L + 1) + 3 * 8 * B


def kernel_us(loader, dev, L, repeats, launches=20):
    """b2_longctr_collate alone: `launches` launches into preallocated outputs captured into one graph, timed as
    replays (so the host's allocation and call overhead stays out), per launch."""
    mask = torch.empty((dev.shape[0], L), dtype=torch.float32, device=dev.device)
    items = torch.empty((len(loader.item_columns), dev.shape[0] * (L + 1)), dtype=torch.int64, device=dev.device)
    loader.store.collate(dev, L, loader.cols, loader.padding, mask, items)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        for _ in range(launches):
            loader.store.collate(dev, L, loader.cols, loader.padding, mask, items)
    return timed(graph.replay, repeats) / launches


def model_of(name, fm):
    from fuxictr_b200 import zoo
    torch.manual_seed(1)
    model = getattr(zoo, name)(fm, gpu=0, **MODELS[name])
    model.train()
    model.use_fused_optimizer()
    return model


def epoch_rate(run, n):
    run()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    run()
    torch.cuda.synchronize()
    return n / (time.perf_counter() - t0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches-per-epoch", type=int, default=6)
    ap.add_argument("--repeats", type=int, default=50)
    ap.add_argument("--num-workers", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tools/longctr_input_times.py measures on the GPU and found none")
    import __graft_entry__
    __graft_entry__.build()
    from fuxictr_b200 import functional as F2
    from fuxictr_b200.longctr_data import LongCTRDataLoader
    from fuxictr_b200.pipeline import LongCTRPipeline
    from fuxictr_b200.schema import FeatureMap
    F2.set_matmul_precision("tf32x3")
    RefLoader = reference_loader_class()
    out = {"card": card(), "matmul": "tf32x3", "batches_per_epoch": args.batches_per_epoch,
           "num_workers_reference": args.num_workers}
    if RefLoader is None:
        out["reference"] = "skipped: %s is missing (build() installs it)" % REF_LOADER
        print(out["reference"], file=sys.stderr)
    for shape, s in SHAPES.items():
        B, L = s["batch"], s["L"]
        tmp = tempfile.mkdtemp(prefix="longctr_input_")
        try:
            data, users, items = write_dataset(tmp, B, L, args.batches_per_epoch)
            fm = FeatureMap.from_specs(FEATURES, embedding_dim=4)
            loader = LongCTRDataLoader(fm, data, users, items, batch_size=B, shuffle=True, max_len=L)
            res = {"batch": B, "max_len": L, "samples": loader.num_samples}
            torch.manual_seed(3)
            mat, Lb = next(iter(loader.matrices()))
            mat = mat.clone()
            dev = mat.cuda()
            us = kernel_us(loader, dev, Lb, args.repeats)
            nbytes = collate_bytes(loader, mat, Lb)
            res["collate_kernel"] = {"L": Lb, "us": round(us, 2), "MB": round(nbytes / 1e6, 2),
                                     "TB_s": round(nbytes / us / 1e6, 3)}
            if RefLoader is not None:
                ref = RefLoader(fm, data, users, items, batch_size=B, shuffle=True, num_workers=args.num_workers,
                                max_len=L)
                t0 = time.perf_counter()
                nb = 0
                for triple in ref:
                    nb += 1
                res["reference_collate_s_per_batch"] = round((time.perf_counter() - t0) / nb, 4)
                bd, idict, mask = triple
                h2d_bytes = sum(v.numel() * v.element_size() for v in list(idict.values()) + [mask]) + \
                    sum(v.numel() * v.element_size() for v in bd.values())

                def h2d():
                    for v in list(bd.values()) + list(idict.values()) + [mask]:
                        v.to("cuda")
                res["reference_h2d"] = {"MB": round(h2d_bytes / 1e6, 1), "ms": round(timed(h2d, 10) / 1000, 2)}
            for name in MODELS:
                rates = {}
                model = model_of(name, fm)
                if RefLoader is not None:
                    def run_ref():
                        for triple in ref:
                            model.fused_train_step(triple)
                    rates["reference_collator"] = round(epoch_rate(run_ref, loader.num_samples))

                def run_eager():
                    for triple in loader:
                        model.fused_train_step(triple)
                rates["loader_eager"] = round(epoch_rate(run_eager, loader.num_samples))
                pipe = LongCTRPipeline(model_of(name, fm), loader, graph=True)
                rates["pipeline_graph"] = round(epoch_rate(pipe.epoch, loader.num_samples))
                res[name + "_samples_per_s"] = rates
                del model, pipe
                torch.cuda.empty_cache()
            out[shape] = res
            print(json.dumps({shape: res}), file=sys.stderr)
        finally:
            shutil.rmtree(tmp, ignore_errors=True)
    print(json.dumps(out))


if __name__ == "__main__":
    main()

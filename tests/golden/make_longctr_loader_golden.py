"""Generates the LongCTR data-loader fixtures by running the REAL reference collator
(model_zoo/LongCTR/longctr_dataloader.py, imported by path).  Run in the build container only:

    python tests/golden/make_longctr_loader_golden.py

1. writes a small SEEDED synthetic LongCTR dataset under tests/golden/data/syn_longctr/: train.parquet and
   valid.parquet (columns label, user_index, timestamp, item_index, user_id, seq_len: the file order is not the
   feature map's, and timestamp is no feature), user_info.parquet (full_item_seq, 30 users, histories of 0 to 40 items
   with a few 0 ids inside), item_info.parquet (item_index, item_id, cate_id, brand_id; row 0 is not zeros) and
   feature_map.json;
2. runs the reference's LongCTRDataLoader (num_workers=0, torch.manual_seed(7) before iterating) over every case in
   CASES and writes tests/golden/longctr_loader_<case>.npz: "meta" (JSON: the case, num_samples, num_batches, the
   batch_dict and item_dict keys) and, for batch i, i/L, i/mask, i/bd/<column>, i/item/<column>.

The train split's seq_len values run from 0 to 50 (beyond every stored history), except rows 96-127, whose seq_len
stays at or below 6: unshuffled with batch 32 and max_len 12 that batch is padded to L < max_len.

keras_preprocessing is not installed, so `pad_sequences` below stands in for
keras_preprocessing.sequence.pad_sequences: keras's semantics for the arguments the collator passes (value 0,
padding = truncating in {pre, post}, int32 output); tests/test_longctr_loader_host.py pins it to keras's documented
examples.
"""
import importlib.util
import json
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
DATA = os.path.join(HERE, "data", "syn_longctr")
REF = os.environ.get("FUXICTR_REFERENCE", "/root/reference")

N_USERS, N_ITEMS, MAX_HIST = 30, 120, 40
FEATURES = [("user_index", {"type": "meta"}), ("item_index", {"type": "meta"}), ("seq_len", {"type": "meta"}),
            ("user_id", {"type": "categorical", "source": "user", "padding_idx": 0, "vocab_size": N_USERS + 1}),
            ("item_id", {"type": "categorical", "source": "item", "padding_idx": 0, "vocab_size": N_ITEMS}),
            ("cate_id", {"type": "categorical", "source": "item", "padding_idx": 0, "vocab_size": 15}),
            ("brand_id", {"type": "categorical", "source": "item", "padding_idx": 0, "vocab_size": 20})]
ONE_ITEM_COLUMN = ["user_index", "item_index", "seq_len", "user_id", "item_id"]
# name -> (split, batch_size, shuffle, max_len, padding, features kept (None: all))
CASES = {
    "train_pre_shuffled_ml12": ("train", 32, True, 12, "pre", None),
    "train_pre_unshuffled_ml12": ("train", 32, False, 12, "pre", None),
    "train_post_unshuffled_ml64": ("train", 48, False, 64, "post", None),
    "train_post_shuffled_ml20_one_col": ("train", 40, True, 20, "post", ONE_ITEM_COLUMN),
    "valid_pre_unshuffled_ml64_one_col": ("valid", 16, False, 64, "pre", ONE_ITEM_COLUMN),
}


def pad_sequences(sequences, maxlen=None, dtype="int32", padding="pre", truncating="pre", value=0.0):
    """keras_preprocessing.sequence.pad_sequences for 1-D integer sequences: an (n, maxlen) array filled with
    `value`; each non-empty sequence is truncated to its last (truncating "pre") or first ("post") maxlen items and
    written right-aligned (padding "pre") or left-aligned ("post").  maxlen None: the longest sequence."""
    if padding not in ("pre", "post") or truncating not in ("pre", "post"):
        raise ValueError("padding and truncating must be 'pre' or 'post'")
    lengths = [len(s) for s in sequences]
    if maxlen is None:
        maxlen = max(lengths) if lengths else 0
    x = np.full((len(sequences), maxlen), value, dtype=dtype)
    for i, s in enumerate(sequences):
        if not len(s):
            continue
        trunc = np.asarray(s[-maxlen:] if truncating == "pre" else s[:maxlen], dtype=dtype)
        if padding == "post":
            x[i, :len(trunc)] = trunc
        else:
            x[i, -len(trunc):] = trunc
    return x


def write_dataset():
    import pandas as pd
    rng = np.random.default_rng(20251019)
    os.makedirs(DATA, exist_ok=True)
    blob = {"dataset_id": "syn_longctr", "num_fields": 4, "total_features": sum(s.get("vocab_size", 0)
                                                                              for _, s in FEATURES),
            "input_length": len(FEATURES), "labels": ["label"], "features": [{k: s} for k, s in FEATURES]}
    with open(os.path.join(DATA, "feature_map.json"), "w") as fd:
        json.dump(blob, fd, indent=1)
    seqs = []
    for u in range(N_USERS):
        n = 0 if u in (3, 17) else int(rng.integers(1, MAX_HIST + 1))
        s = rng.integers(1, N_ITEMS, n)
        if n > 4 and u % 5 == 0:
            s[rng.integers(0, n, 2)] = 0            # a padding id inside a stored history: masked by value
        seqs.append(s.astype(np.int64))
    seqs[7] = rng.integers(1, N_ITEMS, MAX_HIST).astype(np.int64)      # one history of the longest length
    pd.DataFrame({"full_item_seq": [list(s) for s in seqs]}).to_parquet(os.path.join(DATA, "user_info.parquet"))
    ids = np.arange(N_ITEMS, dtype=np.int64)
    items = pd.DataFrame({"item_index": ids, "item_id": ids, "cate_id": ids % 14 + 1, "brand_id": (ids * 7) % 19 + 1})
    items.loc[0, ["item_id", "cate_id", "brand_id"]] = [5, 3, 11]     # row 0 (what padding slots copy) is not zeros
    items.to_parquet(os.path.join(DATA, "item_info.parquet"))
    for split, n in (("train", 203), ("valid", 61)):
        users = rng.integers(0, N_USERS, n)
        seq_len = rng.integers(0, 51, n)
        if split == "train":
            seq_len[96:128] = rng.integers(0, 7, 32)
        seq_len[rng.integers(0, n, 5)] = 0
        df = pd.DataFrame({"label": (rng.random(n) < 0.3).astype(np.int64), "user_index": users,
                           "timestamp": rng.integers(1_600_000_000, 1_700_000_000, n),
                           "item_index": rng.integers(1, N_ITEMS, n), "user_id": users + 1, "seq_len": seq_len})
        df.to_parquet(os.path.join(DATA, split + ".parquet"))


def reference_loader_class():
    """The reference's longctr_dataloader.py with `pad_sequences` taken from the stand-in above."""
    for name in ["h5py", "polars", "keras_preprocessing", "keras_preprocessing.sequence"]:
        sys.modules.setdefault(name, types.ModuleType(name))
    sys.modules["keras_preprocessing.sequence"].pad_sequences = pad_sequences
    sys.modules["keras_preprocessing"].sequence = sys.modules["keras_preprocessing.sequence"]
    sys.path.insert(0, REF)
    spec = importlib.util.spec_from_file_location(
        "longctr_dataloader", os.path.join(REF, "model_zoo", "LongCTR", "longctr_dataloader.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    from fuxictr.features import FeatureMap
    return mod.LongCTRDataLoader, FeatureMap


def write_goldens():
    import torch
    Loader, FeatureMap = reference_loader_class()
    for case, (split, batch_size, shuffle, max_len, padding, keep) in CASES.items():
        fm = FeatureMap("syn_longctr", DATA)
        fm.load(os.path.join(DATA, "feature_map.json"), {"use_features": keep} if keep else {})
        loader = Loader(fm, os.path.join(DATA, split), os.path.join(DATA, "user_info.parquet"),
                        os.path.join(DATA, "item_info.parquet"), batch_size=batch_size, shuffle=shuffle,
                        num_workers=0, max_len=max_len, padding=padding)
        torch.manual_seed(7)
        arrays, bd_keys, item_keys = {}, None, None
        for i, (bd, items, mask) in enumerate(loader):
            bd_keys, item_keys = list(bd), list(items)
            arrays["%d/L" % i] = np.array(mask.shape[1])
            arrays["%d/mask" % i] = mask.numpy()
            for k, v in bd.items():
                arrays["%d/bd/%s" % (i, k)] = v.numpy()
            for k, v in items.items():
                arrays["%d/item/%s" % (i, k)] = v.numpy()
        meta = {"case": case, "split": split, "batch_size": batch_size, "shuffle": shuffle, "max_len": max_len,
                "padding": padding, "features": keep, "num_samples": loader.num_samples,
                "num_batches": len(loader), "batch_keys": bd_keys, "item_keys": item_keys}
        arrays["meta"] = np.array(json.dumps(meta))
        path = os.path.join(HERE, "longctr_loader_%s.npz" % case)
        np.savez_compressed(path, **arrays)
        print("wrote", path, "%.1f KB" % (os.path.getsize(path) / 1024))


if __name__ == "__main__":
    write_dataset()
    write_goldens()

"""The LongCTR data loader without a GPU: batch order, len(), each batch's L and host batch_dict against the
reference collator's goldens; a numpy restatement of b2_longctr_collate against the goldens' item columns and masks;
the construction refusals; RankDataLoader routing; the keras pad_sequences stand-in the goldens were made with; and the
C-ABI checks of b2_longctr_collate."""
import ctypes
import json
import os
import shutil
import sys

import numpy as np
import pytest
import torch

from conftest import GOLDEN

sys.path.insert(0, GOLDEN)
import make_longctr_loader_golden as MK  # noqa: E402
from fuxictr_b200 import _lib  # noqa: E402
from fuxictr_b200.dataloader import RankDataLoader  # noqa: E402
from fuxictr_b200.longctr_data import LongCTRDataLoader  # noqa: E402
from fuxictr_b200.schema import FeatureMap  # noqa: E402

DATA = os.path.join(GOLDEN, "data", "syn_longctr")


def load_golden(case):
    blob = np.load(os.path.join(GOLDEN, "longctr_loader_%s.npz" % case))
    meta = json.loads(str(blob["meta"]))
    batches = []
    for i in range(meta["num_batches"]):
        batches.append({"L": int(blob["%d/L" % i]), "mask": blob["%d/mask" % i],
                        "bd": {k: blob["%d/bd/%s" % (i, k)] for k in meta["batch_keys"]},
                        "item": {k: blob["%d/item/%s" % (i, k)] for k in meta["item_keys"]}})
    return meta, batches


def feature_map(keep=None, embedding_dim=None):
    params = {"embedding_dim": embedding_dim}
    if keep:
        params["use_features"] = keep
    fm = FeatureMap("syn_longctr", DATA)
    fm.load(os.path.join(DATA, "feature_map.json"), params)
    return fm


def make_loader(case, data_dir=DATA, **over):
    split, batch_size, shuffle, max_len, padding, keep = MK.CASES[case]
    kw = dict(batch_size=batch_size, shuffle=shuffle, max_len=max_len, padding=padding)
    kw.update(over)
    return LongCTRDataLoader(feature_map(keep), os.path.join(data_dir, split), os.path.join(data_dir, "user_info.parquet"),
                             os.path.join(data_dir, "item_info.parquet"), **kw)


def collate_numpy(store, mat, L, cols, padding):
    """b2_longctr_collate restated over numpy (its header comment): the reference's semantics as the kernel forms them."""
    B = mat.shape[0]
    ids = np.zeros((B, L + 1), dtype=np.int64)
    for b in range(B):
        u, t, s = (int(mat[b, c]) for c in cols)
        o = store.offsets[u]
        n = min(s, int(store.offsets[u + 1] - o))
        k = min(n, L)
        kept = store.hist[o + (n - k if padding == "pre" else 0):][:k]
        if k:
            if padding == "pre":
                ids[b, L - k:L] = kept
            else:
                ids[b, :k] = kept
        ids[b, L] = t
    return (ids[:, :L] > 0).astype(np.float32), store.table[ids.reshape(-1)].T.astype(np.int64)


@pytest.mark.parametrize("case", list(MK.CASES))
def test_host_batches_match_reference_collator(case):
    meta, batches = load_golden(case)
    loader = make_loader(case)
    assert (loader.num_samples, loader.num_batches, len(loader), loader.num_blocks) == \
        (meta["num_samples"], meta["num_batches"], meta["num_batches"], 1)
    assert loader.batch_columns == meta["batch_keys"] and loader.item_columns == meta["item_keys"]
    torch.manual_seed(7)
    got = [(m.clone(), L) for m, L in loader.matrices()]
    assert len(got) == len(batches)
    for (mat, L), ref in zip(got, batches):
        assert L == ref["L"]
        bd = loader.batch_dict(mat)
        assert list(bd) == meta["batch_keys"]
        for k, v in ref["bd"].items():
            assert bd[k].dtype == torch.from_numpy(v).dtype and np.array_equal(bd[k].numpy(), v), k
        mask, items = collate_numpy(loader.store, mat.numpy(), L, loader.cols, loader.padding)
        assert np.array_equal(mask, ref["mask"])
        for c, k in enumerate(meta["item_keys"]):
            assert np.array_equal(items[c], ref["item"][k]), k


def test_goldens_cover_the_cases_the_loader_must_handle():
    """Cases: shuffled and not, pre and post, max_len below and above the longest history, a batch size that does not
    divide N, seq_len beyond the stored history and 0, row 0 of item_info non-zero, one and three item columns, and
    batches padded to L < max_len."""
    loader = make_loader("train_pre_unshuffled_ml12")
    st = loader.store
    longest = int(np.diff(st.offsets).max())
    mls = [MK.CASES[c][3] for c in MK.CASES]
    assert min(mls) < longest < max(mls)
    assert any(MK.CASES[c][0] == "train" and 203 % MK.CASES[c][1] for c in MK.CASES)
    hist_len = np.diff(st.offsets)[loader.matrix.numpy()[:, loader.cols[0]]]
    assert (loader._seq > hist_len).any() and (loader._seq == 0).any()
    assert (st.table[0] != 0).all()
    assert {len(load_golden(c)[0]["item_keys"]) for c in MK.CASES} == {1, 3}
    assert any(b["L"] < MK.CASES["train_pre_unshuffled_ml12"][3] for b in load_golden("train_pre_unshuffled_ml12")[1])


def test_rank_data_loader_routes_to_the_longctr_loader():
    fm = feature_map()
    rdl = RankDataLoader(fm, stage="train", train_data=os.path.join(DATA, "train"),
                         valid_data=os.path.join(DATA, "valid"), batch_size=32, shuffle=True, data_format="parquet",
                         data_loader=LongCTRDataLoader, user_info=os.path.join(DATA, "user_info.parquet"),
                         item_info=os.path.join(DATA, "item_info.parquet"), max_len=12, padding="pre", num_workers=3,
                         gpu=0)
    train, valid = rdl.make_iterator()
    assert isinstance(train, LongCTRDataLoader) and isinstance(valid, LongCTRDataLoader)
    assert train.shuffle and not valid.shuffle
    assert (len(train), len(valid), train.max_len, valid.padding) == (7, 2, 12, "pre")


# ------------------------------------------------------------------ refusals
def _copy_data(tmp_path):
    dst = tmp_path / "syn_longctr"
    shutil.copytree(DATA, dst)
    return str(dst)


def _rewrite(path, fn):
    import pandas as pd
    df = pd.read_parquet(path)
    fn(df)
    df.to_parquet(path)


@pytest.mark.parametrize("what,edit,message", [
    ("user_index", lambda df: df.__setitem__("user_index", df["user_index"].where(df.index != 5, 30)), "user_index"),
    ("user_index", lambda df: df.__setitem__("user_index", df["user_index"].where(df.index != 5, -1)), "user_index"),
    ("item_index", lambda df: df.__setitem__("item_index", df["item_index"].where(df.index != 9, 120)), "item_index"),
    ("seq_len", lambda df: df.__setitem__("seq_len", df["seq_len"].where(df.index != 2, -3)), "seq_len"),
    ("float", lambda df: df.__setitem__("label", df["label"].astype(np.float64)), "integer"),
])
def test_data_file_refusals(tmp_path, what, edit, message):
    d = _copy_data(tmp_path)
    _rewrite(os.path.join(d, "train.parquet"), edit)
    with pytest.raises(ValueError, match=message):
        make_loader("train_pre_shuffled_ml12", data_dir=d)


@pytest.mark.parametrize("bad", [120, -2, 1 << 31])
def test_history_ids_out_of_range_are_refused(tmp_path, bad):
    import pandas as pd
    d = _copy_data(tmp_path)
    path = os.path.join(d, "user_info.parquet")
    seqs = list(pd.read_parquet(path)["full_item_seq"].map(list))
    seqs[4] = seqs[4] + [bad]
    pd.DataFrame({"full_item_seq": seqs}).to_parquet(path)
    with pytest.raises(ValueError, match="history item ids"):
        make_loader("train_pre_shuffled_ml12", data_dir=d)


def test_item_column_refusals(tmp_path):
    d = _copy_data(tmp_path)
    path = os.path.join(d, "item_info.parquet")
    _rewrite(path, lambda df: df.__setitem__("cate_id", [[1, 2]] * len(df)))
    with pytest.raises(NotImplementedError, match="list-valued"):
        make_loader("train_pre_shuffled_ml12", data_dir=d)
    _rewrite(path, lambda df: df.__setitem__("cate_id", np.linspace(0, 1, len(df))))
    with pytest.raises(ValueError, match="integer"):
        make_loader("train_pre_shuffled_ml12", data_dir=d)


def test_padding_mode_and_max_len_refusals():
    with pytest.raises(ValueError, match="padding"):
        make_loader("train_pre_shuffled_ml12", padding="middle")
    with pytest.raises(ValueError, match="max_len"):
        make_loader("train_pre_shuffled_ml12", max_len=0)


# ------------------------------------------------------------------ the keras stand-in
def test_pad_sequences_stand_in_matches_keras_documented_examples():
    seq = [[1], [2, 3], [4, 5, 6]]
    out = MK.pad_sequences(seq)
    assert out.dtype == np.int32 and out.tolist() == [[0, 0, 1], [0, 2, 3], [4, 5, 6]]
    assert MK.pad_sequences(seq, padding="post").tolist() == [[1, 0, 0], [2, 3, 0], [4, 5, 6]]
    assert MK.pad_sequences(seq, maxlen=2).tolist() == [[0, 1], [2, 3], [5, 6]]
    assert MK.pad_sequences(seq, maxlen=2, truncating="post").tolist() == [[0, 1], [2, 3], [4, 5]]
    assert MK.pad_sequences([[], [7]], maxlen=3, padding="post", truncating="post").tolist() == [[0, 0, 0], [7, 0, 0]]
    assert MK.pad_sequences([[]], maxlen=0).shape == (1, 0)


# ------------------------------------------------------------------ C-ABI
@pytest.fixture(scope="module")
def lib():
    import __graft_entry__
    __graft_entry__.build()
    return _lib.load()


def test_collate_is_declared_bound_and_exported(lib):
    from test_abi import header_prototypes
    assert header_prototypes()["b2_longctr_collate"] == len(_lib.SIGNATURES["b2_longctr_collate"][1]) == 18
    assert hasattr(ctypes.CDLL(_lib.LIB_PATH), "b2_longctr_collate")


def test_collate_rejects_bad_arguments_without_a_gpu(lib):
    p, z = ctypes.c_void_p(256), None

    def call(batch=p, dtype=_lib.B2_I64, rows=8, stride=6, cu=1, ci=3, cs=5, off=p, hist=p, users=30, info=p,
             items_n=120, C=3, L=12, pad=_lib.B2_LONGCTR_PAD_PRE, mask=p, out=p):
        return lib.b2_longctr_collate(batch, dtype, rows, stride, cu, ci, cs, off, hist, users, info, items_n, C, L,
                                      pad, mask, out, None)

    for kw in (dict(batch=z), dict(off=z), dict(hist=z), dict(info=z), dict(out=z), dict(mask=z)):
        assert call(**kw) == -1 and b"NULL" in lib.b2_last_error(), kw
    assert call(dtype=_lib.B2_F64) == -1 and b"int64 or int32" in lib.b2_last_error()
    assert call(pad=2) == -1 and b"padding" in lib.b2_last_error()
    assert call(L=-1) == -1 and call(L=_lib.B2_LONGCTR_MAX_LEN + 1) == -1 and b"L =" in lib.b2_last_error()
    assert call(C=0) == -1 and call(C=_lib.B2_LONGCTR_MAX_COLS + 1) == -1 and b"item columns" in lib.b2_last_error()
    assert call(cs=6) == -1 and call(cu=-1) == -1 and b"outside a row" in lib.b2_last_error()
    assert call(rows=-1) == -1 and call(rows=1 << 31) == -1 and b"rows" in lib.b2_last_error()
    assert call(users=0) == -1 and call(items_n=0) == -1 and b"empty store" in lib.b2_last_error()
    assert call(rows=0) == 0                            # nothing to write: no launch
    assert call(rows=0, mask=z, L=0) == 0               # L = 0 needs no mask

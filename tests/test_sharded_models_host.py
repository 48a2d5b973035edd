"""Row-sharded DCNv2, xDeepFM and DIN without a GPU: which inputs the sharded front refuses (before a table is
sharded, a buffer allocated or a kernel called), the slot layout of sequence fields, and the int32 bounds."""
import pytest
import torch

from fuxictr_b200 import zoo, sharded as SH
from fuxictr_b200.schema import FeatureMap

_CAT = [("C%d" % i, {"type": "categorical", "source": "", "padding_idx": 0, "vocab_size": 11 + 3 * i})
        for i in range(5)]
_SEQ = [
    ("user", {"type": "categorical", "source": "", "padding_idx": 0, "vocab_size": 30}),
    ("item_id", {"type": "categorical", "source": "", "padding_idx": 0, "vocab_size": 50}),
    ("cate_id", {"type": "categorical", "source": "", "padding_idx": 0, "vocab_size": 12}),
    ("click_history", {"type": "sequence", "source": "", "padding_idx": 0, "vocab_size": 50, "max_len": 6,
                       "share_embedding": "item_id"}),
    ("cate_history", {"type": "sequence", "source": "", "padding_idx": 0, "vocab_size": 12, "max_len": 6,
                      "share_embedding": "cate_id"}),
]
_NUM = [("I0", {"type": "numeric", "source": ""})] + _CAT
_MIXED = _CAT[:2] + [("C9", {"type": "categorical", "source": "", "padding_idx": 0, "vocab_size": 9,
                             "embedding_dim": 4})]
_SEQ_FIRST = [
    ("click_history", {"type": "sequence", "source": "", "padding_idx": 0, "vocab_size": 50, "max_len": 6}),
    _SEQ[0], _SEQ[1],
]


def _make(name, specs, dim=8, **kw):
    torch.manual_seed(0)
    fm = FeatureMap.from_specs(specs, embedding_dim=dim)
    if name == "DCNv2":
        return zoo.DCNv2(fm, gpu=-1, embedding_dim=dim, model_structure="parallel", parallel_dnn_hidden_units=[8], **kw)
    if name == "xDeepFM":
        return zoo.xDeepFM(fm, gpu=-1, embedding_dim=dim, dnn_hidden_units=[8], cin_hidden_units=[4], **kw)
    return zoo.DIN(fm, gpu=-1, embedding_dim=dim, dnn_hidden_units=[10], attention_hidden_units=[7], **kw)


def _pooled_din():
    m = _make("DIN", _SEQ)
    from fuxictr_b200.layers import MaskedSumPooling
    m.embedding_layer.feature_encoders["cate_history"] = MaskedSumPooling()
    return m


@pytest.mark.parametrize("case,build,match", [
    ("numeric", lambda: _make("DCNv2", _NUM), "categorical or sequence"),
    ("mixed_dims", lambda: _make("DCNv2", _MIXED), "common embedding dim"),
    ("pooled_sequence", _pooled_din, "encoder"),
    ("lr_over_sequences", lambda: _make("xDeepFM", _SEQ), "over sequence"),
    ("fm_over_sequences", lambda: _make("DIN", _SEQ), "over sequence"),
])
def test_unsupported_inputs_are_refused_before_anything_is_sharded(case, build, match, monkeypatch):
    from fuxictr_b200 import _lib
    model = build()
    calls = []
    monkeypatch.setattr(_lib, "call", lambda *a: calls.append(a[0]))
    monkeypatch.setattr(SH, "shard_rows", lambda *a: calls.append("shard_rows"))
    monkeypatch.setattr(SH.ShardedFront, "__init__", lambda *a, **k: calls.append("ShardedFront"))
    before = {k: v.clone() for k, v in model.state_dict().items()}
    with pytest.raises(NotImplementedError, match=match):
        model.enable_sharding(SH.VirtualPeerGroup(0, 2, {}), 4, 40, want_fm=(case == "fm_over_sequences"))
    assert calls == []
    assert getattr(model, "_sharded_front", None) is None and getattr(model, "_sharded_params", None) is None
    for k, v in model.state_dict().items():
        assert v.shape == before[k].shape and torch.equal(v, before[k]), k


def test_every_in_scope_model_routes_through_the_sharded_front():
    for name in ("DeepFM", "DLRM", "DCNv2", "xDeepFM", "DIN"):
        assert getattr(zoo, name)._routes_sharded_front is True, name


def test_slot_layout_of_din_fields():
    """C4-like: three one-slot fields and two 6-long histories -> 15 slots; a history's slots follow its
    predecessors, its row lands at b*S*D + slot*D."""
    starts, S = SH.slot_layout([1, 1, 1, 6, 6])
    assert starts == [0, 1, 2, 3, 9, 15] and S == 15
    starts, S = SH.slot_layout([1] * 39)
    assert starts == list(range(40)) and S == 39


def test_owned_capacity_and_the_int32_bound():
    # every (requester, sample, slot) candidate of the global batch: the list never overflows
    assert SH.owned_capacity(8, 2048, [1, 1, 1, 50, 50]) == 8 * 2048 * 103
    assert SH.owned_capacity(1, 16, [1] * 7) == 112
    with pytest.raises(ValueError, match="int32"):
        SH.owned_capacity(1, 2 ** 21, [1] * 1024)                 # B * S = 2^31
    with pytest.raises(ValueError, match="int32"):
        SH.owned_capacity(16, 2 ** 20, [1] * 128)                 # world * B * S = 2^31


def test_the_int32_bound_is_enforced_before_anything_is_sharded(monkeypatch):
    from fuxictr_b200 import _lib
    model = _make("DCNv2", _CAT)
    calls = []
    monkeypatch.setattr(_lib, "call", lambda *a: calls.append(a[0]))
    monkeypatch.setattr(SH, "shard_rows", lambda *a: calls.append("shard_rows"))
    with pytest.raises(ValueError, match="int32"):
        model.enable_sharding(SH.VirtualPeerGroup(0, 16, {}), 2 ** 27, 6, want_fm=False)
    assert calls == []


def test_shared_tables_are_one_input_each():
    a, b, c = torch.zeros(3), torch.zeros(3), torch.zeros(3)
    tabs, where = SH._distinct([a, b, a, c, b])
    assert len(tabs) == 3 and tabs[0] is a and tabs[1] is b and tabs[2] is c
    assert where == [0, 1, 0, 2, 1]


@pytest.mark.parametrize("views", [True, False])
def test_batch_matrix_is_recovered_when_the_first_feature_is_a_sequence(views):
    fm = FeatureMap.from_specs(_SEQ_FIRST, embedding_dim=8)
    model = zoo.DIN(fm, gpu=-1, embedding_dim=8, dnn_hidden_units=[10], attention_hidden_units=[7],
                    din_target_field="item_id", din_sequence_field="click_history")
    W = fm.input_length + 1
    mat = torch.arange(5 * W, dtype=torch.float64).view(5, W)
    inputs = fm.batch_views(mat) if views else fm.batch_dict(mat)
    got = model._batch_matrix(inputs)
    assert torch.equal(got, mat)

"""Which steps may update the untouched table granules early (FusedAdam.start_early_tables), without a GPU.

The split is exact only when every table granule a step reads or writes is flagged from its ids before the
side pass starts: the model must read and write its tables through the one front or gather launch that
_table_reads describes, and the optimizer's flags must be final before its gradients exist."""
import types

import pytest
import torch

from fuxictr_b200 import zoo
from fuxictr_b200.arena import FusedAdam, ParamArena, set_early_table_adam
from fuxictr_b200.schema import FeatureMap

_CAT = [("C%d" % i, {"type": "categorical", "source": "", "padding_idx": 0, "vocab_size": 11 + 3 * i})
        for i in range(5)]
_MODELS = {
    "DeepFM": dict(embedding_dim=4, hidden_units=[8]),
    "xDeepFM": dict(embedding_dim=4, dnn_hidden_units=[8], cin_hidden_units=[4]),
    "DLRM": dict(embedding_dim=4, top_mlp_units=[8], bottom_mlp_units=[8]),
    "DCNv2": dict(embedding_dim=4, model_structure="parallel", parallel_dnn_hidden_units=[8]),
}


def _inputs(n=6):
    return {name: torch.randint(0, spec["vocab_size"], (n,)).double() for name, spec in _CAT}


@pytest.mark.parametrize("name", sorted(_MODELS))
def test_table_reads_name_the_one_front_launch(name):
    torch.manual_seed(0)
    kw = _MODELS[name]
    model = getattr(zoo, name)(FeatureMap.from_specs(_CAT, embedding_dim=kw["embedding_dim"]), gpu=-1, **kw)
    X = _inputs()
    reads = model._table_reads(X)
    if name != "DeepFM":       # the serial table pass (general gather, or measured slower with the side pass)
        assert reads is None
        return
    plan, lr_plan, ids, emb_tables, lr_tables = reads
    assert [f.name for f in plan.fields] == [n for n, _ in _CAT]
    assert all(i is X[n] for i, (n, _) in zip(ids, _CAT))
    assert len(emb_tables) == len(_CAT) and all(t.shape[1] == 4 for t in emb_tables)
    assert [f.name for f in lr_plan.fields] == [n for n, _ in _CAT] and all(t.shape[1] == 1 for t in lr_tables)


def _opt(**kw):
    opt = FusedAdam.__new__(FusedAdam)
    opt.arena = types.SimpleNamespace(touched=object())
    opt.sharded, opt.grad_allreduce, opt.zero_grad_in_step, opt.lazy = False, False, True, None
    for k, v in kw.items():
        setattr(opt, k, v)
    return opt


@pytest.mark.parametrize("kw,ok", [
    ({}, True),
    (dict(sharded=True), False),
    (dict(grad_allreduce=True), False),
    (dict(zero_grad_in_step=False), False),
    (dict(lazy=object()), False),
    (dict(arena=types.SimpleNamespace(touched=None)), False),
])
def test_early_tables_only_where_flags_are_final_once_the_ids_are_known(kw, ok):
    assert _opt(**kw).early_tables_ok() == ok
    set_early_table_adam(False)
    try:
        assert not _opt(**kw).early_tables_ok()
    finally:
        set_early_table_adam(True)


def test_a_table_gradient_outside_the_front_is_refused_while_flags_are_frozen():
    a = ParamArena.__new__(ParamArena)
    a.touched = torch.zeros(4, dtype=torch.uint8)
    a.tail_offset, a.flags_frozen = 64, True
    table, dense = types.SimpleNamespace(offset=0, numel=32), types.SimpleNamespace(offset=64, numel=8)
    ParamArena.mark_slot(a, dense)                     # the dense tail has no flags
    with pytest.raises(RuntimeError, match="early"):
        ParamArena.mark_slot(a, table)
    a.flags_frozen = False
    ParamArena.mark_slot(a, table)
    assert a.touched.tolist() == [1, 1, 0, 0]

"""Lazy tables without a GPU: which models may use them, and the per-device row limit.

A lazily evaluated table is only correct when every read of it goes through a kernel that replays the
missed zero-gradient updates (the fused front, the sharded push) and every backward enqueues the rows
it touches.  Models whose forward reads tables through the general gather (DCNv2, DIN) must be refused
before anything is allocated, instead of silently freezing their tables."""
import pytest
import torch

from fuxictr_b200 import zoo
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


@pytest.mark.parametrize("name,specs,kwargs", [
    ("DCNv2", _CAT, dict(embedding_dim=4, model_structure="parallel", parallel_dnn_hidden_units=[8])),
    ("DCNv2", _CAT, dict(embedding_dim=4, model_structure="crossnet_only", num_cross_layers=1)),
    ("DIN", _SEQ, dict(embedding_dim=8, dnn_hidden_units=[10], attention_hidden_units=[7])),
])
def test_lazy_tables_are_refused_for_models_without_a_replaying_read(name, specs, kwargs, monkeypatch):
    from fuxictr_b200 import _lib, arena
    calls = []
    monkeypatch.setattr(_lib, "call", lambda *a: calls.append(a[0]))
    monkeypatch.setattr(arena.ParamArena, "__init__", lambda *a, **k: calls.append("ParamArena"))
    torch.manual_seed(0)
    model = getattr(zoo, name)(FeatureMap.from_specs(specs, embedding_dim=kwargs["embedding_dim"]), gpu=-1, **kwargs)
    with pytest.raises(NotImplementedError, match="lazy"):
        model.use_fused_optimizer(lazy_tables=True)
    assert calls == []                           # refused before the arena (or any kernel) exists
    assert model._arena is None and model._fused_optimizer is None
    assert getattr(model, "_lazy", None) is None


def test_models_that_read_every_table_through_a_replaying_kernel_declare_it():
    for name in ("DeepFM", "xDeepFM", "DLRM"):
        assert getattr(zoo, name)._replays_lazy_tables is True, name
    for name in ("DCNv2", "DIN"):
        assert not getattr(getattr(zoo, name), "_replays_lazy_tables", False), name


def test_lazy_tables_refuse_more_rows_than_int32_worklists_hold():
    """Worklist entries are int32 row numbers: 2^31 rows on one device are refused, not wrapped."""
    from fuxictr_b200.arena import LazyTables

    class _Arena(object):
        P = torch.empty(0, device="meta")
    big = [torch.empty((2 ** 30, 1), device="meta"), torch.empty((2 ** 30, 1), device="meta")]
    with pytest.raises(ValueError, match="2\\^31 - 1"):
        LazyTables(_Arena(), big)


def test_virtual_group_sum_needs_the_lockstep_driver():
    """Several virtual ranks live in one process: their cross-rank sum is composed by lockstep_steps, a
    lone step() call cannot do it.  One virtual rank is its own sum."""
    from fuxictr_b200 import sharded as SH
    buf = torch.ones(3)
    SH.VirtualPeerGroup(0, 1, {}).all_reduce_sum(buf)
    assert torch.equal(buf, torch.ones(3))
    with pytest.raises(RuntimeError, match="lockstep_steps"):
        SH.VirtualPeerGroup(0, 2, {}).all_reduce_sum(buf)


def test_lockstep_sum_composes_every_ranks_buffer():
    from fuxictr_b200 import sharded as SH

    class _Opt(object):
        def __init__(self, r):
            self.buf, self.after = torch.full((2,), float(r + 1)), None

        def step_phases(self):
            yield self.buf
            self.after = self.buf.clone()
    opts = [_Opt(r) for r in range(4)]
    SH.lockstep_steps(opts)
    for o in opts:
        assert torch.equal(o.after, torch.full((2,), 10.0))

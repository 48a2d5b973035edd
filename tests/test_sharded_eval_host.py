"""Evaluation of row-sharded models without a GPU: what the evaluation round refuses before any launch (and
before any collective), the training front's batch-shape check, and the round plan of the sharded loader."""
import numpy as np
import pytest
import torch

from fuxictr_b200 import sharded as SH, zoo
from fuxictr_b200.dataloader import MatrixDataLoader
from fuxictr_b200.schema import FeatureMap

_CAT = [("C%d" % i, {"type": "categorical", "source": "", "padding_idx": 0, "vocab_size": 11 + 3 * i})
        for i in range(4)]
B, W = 8, len(_CAT) + 1


def _front(rank=0, world=2):
    """A ShardedFront's host state only (no peer buffers): enough for every check that precedes a launch."""
    fr = object.__new__(SH.ShardedFront)
    fr.group, fr.B, fr.W = SH.VirtualPeerGroup(rank, world, {}), B, W
    fr._landed = None
    return fr


class _Model(object):
    def __init__(self, rank, world):
        self._sharded_front = _front(rank, world)
        self.device = torch.device("cpu")


class _NoLen(object):
    batch_size = B

    def __iter__(self):
        return iter(())


class _Sized(object):
    def __init__(self, n, batch_size=B):
        self.n, self.batch_size = n, batch_size

    def __len__(self):
        return self.n

    def __iter__(self):
        raise AssertionError("iterated before the rounds were checked")


@pytest.fixture
def no_launch(monkeypatch):
    from fuxictr_b200 import _lib
    calls = []
    monkeypatch.setattr(_lib, "call", lambda *a: calls.append(a[0]))
    return calls


@pytest.mark.parametrize("shape,match", [((B, W + 1), "columns"), ((B, W - 1), "columns"),
                                         ((B + 1, W), "batch_size <= batch_local")])
def test_an_evaluation_batch_the_round_cannot_serve_is_refused_before_any_launch(shape, match, no_launch):
    fr = _front()
    with pytest.raises(ValueError, match=match):
        fr.eval_phase_ids(torch.zeros(shape, dtype=torch.float64))
    assert no_launch == []


@pytest.mark.parametrize("rows", [0, 1, B - 3, B])
def test_ragged_batches_up_to_batch_local_are_accepted(rows):
    assert _front().eval_rows(torch.zeros((rows, W), dtype=torch.float64)) == rows


@pytest.mark.parametrize("shape", [(B - 1, W), (B + 1, W), (B, W + 1), (B, W - 1)])
def test_training_phase_ids_checks_the_batch_shape(shape, no_launch):
    with pytest.raises(ValueError, match=r"\(batch_local, matrix_width\) = \(%d, %d\)" % (B, W)):
        _front().phase_ids(torch.zeros(shape, dtype=torch.float64))
    assert no_launch == []


@pytest.mark.parametrize("world", [2, 8])
def test_virtual_ranks_with_generators_of_different_lengths_are_refused(world, no_launch):
    models = [_Model(r, world) for r in range(world)]
    gens = [_Sized(3) for _ in range(world)]
    gens[-1] = _Sized(4)
    with pytest.raises(ValueError, match="different lengths"):
        SH.lockstep_evaluate(models, gens, ["logloss", "AUC"])
    with pytest.raises(ValueError, match="different lengths"):
        SH.lockstep_predict(models, gens)
    assert no_launch == []


def test_a_generator_without_len_is_refused_by_name(no_launch):
    models = [_Model(r, 2) for r in range(2)]
    with pytest.raises(ValueError, match="rank 1's _NoLen has none"):
        SH.lockstep_evaluate(models, [_Sized(3), _NoLen()], ["logloss"])
    assert no_launch == []


def test_a_loader_with_batches_wider_than_batch_local_is_refused_up_front(no_launch):
    models = [_Model(r, 2) for r in range(2)]
    with pytest.raises(ValueError, match="batch_size <= batch_local"):
        SH.lockstep_evaluate(models, [_Sized(3), _Sized(3, batch_size=B + 1)], ["AUC"])
    assert no_launch == []


def test_group_metrics_stay_refused(no_launch):
    models = [_Model(r, 2) for r in range(2)]
    with pytest.raises(NotImplementedError, match="gAUC"):
        SH.lockstep_evaluate(models, [_Sized(3), _Sized(3)], ["logloss", "gAUC"])
    assert no_launch == []


def test_check_rounds_agrees_on_every_rank():
    SH.check_rounds([(5, B), (5, B), (5, None)], ["a", "b", "c"], B)
    with pytest.raises(ValueError, match="rank 0's x has none"):
        SH.check_rounds([(None, B), (5, B)], ["x", "y"], B)


def test_evaluate_of_a_model_on_virtual_ranks_points_to_the_lockstep_driver(no_launch):
    fm = FeatureMap.from_specs(_CAT, embedding_dim=8)
    torch.manual_seed(0)
    m = zoo.DLRM(fm, gpu=-1, embedding_dim=8, top_mlp_units=[8], bottom_mlp_units=[8])
    m._sharded_front = _front(0, 2)
    with pytest.raises(RuntimeError, match="lockstep_evaluate"):
        m.evaluate(_Sized(3), ["logloss"])
    with pytest.raises(RuntimeError, match="lockstep_predict"):
        m.predict(_Sized(3))
    assert no_launch == []


@pytest.mark.parametrize("world,k", [(8, 2), (2, 1), (4, 0)])
def test_round_plan_of_the_sharded_loader_with_a_tail_smaller_than_world(world, k):
    """k full rounds, then a tail of 3 rows: ranks 0..2 get one row each, the others 0 rows — but every rank
    has the same len(), so every rank runs the same rounds, and the union in rank order is the whole split."""
    fm = FeatureMap.from_specs(_CAT, embedding_dim=8)
    n = k * B * world + 3
    data = np.arange(n * W, dtype=np.float64).reshape(n, W)
    loaders = [MatrixDataLoader(fm, data, batch_size=B, shard=(r, world), drop_last=False, pin=False)
               for r in range(world)]
    assert len(set(len(ld) for ld in loaders)) == 1 and len(loaders[0]) == k + 1
    rounds = [list(ld.matrices()) for ld in loaders]
    seen = []
    for i in range(k + 1):
        sizes = [rounds[r][i].shape[0] for r in range(world)]
        if i < k:
            assert sizes == [B] * world
        else:       # split as evenly as the rows allow, earlier ranks take the remainder
            base, extra = divmod(3, world)
            assert sizes == [base + (1 if r < extra else 0) for r in range(world)]
            if world == 8:
                assert sizes == [1, 1, 1, 0, 0, 0, 0, 0]
        for r in range(world):
            seen.append(rounds[r][i][:, 0])
    first_col = torch.cat(seen).numpy()
    assert np.array_equal(np.sort(first_col), data[:, 0])        # every row once
    SH.check_rounds([(len(ld), ld.batch_size) for ld in loaders], ["loader"] * world, B)

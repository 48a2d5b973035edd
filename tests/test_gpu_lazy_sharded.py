"""Lazy tables (dense Adam semantics evaluated row-wise) over row-sharded tables, and for DLRM.

Row-sharded runs use `world` virtual ranks on ONE GPU (fuxictr_b200.sharded.VirtualPeerGroup): the push /
pull kernels cannot tell a local pointer from an NVLink peer pointer.  `_lockstep_train_step` runs
RankModel.fused_train_step for every rank phase by phase, in the order the barriers of the sharded front
impose on real ranks, and the optimizer steps through sharded.lockstep_steps, which composes the global
gradient norm over the ranks through the same FusedAdam code that sums it with NCCL on real ranks."""
import sys
from collections import OrderedDict

import pytest
import torch

from conftest import close, ROOT

sys.path.insert(0, ROOT)
pytestmark = pytest.mark.gpu

NF, D, B_L = 7, 8, 16


def _specs(nf=NF):
    return [("C%d" % i, {"type": "categorical", "source": "", "padding_idx": 0, "vocab_size": 60 + 17 * i})
            for i in range(nf)]


def _model(name, fm, max_norm):
    from fuxictr_b200 import zoo
    torch.manual_seed(123)
    if name == "DeepFM":
        m = zoo.DeepFM(fm, gpu=0, embedding_dim=D, hidden_units=[32, 16])
    else:
        m = zoo.DLRM(fm, gpu=0, embedding_dim=D, top_mlp_units=[32, 16], bottom_mlp_units=[16], interaction_op="dot")
    with torch.no_grad():
        for mod in m.modules():
            if isinstance(mod, torch.nn.Embedding):
                mod.weight[1:].normal_(0, 0.3)
    m._max_gradient_norm = max_norm
    return m


def _ranks(name, world, lazy, max_norm, fm, width):
    """`world` virtual ranks of one model: same seed, so the dense parameters are replicas and every rank
    keeps its rows of the same tables."""
    from fuxictr_b200 import sharded as SH
    import __graft_entry__
    __graft_entry__.build()
    registry, models = {}, []
    for r in range(world):
        m = _model(name, fm, max_norm)
        m.enable_sharding(SH.VirtualPeerGroup(r, world, registry), B_L, width, torch.float64,
                          want_fm=(name == "DeepFM"))
        m.use_fused_optimizer(lazy_tables=lazy)
        models.append(m)
    return models


def _batch(specs, gen, B):
    ids = torch.cat([torch.randint(0, s["vocab_size"], (B, 1), generator=gen) for _, s in specs], 1)
    return torch.cat([ids.double(), (torch.rand(B, 1, generator=gen) < 0.4).double()], 1).cuda()


def _lockstep_train_step(models, mats, fm, combine=None, before_step=None):
    """fused_train_step of every virtual rank in lock step.  The sharded front's phases run for all ranks
    between its barriers (ids -> push -> reduce; gradient prep -> pull); the rest of each rank's forward
    and backward is the model's own fused_train_step, handed the landed rows.  Returns (losses, landed
    rows (emb, lrw) of every rank as the push delivered them).  before_step() runs after the pulls."""
    from fuxictr_b200 import sharded as SH, functional as F2
    fronts = [m._sharded_front for m in models]
    for m in models:
        m._fused_optimizer.zero_grad()
    for fr, mat in zip(fronts, mats):
        fr.phase_ids(mat)
    for fr in fronts:
        fr.phase_push()
    outs = [fr.phase_reduce() for fr in fronts]
    landed = [(o[0].clone(), fr.lrw.clone() if fr.lr_tables else None) for fr, o in zip(fronts, outs)]
    losses, leaves = [], []
    real_front = SH.sharded_front
    try:
        for m, fr, mat, (emb, logit, _) in zip(models, fronts, mats, outs):
            e = emb.view(fr.B, fr.F, fr.dim).detach().requires_grad_(True)
            lg = logit.detach().requires_grad_(True)
            leaves.append((e, lg))
            SH.sharded_front = lambda front, batch_matrix, _e=e, _lg=lg: (_e, _lg)
            m._fused_optimizer.step = lambda: None       # the ranks step together below
            m._fused_optimizer.zero_grad = lambda: None  # done above, before the push
            losses.append(float(m.fused_train_step(fm.batch_dict(mat)).detach()))
    finally:
        SH.sharded_front = real_front
        for m in models:
            del m._fused_optimizer.step
            del m._fused_optimizer.zero_grad
    for m, fr, (emb, _, sums), (e, lg) in zip(models, fronts, outs, leaves):
        gx = e.grad.reshape(fr.B, -1)
        needs_logit = bool(fr.lr_tables) or fr.want_fm
        gl = (lg.grad.reshape(-1) if lg.grad is not None else torch.zeros(fr.B, device="cuda")) if needs_logit else None
        gbias = F2._grad_buffer(fr.bias, zero=False) if fr.bias is not None else None
        fr.phase_gprep(gx, emb, sums, gl, gbias)
    for fr in fronts:
        egrads = [F2._grad_buffer(t, zero=True) for t in fr.emb_tables]
        lgrads = [F2._grad_buffer(t, zero=True) for t in fr.lr_tables] if fr.lr_tables else None
        fr.phase_pull(egrads, lgrads)
    if before_step is not None:
        before_step()
    SH.lockstep_steps([m._fused_optimizer for m in models], combine=combine)
    return losses, landed


def _sum_in_rank_order(bufs):
    total = bufs[0].clone()
    for b in bufs[1:]:
        total.add_(b)
    for b in bufs:
        b.copy_(total)
    return total


def _expected_worklist(model, mats_all, fm, world, rank):
    """Owned (id % world == rank), non-padding rows touched by ANY rank's samples, as rows of this rank's
    lazy tables: embedding and LR tables alike."""
    fr = model._sharded_front
    rows = []
    for tabs in (fr.emb_tables, fr.lr_tables or []):
        for t, col, pad in zip(tabs, fr.columns, fr.padding):
            ids = mats_all[:, col].long().unique()
            ids = ids[(ids % world == rank) & (ids != pad)]
            rows.append(ids // world + t._b2_grow_base)
    return torch.cat(rows).int().sort().values


@pytest.mark.parametrize("max_norm", [10.0, 0.05])
@pytest.mark.parametrize("name", ["DeepFM", "DLRM"])
@pytest.mark.parametrize("world", [1, 2, 4])
def test_lazy_sharded_optimizer_is_bit_identical_given_identical_gradients(world, name, max_norm):
    """8 steps, rows idle for 0..7 steps.  The lazy ranks receive the dense ranks' gradients (and their
    summed norm term: float-atomic sums differ in the last bit between any two runs).  The rows the push
    delivers from not-yet-materialised shards, and after materialize_tables() the parameters and both
    Adam moments, must be BIT-identical; every rank's worklist holds exactly its owned, non-padding,
    touched rows, once each."""
    from fuxictr_b200.schema import FeatureMap
    specs = _specs()
    fm = FeatureMap.from_specs(specs, embedding_dim=D)
    width = NF + 1
    dense = _ranks(name, world, False, max_norm, fm, width)
    lazy = _ranks(name, world, True, max_norm, fm, width)
    for d, l in zip(dense, lazy):
        assert d._arena.numel == l._arena.numel and d._arena.tail_offset == l._arena.tail_offset
    gen = torch.Generator().manual_seed(9)
    dense_sums, clipped = [], []
    for step in range(8):
        mat = _batch(specs, gen, B_L * world)
        mats = [mat[r * B_L:(r + 1) * B_L].contiguous() for r in range(world)]
        grads = []                                       # the dense step consumes (zeroes) its gradients
        _, landed_d = _lockstep_train_step(dense, mats, fm,
                                           combine=lambda bufs: dense_sums.append(_sum_in_rank_order(bufs)),
                                           before_step=lambda: grads.extend(d._arena.G.clone() for d in dense))

        def hand_over():
            for g, l in zip(grads, lazy):
                l._arena.G.copy_(g)                      # identical gradients

        def combine_lazy(bufs):
            total = _sum_in_rank_order(bufs)
            ref = dense_sums[-1]
            # the norm term composed over the ranks from the worklists matches the dense one ...
            assert abs(float(total[-1]) - float(ref[-1])) <= 1e-5 * float(ref[-1]) + 1e-30, step
            for b in bufs:                           # ... and is handed over like the gradients
                b.copy_(ref)
        _, landed_l = _lockstep_train_step(lazy, mats, fm, combine=combine_lazy, before_step=hand_over)
        for r in range(world):
            assert torch.equal(landed_d[r][0], landed_l[r][0]), (step, r)
            if landed_d[r][1] is not None:
                assert torch.equal(landed_d[r][1], landed_l[r][1]), (step, r)
        torch.cuda.synchronize()
        for r, l in enumerate(lazy):
            lz = l._lazy
            n = int(lz.counter)
            got = lz.worklist[:n].sort().values
            assert torch.equal(got.unique(), got), (step, r)                 # once each
            assert torch.equal(got, _expected_worklist(l, mat, fm, world, r).cuda()), (step, r)
        clipped.append(float(dense[0]._fused_optimizer.sumsq) > max_norm ** 2)
    assert any(clipped) if max_norm < 1 else not any(clipped)     # clipping active / inactive
    # rows really were left behind, for every span of idle steps
    idle = set()
    for l in lazy:
        idle |= set((8 - l._lazy.last_step).tolist())
    assert set(range(8)) <= idle, sorted(idle)
    for l in lazy:
        l.materialize_tables()
    torch.cuda.synchronize()
    for d, l in zip(dense, lazy):
        assert torch.equal(d._arena.P, l._arena.P)
        assert torch.equal(d._fused_optimizer.M, l._fused_optimizer.M)
        assert torch.equal(d._fused_optimizer.V, l._fused_optimizer.V)
        assert float(l._arena.G.abs().sum()) == 0.0


@pytest.mark.parametrize("max_norm", [10.0, 0.05])
@pytest.mark.parametrize("name", ["DeepFM", "DLRM"])
@pytest.mark.parametrize("world", [1, 2, 4])
def test_lazy_sharded_training_matches_dense_sharded_training(world, name, max_norm, monkeypatch):
    """End to end, each mode with its own backward and its own norm composed over the ranks: 7 steps
    agree to 1e-6 (the residual is the float-atomic summation order, which also separates two runs of
    the same mode).  The gradient arena is left all-zero, and no optimizer-side launch of a lazy step
    covers the table slice of the arenas."""
    from fuxictr_b200 import _lib
    from fuxictr_b200.schema import FeatureMap
    specs = _specs()
    fm = FeatureMap.from_specs(specs, embedding_dim=D)
    dense = _ranks(name, world, False, max_norm, fm, NF + 1)
    lazy = _ranks(name, world, True, max_norm, fm, NF + 1)
    gen = torch.Generator().manual_seed(5)
    real_call = _lib.call
    for step in range(7):
        mat = _batch(specs, gen, B_L * world)
        mats = [mat[r * B_L:(r + 1) * B_L].contiguous() for r in range(world)]
        l0, _ = _lockstep_train_step(dense, mats, fm)
        record = []

        def recording():
            monkeypatch.setattr(_lib, "call", lambda fn, *a: (record.append((fn, a)), real_call(fn, *a))[1])
        l1, _ = _lockstep_train_step(lazy, mats, fm, before_step=recording)
        monkeypatch.setattr(_lib, "call", real_call)
        for a, b in zip(l0, l1):
            assert abs(a - b) <= 1e-6 * abs(a), step
        names = [fn for fn, _ in record]
        assert names.count("b2_lazy_adam_step") == world and "b2_adam_step" not in names, names
        assert names.count("b2_lazy_sumsq") == world, names
        for fn, args in record:         # launches over arena memory start at the dense tail, or walk the worklist
            if fn in ("b2_sumsq", "b2_adam_step_sched"):
                ptrs = [int(x.value) for x in args if hasattr(x, "value") and isinstance(x.value, int)]
                for m in lazy:
                    a = m._arena
                    lo = a.G.data_ptr()
                    tail = lo + 4 * a.tail_offset
                    assert not any(lo <= p < tail for p in ptrs), (fn, step)
                    plo, ptail = a.P.data_ptr(), a.P.data_ptr() + 4 * a.tail_offset
                    assert not any(plo <= p < ptail for p in ptrs), (fn, step)
            else:
                assert fn in ("b2_lazy_sumsq", "b2_adam_sched", "b2_lazy_adam_step"), fn
    for m in lazy:
        assert float(m._arena.G.abs().sum()) == 0.0
    for d, l in zip(dense, lazy):
        sd0, sd1 = d.state_dict(), l.state_dict()           # state_dict() materialises the lazy shards
        for k in sd0:
            assert close(sd0[k], sd1[k], 1e-6, atol=1e-9), k


@pytest.mark.parametrize("name", ["DeepFM", "DLRM"])
def test_one_virtual_rank_trains_lazily_through_fused_train_step(name):
    """World 1 needs no lock step: the sharded model's own fused_train_step (sharded front autograd,
    FusedAdam.step summing through the group) with lazy tables tracks the dense run to 1e-6."""
    from fuxictr_b200.schema import FeatureMap
    specs = _specs()
    fm = FeatureMap.from_specs(specs, embedding_dim=D)
    dense = _ranks(name, 1, False, 0.05, fm, NF + 1)[0]
    lazy = _ranks(name, 1, True, 0.05, fm, NF + 1)[0]
    gen = torch.Generator().manual_seed(3)
    for step in range(7):
        mat = _batch(specs, gen, B_L)
        l0 = float(dense.fused_train_step(fm.batch_dict(mat)))
        l1 = float(lazy.fused_train_step(fm.batch_dict(mat)))
        assert abs(l0 - l1) <= 1e-6 * abs(l0), step
    sd0, sd1 = dense.state_dict(), lazy.state_dict()
    for k in sd0:
        assert close(sd0[k], sd1[k], 1e-6, atol=1e-9), k
    assert float(lazy._arena.G.abs().sum()) == 0.0


# ------------------------------------------------------------------ DLRM, unsharded
def _dlrm_specs(numeric):
    specs = [("C%d" % i, {"type": "categorical", "source": "", "padding_idx": 0, "vocab_size": 200 + 17 * i})
             for i in range(9)]
    if numeric:
        specs = [("I0", {"type": "numeric", "source": ""}), ("I1", {"type": "numeric", "source": ""})] + specs
    return specs


def _dlrm_batch(specs, gen, B=48):
    cols = []
    for _, s in specs:
        if s["type"] == "numeric":
            cols.append(torch.rand(B, 1, generator=gen).double())
        else:
            cols.append(torch.randint(0, s["vocab_size"], (B, 1), generator=gen).double())
    return torch.cat(cols + [(torch.rand(B, 1, generator=gen) < 0.4).double()], 1).cuda()


def _dlrm_inputs(fm, mat):
    """The batch dict; numeric columns as (B, 1) float32, the shape the bottom MLP concatenates."""
    batch = fm.batch_dict(mat)
    for name, spec in fm.features.items():
        if spec["type"] == "numeric":
            col = fm.get_column_index(name)
            batch[name] = mat[:, col:col + 1].float()
    return batch


def _dlrm_pair(numeric):
    from fuxictr_b200 import zoo
    from fuxictr_b200.schema import FeatureMap
    import __graft_entry__
    __graft_entry__.build()
    specs = _dlrm_specs(numeric)
    fm = FeatureMap.from_specs(specs, embedding_dim=8)

    def build(lazy, max_norm):
        torch.manual_seed(123)
        m = zoo.DLRM(fm, gpu=0, embedding_dim=8, top_mlp_units=[32, 16], bottom_mlp_units=[16],
                     interaction_op="dot")
        with torch.no_grad():
            for mod in m.modules():
                if isinstance(mod, torch.nn.Embedding):
                    mod.weight[1:].normal_(0, 0.3)
        m._max_gradient_norm = max_norm
        m.use_fused_optimizer(lazy_tables=lazy)
        return m
    return fm, specs, build


@pytest.mark.parametrize("numeric", [False, True])
def test_dlrm_lazy_optimizer_is_bit_identical_given_identical_gradients(numeric):
    """DLRM reads its tables through the replaying fused front when they are lazy: after 8 steps with
    rows idle for 0..7 steps, the rows it reads from not-yet-materialised tables, and after
    materialize_tables() the parameters and both moments, equal the dense run's bit for bit."""
    from fuxictr_b200 import layers
    fm, specs, build = _dlrm_pair(numeric)
    dense, lazy = build(False, 10.0), build(True, 10.0)
    assert dense._arena.numel == lazy._arena.numel and dense._arena.tail_offset == lazy._arena.tail_offset
    lz = lazy._lazy
    gen = torch.Generator().manual_seed(9)
    dn, ln = dict(dense.named_parameters()), dict(lazy.named_parameters())
    for step in range(8):
        mat = _dlrm_batch(specs, gen)
        batch = _dlrm_inputs(fm, mat)
        dense._fused_optimizer.zero_grad()
        lazy._fused_optimizer.zero_grad()
        dense.compute_loss(dense.forward(batch), dense.get_labels(batch)).backward()
        lazy.compute_loss(lazy.forward(batch), lazy.get_labels(batch)).backward()    # enqueues the touched rows
        lazy._arena.G.copy_(dense._arena.G)      # identical gradients (the two arenas share one layout)
        torch.cuda.synchronize()
        rows = []
        for p in lz.tables:
            feat = [k for k, q in ln.items() if q is p][0].split("embedding_layers.")[1].split(".")[0]
            r = mat[:, fm.get_column_index(feat)].long().unique()
            rows.append(r[r != 0] + p._b2_grow_base)
        want = torch.cat(rows).int().sort().values
        got = lz.worklist[:int(lz.counter)].sort().values
        assert torch.equal(got, want.cuda()), step             # the front's backward enqueued them, once each
        dense._fused_optimizer.step()
        lazy._fused_optimizer.step()
    torch.cuda.synchronize()
    probe = _dlrm_batch(specs, torch.Generator().manual_seed(77), B=256)
    X = OrderedDict((k, v) for k, v in _dlrm_inputs(fm, probe).items() if k != "label")
    with torch.no_grad():
        e_dense = dense.embedding_layer(X)
        e_lazy, _ = layers.fused_front(lazy.embedding_layer, None, X, False)
    assert torch.equal(e_dense, e_lazy)
    assert int((lz.last_step < int(lazy._fused_optimizer.step_dev)).sum()) > 0
    lazy.materialize_tables()
    torch.cuda.synchronize()
    for k, p in dn.items():
        assert torch.equal(p.data, ln[k].data), k
    assert torch.equal(dense._arena.P, lazy._arena.P)
    assert torch.equal(dense._fused_optimizer.M, lazy._fused_optimizer.M)
    assert torch.equal(dense._fused_optimizer.V, lazy._fused_optimizer.V)
    assert float(lazy._arena.G.abs().sum()) == 0.0


@pytest.mark.parametrize("max_norm", [10.0, 0.05])
@pytest.mark.parametrize("numeric", [False, True])
def test_dlrm_lazy_training_matches_dense_training(numeric, max_norm, monkeypatch):
    """End to end, own backward in each model: 7 steps agree to 1e-6.  The dense DLRM's forward still
    reads its tables through the general gather, launch for launch as before."""
    from fuxictr_b200 import _lib
    fm, specs, build = _dlrm_pair(numeric)
    dense, lazy = build(False, max_norm), build(True, max_norm)
    gen = torch.Generator().manual_seed(9)
    real_call = _lib.call
    for step in range(7):
        mat = _dlrm_batch(specs, gen)
        names = []
        monkeypatch.setattr(_lib, "call", lambda fn, *a: (names.append(fn), real_call(fn, *a))[1])
        l0 = dense.fused_train_step(_dlrm_inputs(fm, mat))
        monkeypatch.setattr(_lib, "call", real_call)
        assert "b2_front_fwd" not in names and "b2_front_bwd" not in names
        assert any(n.startswith("b2_embed_gather") for n in names) and "b2_adam_step" in names
        lnames = []
        monkeypatch.setattr(_lib, "call", lambda fn, *a: (lnames.append(fn), real_call(fn, *a))[1])
        l1 = lazy.fused_train_step(_dlrm_inputs(fm, mat))
        monkeypatch.setattr(_lib, "call", real_call)
        assert "b2_front_fwd" in lnames and "b2_front_bwd" in lnames and "b2_lazy_adam_step" in lnames
        assert not any(n.startswith("b2_embed_gather") for n in lnames)
        assert abs(float(l0) - float(l1)) <= 1e-6 * abs(float(l0)), step
    sd0, sd1 = dense.state_dict(), lazy.state_dict()
    for k in sd0:
        assert close(sd0[k], sd1[k], 1e-6, atol=1e-9), k
    assert float(lazy._arena.G.abs().sum()) == 0.0

"""Touched-granule flags of the table prefix of the gradient arena (b2_touch, ParamArena.touched).

The backward kernels flag every 64-byte granule of G[:tail_offset] they add a table gradient into, and
FusedAdam's clip and Adam passes read G only in flagged granules.  That is exact as long as the invariant
holds: every nonzero float of G[:tail_offset] lies in a flagged granule.  These tests check the invariant
after the backward of every model, unsharded and row-sharded, and on the host paths that bypass the
kernels; and that the flagged passes compute what the full passes compute."""
import ctypes
import sys

import pytest
import torch

from conftest import close, ROOT

sys.path.insert(0, ROOT)
pytestmark = pytest.mark.gpu

from test_gpu_parity import Golden, build_model                      # noqa: E402
from test_gpu_lazy_sharded import (NF, D, B_L, _specs, _model, _ranks, _batch,   # noqa: E402
                                   _lockstep_train_step)


def _assert_invariant(arena, what):
    t = arena.tail_offset
    assert arena.touched is not None and t > 0, what
    g = arena.G[:t]
    flagged = arena.touched.repeat_interleave(16)[:t] != 0
    stray = (g != 0) & ~flagged
    assert not bool(stray.any()), (what, int(stray.sum()), int(stray.nonzero()[0]))


def _checking_calls(monkeypatch, arenas, seen):
    """Wraps _lib.call: the invariant is checked right before every flagged optimizer pass."""
    from fuxictr_b200 import _lib
    real = _lib.call

    def call(fn, *a):
        if fn in ("b2_sumsq_ex", "b2_adam_step_ex"):
            for ar in arenas:
                if a[0].value == ar.G.data_ptr() or (fn == "b2_adam_step_ex" and a[1].value == ar.G.data_ptr()):
                    _assert_invariant(ar, fn)
            seen.append(fn)
        return real(fn, *a)
    monkeypatch.setattr(_lib, "call", call)


@pytest.mark.parametrize("name", ["DeepFM", "xDeepFM", "DLRM", "DCNv2", "DIN"])
def test_flags_cover_every_table_gradient_after_backward(name, monkeypatch):
    g = Golden("model_" + name)
    fm, model = build_model(name, g, True)
    B = g.meta["batch"]
    mat = g["in"]["matrix"].cuda()
    a, opt = model._arena, model._fused_optimizer
    seen = []
    _checking_calls(monkeypatch, [a], seen)
    for i in range(3):
        batch = fm.batch_dict(mat[i * B:(i + 1) * B])
        opt.zero_grad()
        model.compute_loss(model.forward(batch), model.get_labels(batch)).backward()
        torch.cuda.synchronize()
        _assert_invariant(a, (name, i))
        assert float(a.G[:a.tail_offset].abs().sum()) > 0.0, (name, i)
        opt.step()
        torch.cuda.synchronize()
        assert int(a.touched.sum()) == 0, (name, i)              # cleared with the gradients
        assert float(a.G.abs().sum()) == 0.0, (name, i)
    assert "b2_adam_step_ex" in seen and "b2_sumsq_ex" in seen


def test_unsharded_front_flags_only_the_touched_rows():
    """DeepFM's fused front flags the granules of the rows a batch touched, not whole tables."""
    from fuxictr_b200.schema import FeatureMap
    fm = FeatureMap.from_specs(_specs(), embedding_dim=D)
    m = _model("DeepFM", fm, 10.0)
    m.use_fused_optimizer()
    a = m._arena
    mat = _batch(_specs(), torch.Generator().manual_seed(4), B_L)
    batch = fm.batch_dict(mat)
    m._fused_optimizer.zero_grad()
    m.compute_loss(m.forward(batch), m.get_labels(batch)).backward()
    torch.cuda.synchronize()
    _assert_invariant(a, "DeepFM")
    frac = float(a.touched.float().mean())
    assert 0.0 < frac < 0.6, frac


@pytest.mark.parametrize("name", ["DeepFM", "DLRM"])
@pytest.mark.parametrize("world", [2, 4])
def test_shard_pull_flags_cover_every_table_gradient(world, name, monkeypatch):
    """Row-sharded virtual ranks: the pull alone flags what it writes (every gradient buffer is handed out
    as `marks=True`, so no slot is flagged wholesale), and each rank's step reads only flagged granules."""
    from fuxictr_b200 import functional as F2
    from fuxictr_b200.schema import FeatureMap
    specs = _specs()
    fm = FeatureMap.from_specs(specs, embedding_dim=D)
    ranks = _ranks(name, world, False, 0.05, fm, NF + 1)
    real = F2._grad_buffer
    monkeypatch.setattr(F2, "_grad_buffer", lambda p, zero, marks=False: real(p, zero, marks=True))
    seen = []
    _checking_calls(monkeypatch, [m._arena for m in ranks], seen)
    gen = torch.Generator().manual_seed(11)
    for step in range(3):
        mat = _batch(specs, gen, B_L * world)
        mats = [mat[r * B_L:(r + 1) * B_L].contiguous() for r in range(world)]

        def check():
            torch.cuda.synchronize()
            for r, m in enumerate(ranks):
                _assert_invariant(m._arena, (step, r))
        _lockstep_train_step(ranks, mats, fm, before_step=check)
        torch.cuda.synchronize()
        for m in ranks:
            assert int(m._arena.touched.sum()) == 0 and float(m._arena.G.abs().sum()) == 0.0
    assert seen.count("b2_sumsq_ex") == 3 * world and seen.count("b2_adam_step_ex") == 3 * world


@pytest.mark.parametrize("max_norm", [10.0, 0.05])
def test_flagged_passes_match_the_full_passes(max_norm):
    """Given identical G and the same sumsq, the flagged Adam leaves P, M, V and G equal to the flag-less
    pass on copies, and clears every flag; the flagged sumsq equals the full one up to atomic order."""
    from fuxictr_b200 import _lib
    from fuxictr_b200.schema import FeatureMap
    fm = FeatureMap.from_specs(_specs(), embedding_dim=D)
    m = _model("DeepFM", fm, max_norm)
    m.use_fused_optimizer()
    a, opt = m._arena, m._fused_optimizer
    gen = torch.Generator().manual_seed(2)
    for _ in range(3):                                    # nonzero moments everywhere
        m.fused_train_step(fm.batch_dict(_batch(_specs(), gen, B_L)))
    batch = fm.batch_dict(_batch(_specs(), gen, B_L))
    opt.zero_grad()
    m.compute_loss(m.forward(batch), m.get_labels(batch)).backward()
    torch.cuda.synchronize()
    n, t = a.numel, a.tail_offset
    assert 0 < int(a.touched.sum()) < a.touched.numel()
    vp = ctypes.c_void_p
    st = vp(torch.cuda.current_stream().cuda_stream)
    full, flagged = torch.zeros((), device="cuda"), torch.zeros((), device="cuda")
    _lib.call("b2_sumsq", vp(a.G.data_ptr()), n, vp(full.data_ptr()), st)
    _lib.call("b2_sumsq_ex", vp(a.G.data_ptr()), n, vp(flagged.data_ptr()), vp(a.touched.data_ptr()), t, st)
    assert close(flagged, full, 1e-6)
    assert (float(full) > max_norm ** 2) == (max_norm < 1)           # clipping active / inactive
    opt.step_dev.add_(1)
    ref = [x.clone() for x in (a.P, a.G, opt.M, opt.V)]
    got = [x.clone() for x in (a.P, a.G, opt.M, opt.V)]
    flags = a.touched.clone()
    args = (vp(full.data_ptr()), max_norm, 1e-3, 0.9, 0.999, 1e-8, vp(opt.step_dev.data_ptr()), 1)
    _lib.call("b2_adam_step", *[vp(x.data_ptr()) for x in ref], n, *args, st)
    _lib.call("b2_adam_step_ex", *[vp(x.data_ptr()) for x in got], n, *args, vp(flags.data_ptr()), t, st)
    torch.cuda.synchronize()
    for r, g_ in zip(ref, got):
        assert torch.equal(r, g_)
    assert float(got[1].abs().sum()) == 0.0 and int(flags.sum()) == 0


def test_copied_p_grad_of_a_table_is_flagged(monkeypatch):
    """A table gradient that arrives in p.grad (not written by a kernel) is copied into the arena by the
    step, which flags the whole slot: every row of it is updated with its gradient."""
    from fuxictr_b200.schema import FeatureMap
    fm = FeatureMap.from_specs(_specs(), embedding_dim=D)
    m = _model("DeepFM", fm, 10.0)
    m.use_fused_optimizer()
    a, opt = m._arena, m._fused_optimizer
    seen = []
    _checking_calls(monkeypatch, [a], seen)
    batch = fm.batch_dict(_batch(_specs(), torch.Generator().manual_seed(6), B_L))
    opt.zero_grad()
    m.compute_loss(m.forward(batch), m.get_labels(batch)).backward()
    table = a.params[0]
    assert table._b2_slot.offset < a.tail_offset
    dense_grad = torch.randn_like(table) * 1e-3
    table.grad = dense_grad                               # a fresh tensor: copied in by the step
    before = table.detach().clone()
    opt.step()
    torch.cuda.synchronize()
    assert "b2_adam_step_ex" in seen
    moved = (table.detach() != before).all(dim=1)
    assert bool(moved.all())                              # every row received its (nonzero) gradient
    assert int(a.touched.sum()) == 0 and float(a.G.abs().sum()) == 0.0


def test_dp_allreduce_keeps_the_invariant(tmp_path, monkeypatch):
    """Data-parallel replicas (grad_allreduce): the flags are OR-ed over the ranks with the gradients."""
    import torch.distributed as dist
    from fuxictr_b200.schema import FeatureMap
    dist.init_process_group("gloo", init_method="file://%s" % (tmp_path / "store"), rank=0, world_size=1)
    try:
        fm = FeatureMap.from_specs(_specs(), embedding_dim=D)
        m = _model("DeepFM", fm, 10.0)
        m.use_fused_optimizer().grad_allreduce = True
        a = m._arena
        seen = []
        _checking_calls(monkeypatch, [a], seen)
        gen = torch.Generator().manual_seed(8)
        for _ in range(2):
            m.fused_train_step(fm.batch_dict(_batch(_specs(), gen, B_L)))
        torch.cuda.synchronize()
        assert seen.count("b2_adam_step_ex") == 2
        assert int(a.touched.sum()) == 0 and float(a.G.abs().sum()) == 0.0
    finally:
        dist.destroy_process_group()

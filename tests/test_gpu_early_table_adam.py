"""The table Adam split in two (FusedAdam.start_early_tables): the granules a batch does not touch get their g = 0
update on a side stream while the forward and backward run (b2_table_mark + b2_adam_untouched), the touched ones
after the norm (b2_adam_touched).  Given the same gradients the split leaves P, M, V, G and the flags bit-identical
to b2_adam_step_ex; the marks made from the ids cover every granule a backward flags; whole training steps,
eager and replayed from a CUDA graph, follow the serial ones; and every other configuration keeps the serial pass."""
import ctypes
import sys

import pytest
import torch

from conftest import ROOT

sys.path.insert(0, ROOT)
pytestmark = pytest.mark.gpu

from test_gpu_parity import Golden, build_model                          # noqa: E402
from test_gpu_lazy_sharded import D, B_L, _specs, _model, _batch           # noqa: E402

TOL = 1e-5      # test_gpu_backward_fork.py: float atomics in no fixed order, relative to the largest magnitude


@pytest.fixture(autouse=True)
def _restore():
    yield
    from fuxictr_b200 import arena
    arena.set_early_table_adam(True)


def _recording(monkeypatch):
    from fuxictr_b200 import _lib
    real, seen = _lib.call, []

    def call(fn, *a):
        seen.append(fn)
        return real(fn, *a)
    monkeypatch.setattr(_lib, "call", call)
    return seen


def _odd_batch(specs, gen, B):
    """Repeated ids, padding rows (id 0) and ids outside the tables (the front reads and writes nothing there)."""
    mat = _batch(specs, gen, B)
    mat[: B // 4, 0] = 3.0                                   # one row hit by a quarter of the batch
    mat[B // 4: B // 2, 1] = 0.0                             # padding
    mat[B // 2, 2] = float(specs[2][1]["vocab_size"] + 5)    # out of range
    mat[B // 2 + 1, 3] = -1.0
    return mat


@pytest.mark.parametrize("max_norm", [10.0, 0.05])
def test_split_table_pass_matches_adam_step_ex(max_norm):
    name = "DeepFM"
    from fuxictr_b200 import _lib, arena, functional as F2
    from fuxictr_b200.schema import FeatureMap
    specs = _specs()
    fm = FeatureMap.from_specs(specs, embedding_dim=D)
    m = _model(name, fm, max_norm)
    m.use_fused_optimizer()
    a, opt = m._arena, m._fused_optimizer
    gen = torch.Generator().manual_seed(2)
    for _ in range(3):                                        # nonzero moments everywhere
        m.fused_train_step(fm.batch_dict(_batch(specs, gen, B_L)))
    arena.set_early_table_adam(False)
    batch = fm.batch_dict(_odd_batch(specs, gen, 4 * B_L))
    opt.zero_grad()
    m.compute_loss(m.forward(batch), m.get_labels(batch)).backward()
    torch.cuda.synchronize()
    t = a.tail_offset
    assert 0 < int(a.touched.sum()) < a.touched.numel()
    vp = ctypes.c_void_p
    st = vp(torch.cuda.current_stream().cuda_stream)
    sumsq = torch.zeros((), device="cuda")
    _lib.call("b2_sumsq", vp(a.G.data_ptr()), t, vp(sumsq.data_ptr()), st)
    ref = [x[:t].clone() for x in (a.P, a.G, opt.M, opt.V)] + [a.touched.clone()]
    got = [x[:t].clone() for x in (a.P, a.G, opt.M, opt.V)] + [torch.zeros_like(a.touched)]
    step = opt.step_dev.clone()
    # mark from the ids alone (table pointers into the live arena, flags into the copy), then the untouched pass
    touch = _lib.b2_touch(got[4].data_ptr(), a.P.data_ptr(), t)
    F2.table_mark(*m._table_reads(m.get_inputs(batch)), touch)
    torch.cuda.synchronize()
    stray = (ref[4] != 0) & (got[4] == 0)
    assert not bool(stray.any()), int(stray.sum())                   # every granule the backward wrote is marked
    got[4] |= ref[4]                                                  # the backward's own (idempotent) marks
    P, G, M, V, flags = [vp(x.data_ptr()) for x in got]
    _lib.call("b2_adam_untouched", P, M, V, t, flags, 1e-3, 0.9, 0.999, 1e-8, vp(step.data_ptr()), 7, st)
    step.add_(1)
    common = (vp(sumsq.data_ptr()), max_norm, 1e-3, 0.9, 0.999, 1e-8, vp(step.data_ptr()))
    _lib.call("b2_adam_touched", P, G, M, V, t, *common, flags, st)
    _lib.call("b2_adam_step_ex", *[vp(x.data_ptr()) for x in ref[:4]], t, *common, 1, vp(ref[4].data_ptr()), t, st)
    torch.cuda.synchronize()
    for what, r, g in zip("PGMV", ref[:4], got[:4]):
        assert torch.equal(r, g), what
    assert int(got[4].sum()) == 0 and int(ref[4].sum()) == 0 and float(got[1].abs().sum()) == 0.0
    opt.zero_grad()


def test_marks_from_ids_cover_the_backward_flags():
    from fuxictr_b200 import _lib, arena, functional as F2
    arena.set_early_table_adam(False)
    name = "DeepFM"
    g = Golden("model_" + name)
    fm, model = build_model(name, g, True)
    B = g.meta["batch"]
    mat = g["in"]["matrix"].cuda()
    a, opt = model._arena, model._fused_optimizer
    for i in range(3):
        batch = fm.batch_dict(mat[i * B:(i + 1) * B])
        reads = model._table_reads(model.get_inputs(batch))
        assert reads is not None, name
        marks = torch.zeros_like(a.touched)
        F2.table_mark(*reads, _lib.b2_touch(marks.data_ptr(), a.P.data_ptr(), a.tail_offset))
        opt.zero_grad()
        model.compute_loss(model.forward(batch), model.get_labels(batch)).backward()
        torch.cuda.synchronize()
        assert int(a.touched.sum()) > 0
        stray = (a.touched != 0) & (marks == 0)
        assert not bool(stray.any()), (name, i, int(stray.sum()))
        opt.step()


def _close(r, g, tag):
    err = float((r - g).abs().max()) / max(float(r.abs().max()), 1e-30)
    assert err <= TOL, (tag, err)


def _pair(name):
    from fuxictr_b200.schema import FeatureMap
    specs = _specs()
    fm = FeatureMap.from_specs(specs, embedding_dim=D)
    models = []
    for _ in range(2):
        m = _model(name, fm, 10.0)
        m.use_fused_optimizer()
        models.append(m)
    return specs, fm, models


def test_early_steps_follow_serial_steps_eager(monkeypatch):
    from fuxictr_b200 import arena
    specs, fm, (ser, ear) = _pair("DeepFM")
    seen = _recording(monkeypatch)
    gen = torch.Generator().manual_seed(5)
    for step in range(4):
        batch = fm.batch_dict(_odd_batch(specs, gen, 4 * B_L))
        arena.set_early_table_adam(False)
        l0 = ser.fused_train_step(batch)
        del seen[:]
        arena.set_early_table_adam(True)
        l1 = ear.fused_train_step(batch)
        # fork first (mark, then the untouched pass), the flagged pass last among the table launches
        assert seen[:2] == ["b2_table_mark", "b2_adam_untouched"], seen[:3]
        assert "b2_adam_touched" in seen and "b2_adam_step_ex" not in seen
        assert seen.index("b2_adam_touched") > seen.index("b2_sumsq_ex")
        torch.cuda.synchronize()
        _close(l0.detach(), l1.detach(), (step, "loss"))
    for p0, p1 in zip(ser._arena.params, ear._arena.params):
        _close(p0.detach(), p1.detach(), tuple(p0.shape))
    _close(ser._fused_optimizer.V, ear._fused_optimizer.V, "V")
    assert int(ear._arena.touched.sum()) == 0 and float(ear._arena.G.abs().sum()) == 0.0


def test_early_steps_follow_serial_steps_in_a_graph():
    from fuxictr_b200 import arena
    from fuxictr_b200.pipeline import TrainPipeline
    specs, fm, (ser, ear) = _pair("DeepFM")
    gen = torch.Generator().manual_seed(9)
    mats = [_batch(specs, gen, 4 * B_L) for _ in range(5)]
    pipes = []
    for m, on in ((ser, False), (ear, True)):
        arena.set_early_table_adam(on)
        p = TrainPipeline(m, 4 * B_L, mats[0].shape[1], torch.float64, graph=False)
        p.prime(mats[0])
        p.capture(3)
        pipes.append(p)
    for i, mat in enumerate(mats):
        losses = [p.step_device(mat).clone() for p in pipes]
        torch.cuda.synchronize()
        _close(losses[0], losses[1], (i, "loss"))
    for p0, p1 in zip(ser._arena.params, ear._arena.params):
        _close(p0.detach(), p1.detach(), tuple(p0.shape))
    assert int(ear._arena.touched.sum()) == 0 and float(ear._arena.G.abs().sum()) == 0.0


@pytest.mark.parametrize("case", ["switch_off", "regulariser", "lazy", "xDeepFM", "DLRM", "DCNv2", "DIN"])
def test_ineligible_steps_keep_the_serial_pass(case, monkeypatch):
    from fuxictr_b200 import arena
    from fuxictr_b200.schema import FeatureMap
    if case in ("xDeepFM", "DLRM", "DCNv2", "DIN"):
        g = Golden("model_" + case)
        fm, model = build_model(case, g, True)
        B = g.meta["batch"]
        batch = fm.batch_dict(g["in"]["matrix"].cuda()[:B])
    else:
        specs = _specs()
        fm = FeatureMap.from_specs(specs, embedding_dim=D)
        model = _model("DeepFM", fm, 10.0)
        model.use_fused_optimizer(lazy_tables=(case == "lazy"))
        if case == "regulariser":
            model._embedding_regularizer = 1e-4
        batch = fm.batch_dict(_batch(specs, torch.Generator().manual_seed(3), B_L))
    arena.set_early_table_adam(case != "switch_off")
    seen = _recording(monkeypatch)
    model.fused_train_step(batch)
    torch.cuda.synchronize()
    assert "b2_table_mark" not in seen and "b2_adam_untouched" not in seen and "b2_adam_touched" not in seen
    if case != "lazy":
        assert "b2_adam_step_ex" in seen

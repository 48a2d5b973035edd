"""clip + Adam against float64 torch at every branch of the optimizer kernels' launch plans.

Every kernel of the optimizer step (b2_sumsq[_ex], b2_adam_step[_ex|_sched], b2_adam_untouched + b2_adam_touched,
the lazy row-wise kernels and FusedAdam's paths through them) runs a prescribed gradient sequence (no feedback
from P) and is compared with torch.nn.utils.clip_grad_norm_ + torch.optim.Adam on the CPU, in float64 (the exact
answer) and in float32 (what the reference computes).  The bar is the kernel sweep's, applied to the parameter
displacement P_T - P_0 (|P| would hide update errors), to M and V, and to the sum of squares:
    err(ours, fp64) <= max(1e-5, 3 * err(torch fp32, fp64))          (max-norm, relative)
Gradients mix magnitudes from 1e-8 to 1e3, all-zero granules and all-zero rows (tests/test_adam_host.py)."""
import ctypes
import math
import sys

import numpy as np
import pytest
import torch

from conftest import rel_err, ROOT

sys.path.insert(0, ROOT)
pytestmark = pytest.mark.gpu

from test_adam_host import BETAS, adam_state, clip_coef, grad_seq, torch_adam      # noqa: E402

RTOL = 1e-5
SUMSQ_CAP = 132 * 8 * 1024 * 4     # b2_sumsq: 1056 CTAs of 256 threads x 4 float4s, grid-stride beyond
ADAM_CAP = 132 * 8 * 512 * 4       # adam_kernel: 1056 CTAs of 256 threads x 2 float4s = 2,162,688 floats
SCHED_LEN = 1 << 20
vp = ctypes.c_void_p


@pytest.fixture(scope="module", autouse=True)
def _built():
    import __graft_entry__
    __graft_entry__.build()
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"


def bar(ours, ref32, ref64, what):
    e_ours, e_ref = rel_err(ours, ref64), rel_err(ref32, ref64)
    print("adam-sweep %s err %.3g torch-fp32 %.3g" % (what, e_ours, e_ref))
    assert e_ours <= max(RTOL, 3 * e_ref), (what, e_ours, e_ref)


def ptr(x):
    return vp(x.data_ptr())


def stream():
    return vp(torch.cuda.current_stream().cuda_stream)


def check_state(p0, ours, r32, r64, tag):
    """Displacement, M and V of (P, M, V) = ours against the torch results r32 / r64 started from p0."""
    p0 = p0.cpu()
    P, M, V = [x.cpu() for x in ours]
    bar(P - p0, r32[0] - p0, r64[0] - p0.double(), (tag, "dP"))
    bar(M, r32[1], r64[1], (tag, "M"))
    bar(V, r32[2], r64[2], (tag, "V"))


def granule_flags(g, n_flagged, extra_seed=None):
    """One byte per 16 floats of g[:n_flagged]: set where the granule holds a nonzero (plus, with extra_seed, a
    few all-zero granules: marking more is always safe)."""
    nfl = (n_flagged + 15) // 16
    pad = torch.zeros(nfl * 16)
    pad[:n_flagged] = g[:n_flagged]
    f = (pad.view(nfl, 16) != 0).any(1)
    if extra_seed is not None:
        f |= torch.rand(nfl, generator=torch.Generator().manual_seed(extra_seed)) < 0.1
    return f.to(torch.uint8)


# ------------------------------------------------------------------ sum of squares
def _sumsq_cases():
    cases = []
    for n in (1, 3, 4, 5, 4097, SUMSQ_CAP - 4, SUMSQ_CAP + 4):
        nf_opts = {0, 16, (n // 2) // 16 * 16 + 4, n & ~3}
        for nf in sorted(x for x in nf_opts if x <= n):
            for pattern in (("none", "all", "alternating", "one") if nf else ("none",)):
                cases.append((n, nf, pattern))
    return cases


@pytest.mark.parametrize("n,n_flagged,pattern", _sumsq_cases())
def test_sumsq_sweep(n, n_flagged, pattern):
    """out += sum g^2 over the elements past n_flagged and the flagged granules of the prefix; an unflagged
    granule is never read (it holds 1e3 garbage here), and out keeps what it held."""
    g = grad_seq(n, 1, seed=n + n_flagged)[0]
    nfl = (n_flagged + 15) // 16
    flags = torch.zeros(max(nfl, 1), dtype=torch.uint8)
    if pattern == "all":
        flags[:nfl] = 1
    elif pattern == "alternating":
        flags[:nfl:2] = 1
    elif pattern == "one" and nfl:
        flags[nfl // 2] = 1
    seen = torch.ones(n, dtype=torch.bool)
    if nfl:
        seen[:n_flagged] = flags[:nfl].repeat_interleave(16)[:n_flagged] != 0
    g_dev = torch.where(seen, g, torch.full_like(g, 1e3))
    s64 = float((g.double()[seen] ** 2).sum())
    out0 = 0.25 * s64 + 1.0
    exp32 = torch.tensor(out0, dtype=torch.float32) + (g[seen] ** 2).sum()
    gd, fd = g_dev.cuda(), flags.cuda()
    outs = []
    for use_flags in ((False, True) if n_flagged else (True,)):
        out = torch.full((), out0, dtype=torch.float32, device="cuda")
        if use_flags:
            from fuxictr_b200 import _lib
            _lib.call("b2_sumsq_ex", ptr(gd), n, ptr(out), ptr(fd), n_flagged, stream())
        else:
            plain = torch.where(seen, g, torch.zeros_like(g)).cuda()
            from fuxictr_b200 import _lib
            _lib.call("b2_sumsq", ptr(plain), n, ptr(out), stream())
        outs.append(out)
    torch.cuda.synchronize()
    for out in outs:
        bar(out.view(1), exp32.view(1), torch.tensor([out0 + s64], dtype=torch.float64), ("sumsq", n, n_flagged, pattern))


def test_sumsq_50m_elements():
    from fuxictr_b200 import _lib
    n = 50_000_003
    gen = torch.Generator().manual_seed(11)
    g = (torch.pow(10.0, torch.rand(n, generator=gen) * 6.0 - 3.0) * torch.randn(n, generator=gen).sign())
    s64 = float((g.double() ** 2).sum())
    s32 = (g * g).sum()
    gd = g.cuda()
    out = torch.zeros((), device="cuda")
    _lib.call("b2_sumsq", ptr(gd), n, ptr(out), stream())
    half = n // 2 // 16 * 16
    flags = torch.ones((half + 15) // 16, dtype=torch.uint8, device="cuda")
    out_ex = torch.zeros((), device="cuda")
    _lib.call("b2_sumsq_ex", ptr(gd), n, ptr(out_ex), ptr(flags), half, stream())
    torch.cuda.synchronize()
    ref = torch.tensor([s64], dtype=torch.float64)
    bar(out.view(1), s32.view(1), ref, "sumsq 5e7")
    bar(out_ex.view(1), s32.view(1), ref, "sumsq_ex 5e7")


# ------------------------------------------------------------------ dense Adam entry points
CLIPS = {   # name -> (max_norm, injected sumsq or None (b2_sumsq of the gradient) or "null" (no norm at all))
    "inactive": (1e30, None),
    "active": (1.0, None),
    "at_one": (float(np.float32(2.0) + np.float32(1e-6)), 4.0),      # sqrtf(4) + 1e-6f == max_norm: clip 1 exactly
    "sumsq_zero": (1.0, 0.0),
    "sumsq_inf": (1.0, math.inf),                                   # clip 0, as torch
    "sumsq_null": (None, "null"),
}


def _dense_run(kind, n, t0=0, steps=2, betas=(0.9, 0.999), eps=1e-8, lr=1e-3, clip="active", zero_grad=1,
               n_flagged=None, max_ctas=32, seed=0):
    """`steps` optimizer steps t0+1 .. t0+steps through entry point `kind` from an arbitrary state at t0:
    plain (b2_adam_step), ex (b2_adam_step_ex, flagged prefix + flag-less suffix), sched (b2_adam_sched +
    b2_adam_step_sched), split (b2_adam_untouched at max_ctas CTAs, then b2_adam_touched)."""
    from fuxictr_b200 import _lib
    max_norm, inject = CLIPS[clip]
    p0, m0, v0 = adam_state(n, t0, seed)
    grads = grad_seq(n, steps, seed + 1)
    dev = "cuda"
    P, M, V = p0.to(dev), m0.to(dev), v0.to(dev)
    G = torch.zeros(n, device=dev)
    step = torch.zeros((), dtype=torch.int64, device=dev)
    sumsq = torch.zeros((), device=dev)
    sched = torch.zeros((SCHED_LEN, 2), device=dev) if kind == "sched" else None
    nf = n if kind == "split" else (n_flagged if n_flagged is not None else n & ~3)
    st = stream()
    for k, g in enumerate(grads, t0 + 1):
        gd = g.to(dev)
        G.copy_(gd)
        flags = granule_flags(g, nf, extra_seed=k).to(dev) if kind in ("ex", "split") else None
        if inject == "null":
            sp = vp(0)
        elif inject is None:
            sumsq.zero_()
            _lib.call("b2_sumsq", ptr(G), n, ptr(sumsq), st)
            sp = ptr(sumsq)
        else:
            sumsq.fill_(inject)
            sp = ptr(sumsq)
        mn = float(max_norm or 0.0)
        step.fill_(k)
        if kind == "plain":
            _lib.call("b2_adam_step", ptr(P), ptr(G), ptr(M), ptr(V), n, sp, mn, lr, betas[0], betas[1], eps,
                      ptr(step), zero_grad, st)
        elif kind == "ex":
            _lib.call("b2_adam_step_ex", ptr(P), ptr(G), ptr(M), ptr(V), n, sp, mn, lr, betas[0], betas[1], eps,
                      ptr(step), zero_grad, ptr(flags), nf, st)
        elif kind == "sched":
            _lib.call("b2_adam_sched", ptr(step), lr, betas[0], betas[1], ptr(sched), SCHED_LEN, st)
            _lib.call("b2_adam_step_sched", ptr(P), ptr(G), ptr(M), ptr(V), n, sp, mn, betas[0], betas[1], eps,
                      ptr(step), ptr(sched), zero_grad, st)
        else:
            step.fill_(k - 1)                   # the untouched pass runs before the optimizer counts the step
            _lib.call("b2_adam_untouched", ptr(P), ptr(M), ptr(V), n, ptr(flags), lr, betas[0], betas[1], eps,
                      ptr(step), max_ctas, st)
            step.fill_(k)
            _lib.call("b2_adam_touched", ptr(P), ptr(G), ptr(M), ptr(V), n, sp, mn, lr, betas[0], betas[1], eps,
                      ptr(step), ptr(flags), st)
        torch.cuda.synchronize()
        if zero_grad or kind == "split":
            assert float(G.abs().max()) == 0.0, (kind, k, "G not zeroed")
            if flags is not None:
                assert int(flags.sum()) == 0, (kind, k, "flags not cleared")
        else:
            assert torch.equal(G, gd), (kind, k, "G changed without zero_grad")
    state = (t0, m0, v0) if t0 else None
    norm = None if inject in (None, "null") else math.sqrt(inject)
    mnr = None if inject == "null" else max_norm
    r64 = torch_adam(p0, grads, torch.float64, lr, betas, eps, mnr, norm, state)
    r32 = torch_adam(p0, grads, torch.float32, lr, betas, eps, mnr, norm, state)
    check_state(p0, (P, M, V), r32, r64, (kind, n, t0, betas, eps, clip))


def _dense_cases():
    c = []
    for kind in ("plain", "ex", "sched"):
        c += [dict(kind=kind, n=n) for n in (4096, 4097, 4098, 4099)]           # n % 4: the scalar tail
    c += [dict(kind="split", n=n) for n in (4096, 4100)]
    # either side of the grid-stride cap; the flagged prefix of _ex ends mid-granule, the suffix is flag-less
    c += [dict(kind="plain", n=n) for n in (ADAM_CAP - 4, ADAM_CAP + 4, ADAM_CAP + 5)]
    c += [dict(kind="ex", n=ADAM_CAP + 4, n_flagged=ADAM_CAP // 2 + 4), dict(kind="sched", n=ADAM_CAP + 5)]
    c += [dict(kind="split", n=ADAM_CAP + 4, max_ctas=m) for m in (1, 32)]
    c += [dict(kind="ex", n=4100, n_flagged=nf) for nf in (0, 16, 2052)]
    for t0 in (1, 9, 999, 10 ** 6 - 1):                                         # t = 2, 10, 1000, 10^6
        c += [dict(kind=k, n=4100, t0=t0, steps=1) for k in ("plain", "sched", "split")]
    for betas in BETAS:
        c += [dict(kind="plain", n=4100, betas=betas, steps=3), dict(kind="split", n=4100, betas=betas, t0=999, steps=1),
              dict(kind="sched", n=4099, betas=betas, t0=10 ** 6 - 1, steps=1)]
    c += [dict(kind=k, n=4100, eps=1e-3) for k in ("plain", "split")]
    for clip in CLIPS:
        c += [dict(kind=k, n=4099 if k != "split" else 4100, clip=clip) for k in ("plain", "ex", "sched", "split")]
    c += [dict(kind=k, n=4099, zero_grad=0) for k in ("plain", "ex", "sched")]
    return c


def _case_id(c):
    return "-".join("%s=%s" % (k, v) for k, v in c.items())


@pytest.mark.parametrize("case", _dense_cases(), ids=_case_id)
def test_dense_adam_sweep(case):
    _dense_run(**case)


@pytest.mark.parametrize("kind", ["plain", "split"])
def test_nan_norm_steps_unclipped(kind):
    """A NaN norm is where the kernels leave torch (include/fuxictr_b200.h): torch's clip coefficient is NaN and
    every parameter becomes NaN; fminf gives clip = 1 here and the step runs unclipped.  The untouched pass
    runs before the norm exists, so no pass could follow torch."""
    from fuxictr_b200 import _lib
    n, lr, betas, eps = 4100, 1e-3, (0.9, 0.999), 1e-8
    p0, m0, v0 = adam_state(n, 5, 3)
    g = grad_seq(n, 1, 4)[0]
    P, M, V, G = p0.cuda(), m0.cuda(), v0.cuda(), g.cuda()
    sumsq = torch.full((), math.nan, device="cuda")
    step = torch.full((), 6, dtype=torch.int64, device="cuda")
    st = stream()
    if kind == "plain":
        _lib.call("b2_adam_step", ptr(P), ptr(G), ptr(M), ptr(V), n, ptr(sumsq), 1.0, lr, *betas, eps, ptr(step), 1, st)
    else:
        flags = granule_flags(g, n).cuda()
        step.fill_(5)
        _lib.call("b2_adam_untouched", ptr(P), ptr(M), ptr(V), n, ptr(flags), lr, *betas, eps, ptr(step), 32, st)
        step.fill_(6)
        _lib.call("b2_adam_touched", ptr(P), ptr(G), ptr(M), ptr(V), n, ptr(sumsq), 1.0, lr, *betas, eps,
                  ptr(step), ptr(flags), st)
    torch.cuda.synchronize()
    assert bool(torch.isnan(clip_coef(math.nan, 1.0, torch.float32)))
    nan_ref = torch_adam(p0, [g], torch.float32, lr, betas, eps, 1.0, math.nan, (5, m0, v0))
    assert bool(torch.isnan(nan_ref[0]).all())                                   # torch: every parameter NaN
    r64 = torch_adam(p0, [g], torch.float64, lr, betas, eps, None, None, (5, m0, v0))
    r32 = torch_adam(p0, [g], torch.float32, lr, betas, eps, None, None, (5, m0, v0))
    check_state(p0, (P, M, V), r32, r64, ("nan-norm", kind))


def test_adam_sched_writes_only_inside_the_table():
    from fuxictr_b200 import _lib
    L, lr, betas = 64, 1e-3, (0.95, 0.9999)
    sched = torch.full((L, 2), -7.0, device="cuda")
    step = torch.zeros((), dtype=torch.int64, device="cuda")
    for t in (0, L, L + 3):
        step.fill_(t)
        _lib.call("b2_adam_sched", ptr(step), lr, betas[0], betas[1], ptr(sched), L, stream())
    torch.cuda.synchronize()
    assert bool((sched == -7.0).all())
    for t in (1, L - 1):
        step.fill_(t)
        _lib.call("b2_adam_sched", ptr(step), lr, betas[0], betas[1], ptr(sched), L, stream())
    torch.cuda.synchronize()
    for t in (1, L - 1):
        want = (lr / (1.0 - betas[0] ** t), 1.0 / math.sqrt(1.0 - betas[1] ** t))
        for got, w in zip(sched[t].tolist(), want):
            assert abs(got - w) <= 1.2e-7 * w, (t, got, w)
    assert int((sched != -7.0).any(1).sum()) == 2


# ------------------------------------------------------------------ lazy row-wise kernels
def _lazy_run(dims, rows, touches, T, misalign=False, betas=(0.9, 0.999), eps=1e-8, lr=1e-3, max_norm=1.0,
              over_capacity=(), seed=0):
    """Tables of `rows` rows and dims `dims` in one arena (P, G, M, V regions of L floats each; L % 4 != 0 with
    `misalign`, so every delta is misaligned and even dim 16 takes the scalar path).  touches: {step: global rows}.
    Steps 1..T through b2_adam_sched + b2_lazy_sumsq + b2_lazy_adam_step, then b2_lazy_materialize; the result
    must be dense Adam with zero gradients on every row a step did not touch.  over_capacity: steps whose counter
    exceeds the worklist capacity (the kernels read min(counter, capacity) rows)."""
    from fuxictr_b200 import _lib
    dev = "cuda"
    offs, off = [], 0
    for d in dims:
        offs.append(off)
        off += (rows * d + 3) // 4 * 4
    L = off + (1 if misalign else 0)
    total_rows = rows * len(dims)
    buf = torch.zeros(4 * L, device=dev)
    P, G = buf[:L], buf[L:2 * L]
    descs = (_lib.b2_lazy_table * len(dims))()
    for i, (d, o) in enumerate(zip(dims, offs)):
        descs[i].param, descs[i].rows, descs[i].grow_base, descs[i].dim = P.data_ptr() + 4 * o, rows, i * rows, d
    tables = torch.frombuffer(bytearray(bytes(descs)), dtype=torch.uint8).to(dev)
    flat_idx = torch.cat([torch.arange(o, o + rows * d) for d, o in zip(dims, offs)])

    def row_slice(grow):
        i, r = divmod(grow, rows)
        return offs[i] + r * dims[i], dims[i]

    gen = torch.Generator().manual_seed(seed)
    p0 = torch.randn(L, generator=gen) * 0.1
    P.copy_(p0)
    last = torch.zeros(total_rows, dtype=torch.int32, device=dev)
    sched = torch.zeros((SCHED_LEN, 2), device=dev)
    step = torch.zeros((), dtype=torch.int64, device=dev)
    sumsq = torch.zeros((), device=dev)
    counter = torch.zeros(1, dtype=torch.int32, device=dev)
    n_flat = flat_idx.numel()
    grads = []
    st = stream()
    for k in range(1, T + 1):
        step.fill_(k)
        _lib.call("b2_adam_sched", ptr(step), lr, betas[0], betas[1], ptr(sched), SCHED_LEN, st)
        touched = sorted(set(touches.get(k, ())))
        g_full = torch.zeros(L)
        if touched:
            vals = grad_seq(L, 1, seed=seed * 10007 + k, zero_frac=0.0)[0]
            for grow in touched:
                o, d = row_slice(grow)
                g_full[o:o + d] = vals[o:o + d]
            G.copy_(g_full)
        grads.append(g_full[flat_idx])
        cap = len(touched) if k in over_capacity else total_rows
        work = torch.zeros(max(cap, 1), dtype=torch.int32)
        work[:len(touched)] = torch.tensor(touched, dtype=torch.int32) if touched else work[:0]
        work = work.to(dev)
        counter.fill_(len(touched) + (7 if k in over_capacity else 0))
        sp = vp(0)
        if max_norm is not None:
            sumsq.zero_()
            _lib.call("b2_lazy_sumsq", ptr(tables), len(dims), ptr(work), ptr(counter), max(cap, 1), L, ptr(sumsq), st)
            sp = ptr(sumsq)
            if touched:
                torch.cuda.synchronize()
                g = grads[-1]
                bar(sumsq.view(1).cpu(), (g * g).sum().view(1), (g.double() ** 2).sum().view(1), ("lazy sumsq", k))
        _lib.call("b2_lazy_adam_step", ptr(tables), len(dims), ptr(work), ptr(counter), max(cap, 1), L, 2 * L, 3 * L,
                  ptr(last), ptr(sched), ptr(step), sp, float(max_norm or 0.0), betas[0], betas[1], eps, st)
    _lib.call("b2_lazy_materialize", ptr(tables), len(dims), total_rows, 2 * L, 3 * L, ptr(last), ptr(sched),
              ptr(step), betas[0], betas[1], eps, st)
    torch.cuda.synchronize()
    assert bool((last == T).all())
    assert float(G.abs().max()) == 0.0
    ours = [x.cpu()[flat_idx] for x in (buf[:L], buf[2 * L:3 * L], buf[3 * L:])]
    q0 = p0[flat_idx]
    r64 = torch_adam(q0, grads, torch.float64, lr, betas, eps, max_norm)
    r32 = torch_adam(q0, grads, torch.float32, lr, betas, eps, max_norm)
    assert n_flat == q0.numel()
    check_state(q0, ours, r32, r64, ("lazy", tuple(dims[:3]), misalign, T))


GAPS = (0, 1, 7, 500, 5000)


def _gap_touches(rows, ntables):
    """Row 2 + i of table 0 is touched at step 1 and again after an idle gap of GAPS[i] steps; the first and
    last row of every table at steps 1 and 3."""
    t = {}
    for i, gap in enumerate(GAPS):
        for s in (1, gap + 2):
            t.setdefault(s, []).append(2 + i)
    for j in range(ntables):
        for s in (1, 3):
            t.setdefault(s, []).extend([j * rows, j * rows + rows - 1])
    return t


@pytest.mark.parametrize("dims,misalign", [((1,), False), ((3,), False), ((10,), False), ((16,), False),
                                           ((64,), False), ((16,), True), ((3, 16), False)])
def test_lazy_idle_gaps(dims, misalign):
    rows = 12
    _lazy_run(list(dims), rows, _gap_touches(rows, len(dims)), T=5010, misalign=misalign, seed=len(dims))


@pytest.mark.parametrize("betas,eps", [((0.95, 0.9999), 1e-8), ((0.5, 0.9), 1e-3)])
def test_lazy_betas_eps(betas, eps):
    rows = 12
    _lazy_run([16, 3], rows, _gap_touches(rows, 2), T=520, betas=betas, eps=eps, seed=5)


def test_lazy_forty_tables_and_counter_over_capacity():
    """find_table over 40 tables: the first and the last row of each, on different steps; step 4's counter
    exceeds the worklist's capacity."""
    dims = [(1, 3, 10, 16, 64)[i % 5] for i in range(40)]
    rows = 5
    t = {}
    for j in range(40):
        t.setdefault(1 + j % 3, []).append(j * rows)
        t.setdefault(2 + j % 4, []).append(j * rows + rows - 1)
    t[6] = [j * rows + 2 for j in range(0, 40, 3)]
    _lazy_run(dims, rows, t, T=9, over_capacity=(4, 6), seed=7)


def test_lazy_without_clip():
    rows = 12
    _lazy_run([16], rows, _gap_touches(rows, 1), T=12, max_norm=None, seed=9)


# ------------------------------------------------------------------ FusedAdam over an arena with tables first
class _Tables(torch.nn.Module):
    def __init__(self):
        super(_Tables, self).__init__()
        gen = torch.Generator().manual_seed(1)
        self.t0 = torch.nn.Parameter(torch.randn(37, 16, generator=gen) * 0.1)
        self.t1 = torch.nn.Parameter(torch.randn(50, 8, generator=gen) * 0.1)
        self.w = torch.nn.Parameter(torch.randn(33, 7, generator=gen) * 0.1)
        self.b = torch.nn.Parameter(torch.randn(5, generator=gen) * 0.1)


@pytest.mark.parametrize("path", ["serial", "pending", "lazy", "no_clip", "no_zero_grad"])
def test_fused_adam_paths(path):
    """FusedAdam.step_phases over 50 steps with prescribed gradients written into G: table rows (their granules
    flagged, or enqueued on the lazy worklist) and the dense tail (on a side stream, joined by the step, for
    `pending`)."""
    from fuxictr_b200 import arena
    mod = _Tables().cuda()
    a = arena.ParamArena(mod, first=[mod.t0, mod.t1])
    lr, betas, eps = 2e-3, (0.9, 0.99), 1e-8
    max_norm = None if path == "no_clip" else 5.0
    opt = arena.FusedAdam(a, lr=lr, betas=betas, eps=eps, max_norm=max_norm,
                          zero_grad_in_step=(path != "no_zero_grad"))
    lz = opt.enable_lazy([mod.t0, mod.t1]) if path == "lazy" else None
    p0 = a.P.detach().cpu().clone()
    tabs = [(mod.t0, 0), (mod.t1, 37)]
    side = torch.cuda.Stream()
    gen = torch.Generator().manual_seed(3)
    grads = []
    for k in range(50):
        opt.zero_grad()
        vals = grad_seq(a.numel, 1, seed=100 + k)[0]
        g = torch.zeros(a.numel)
        rows = []
        for p, base in tabs:
            off, d = p._b2_slot.offset, p.shape[1]
            for r in torch.nonzero(torch.rand(p.shape[0], generator=gen) < 0.3).flatten().tolist():
                g[off + r * d:off + (r + 1) * d] = vals[off + r * d:off + (r + 1) * d]
                rows.append(base + r)
        g[a.tail_offset:] = vals[a.tail_offset:]
        grads.append(g)
        gd = g.cuda()
        if path == "no_zero_grad":
            a.G.zero_()
        a.G[:a.tail_offset].copy_(gd[:a.tail_offset])
        if lz is not None:
            lz.worklist[:len(rows)].copy_(torch.tensor(rows, dtype=torch.int32))
            lz.counter.fill_(len(rows))
        elif a.touched is not None:
            a.touched |= granule_flags(g, a.tail_offset).cuda()
        if path == "pending":
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                a.G[a.tail_offset:].copy_(gd[a.tail_offset:])
                ev = torch.cuda.Event()
                ev.record(side)
            a.pending.append((ev, gd))
        else:
            a.G[a.tail_offset:].copy_(gd[a.tail_offset:])
        for p in a.params:
            p.grad = None
        opt.step()
        if path == "no_zero_grad":
            torch.cuda.synchronize()
            assert torch.equal(a.G, gd), k
    if lz is not None:
        lz.materialize()
    torch.cuda.synchronize()
    if path != "no_zero_grad":
        assert float(a.G.abs().max()) == 0.0
        if a.touched is not None:
            assert int(a.touched.sum()) == 0
    r64 = torch_adam(p0, grads, torch.float64, lr, betas, eps, max_norm)
    r32 = torch_adam(p0, grads, torch.float32, lr, betas, eps, max_norm)
    check_state(p0, (a.P, opt.M, opt.V), r32, r64, ("fused", path))


def test_early_table_split_matches_float64_adam():
    """DeepFM steps through the early split (b2_table_mark + b2_adam_untouched on the side stream, then
    b2_adam_touched): after each backward G is overwritten with a prescribed gradient inside the granules the
    ids marked (zero elsewhere), and the step must be one float64 Adam step from the state before it."""
    from fuxictr_b200 import arena
    from fuxictr_b200.schema import FeatureMap
    from test_gpu_lazy_sharded import D, B_L, _specs, _model, _batch
    arena.set_early_table_adam(True)
    specs = _specs()
    fm = FeatureMap.from_specs(specs, embedding_dim=D)
    m = _model("DeepFM", fm, 1.0)
    m.use_fused_optimizer()
    a, opt = m._arena, m._fused_optimizer
    gen = torch.Generator().manual_seed(4)
    for _ in range(3):
        m.fused_train_step(fm.batch_dict(_batch(specs, gen, B_L)))
    for s in range(3):
        batch = fm.batch_dict(_batch(specs, gen, 4 * B_L))
        torch.cuda.synchronize()
        p0, m0, v0 = a.P.cpu().clone(), opt.M.cpu().clone(), opt.V.cpu().clone()
        t0 = int(opt.step_dev)
        opt.zero_grad()
        assert opt.early_tables_ok()
        opt.start_early_tables(*m._table_reads(m.get_inputs(batch)))
        m.compute_loss(m.forward(batch), m.get_labels(batch)).backward()
        torch.cuda.synchronize()
        t = a.tail_offset
        marked = a.touched.cpu().repeat_interleave(16)[:t] != 0
        assert 0 < int(marked.sum()) < t
        vals = grad_seq(a.numel, 1, seed=200 + s)[0]
        g = vals.clone()
        g[:t][~marked] = 0.0
        a.G.copy_(g.cuda())
        for p in a.params:
            p.grad = None
        opt.step()
        torch.cuda.synchronize()
        assert opt._early is None and int(a.touched.sum()) == 0 and float(a.G.abs().max()) == 0.0
        r64 = torch_adam(p0, [g], torch.float64, opt.lr, opt.betas, opt.eps, opt.max_norm, None, (t0, m0, v0))
        r32 = torch_adam(p0, [g], torch.float32, opt.lr, opt.betas, opt.eps, opt.max_norm, None, (t0, m0, v0))
        check_state(p0, (a.P, opt.M, opt.V), r32, r64, ("early split", s))

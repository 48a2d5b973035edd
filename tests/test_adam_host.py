"""The Adam constants without a GPU: the fp32 constants the lazy replay reads (b2_lazy_ctx, formed by
LazyTables._new_ctx) are 1 - beta taken in double and rounded once, as torch.optim.Adam rounds the Python float
1 - beta2 it passes to addcmul_; and b2_adam_apply (csrc/adam_common.cuh), restated here in numpy float32 with
its explicit roundings and those constants, meets the float64 sweep's bar against torch.optim.Adam for the
parameter displacement, M and V:
    err(ours, fp64) <= max(1e-5, 3 * err(torch fp32, fp64))          (max-norm, relative)
The torch reference here is shared with tests/test_gpu_adam_sweep.py."""
import math
import types

import numpy as np
import pytest
import torch

from conftest import rel_err

RTOL = 1e-5
BETAS = [(0.9, 0.999), (0.9, 0.99), (0.95, 0.9999), (0.5, 0.9)]


def clip_coef(norm, max_norm, dtype):
    """torch.nn.utils.clip_grad_norm_'s coefficient for a given total norm, in `dtype`."""
    total = torch.tensor(norm, dtype=dtype)
    return torch.clamp(max_norm / (total + 1e-6), max=1.0)


def torch_adam(p0, grads, dtype, lr, betas, eps, max_norm=None, norm=None, state=None):
    """clip_grad_norm_ + torch.optim.Adam (single tensor, CPU) in `dtype` over the gradient sequence `grads`.
    norm: None = the norm of each gradient (clip_grad_norm_); a float = that total norm at every step (the
    value a test hands the kernel as sumsq).  state: (t, m, v) to start from, as after t steps.
    Returns (P, M, V)."""
    p = torch.nn.Parameter(p0.detach().to(dtype).clone())
    opt = torch.optim.Adam([p], lr=lr, betas=betas, eps=eps, foreach=False)
    if state is not None:
        t, m, v = state
        opt.state[p] = {"step": torch.tensor(float(t)), "exp_avg": m.detach().to(dtype).clone(),
                        "exp_avg_sq": v.detach().to(dtype).clone()}
    for g in grads:
        p.grad = g.detach().to(dtype).clone()
        if max_norm is not None:
            if norm is None:
                torch.nn.utils.clip_grad_norm_([p], max_norm)
            else:
                p.grad.mul_(clip_coef(norm, max_norm, dtype))
        opt.step()
    st = opt.state[p]
    return p.detach(), st["exp_avg"], st["exp_avg_sq"]


def grad_seq(n, steps, seed, zero_frac=0.3, row=64):
    """`steps` prescribed gradients of n floats: magnitudes log-uniform over [1e-8, 1e3] with random signs,
    a fraction of all-zero 16-float granules and of all-zero `row`-float rows (an embedding row no sample hit)."""
    gen = torch.Generator().manual_seed(seed)
    out = []
    for _ in range(steps):
        mag = torch.pow(10.0, torch.rand(n, generator=gen, dtype=torch.float64) * 11.0 - 8.0)
        sign = torch.where(torch.rand(n, generator=gen) < 0.5, -1.0, 1.0).double()
        g = (mag * sign).float()
        gran = (torch.rand((n + 15) // 16, generator=gen) < zero_frac).repeat_interleave(16)[:n]
        rows = (torch.rand((n + row - 1) // row, generator=gen) < zero_frac).repeat_interleave(row)[:n]
        g[gran | rows] = 0.0
        out.append(g)
    return out


def adam_state(n, t, seed):
    """An arbitrary Adam state (P, M, V) as after t steps (zero moments at t = 0)."""
    gen = torch.Generator().manual_seed(seed)
    p = torch.randn(n, generator=gen) * 0.1
    if t == 0:
        return p, torch.zeros(n), torch.zeros(n)
    m = torch.randn(n, generator=gen) * 0.5
    v = m * m * 2.0 + torch.rand(n, generator=gen) * 1e-2
    return p, m, v


def ctx_consts(betas, eps=1e-8):
    """(w1, beta2, w2, eps) of the b2_lazy_ctx that LazyTables._new_ctx builds for these betas."""
    from fuxictr_b200 import arena
    z = torch.zeros(4, dtype=torch.int32)
    lz = arena.LazyTables.__new__(arena.LazyTables)
    lz.arena = types.SimpleNamespace(P=torch.zeros(4))
    lz.opt = types.SimpleNamespace(betas=betas, eps=eps, step_dev=torch.zeros(1, dtype=torch.int64),
                                   M=torch.zeros(4), V=torch.zeros(4))
    lz.last_step = lz.mark = lz.worklist = lz.counter = z
    lz.sched, lz.capacity = torch.zeros(2, 2), 4
    ctx = lz._new_ctx([], None)
    return ctx.w1, ctx.beta2, ctx.w2, ctx.eps


@pytest.mark.parametrize("betas", BETAS + [(0.8, 0.95), (0.99, 0.99999)])
def test_lazy_ctx_rounds_one_minus_beta_once(betas):
    w1, b2, w2, eps = ctx_consts(betas, 1e-3)
    assert w1 == float(np.float32(1.0 - betas[0])), (betas, w1)
    assert w2 == float(np.float32(1.0 - betas[1])), (betas, w2)
    assert b2 == float(np.float32(betas[1])) and eps == float(np.float32(1e-3))


def test_lazy_ctx_differs_from_rounding_beta_first():
    """The rule is observable: for 0.999, fl32(1 - fl32(0.999)) is 1.3e-5 (relative) below fl32(1 - 0.999)."""
    _, _, w2, _ = ctx_consts((0.9, 0.999))
    first = float(np.float32(1.0 - float(np.float32(0.999))))
    assert w2 == float(np.float32(1e-3)) and abs(first - w2) / w2 > 1e-5


def _fma(a, b, c):
    """fmaf: a * b is exact in float64 for float32 operands; the sum is rounded to float64, then to float32."""
    return (a.astype(np.float64) * b + c).astype(np.float32)


def restated_adam(p, m, v, grads, t0, lr, betas, eps, consts):
    """b2_adam_apply (csrc/adam_common.cuh) in numpy float32, with the step scalars of adam_step_scalars
    (csrc/dense.cu): step_size = fl32(lr / (1 - beta1^t)), ibc2 = fl32(1 / sqrt(1 - beta2^t)) from the doubles."""
    f32 = np.float32
    w1, b2, w2 = f32(consts[0]), f32(consts[1]), f32(consts[2])
    eps = f32(eps)
    p, m, v = p.copy(), m.copy(), v.copy()
    for k, g in enumerate(grads, t0 + 1):
        step_size = f32(lr / (1.0 - betas[0] ** k))
        ibc2 = f32(1.0 / math.sqrt(1.0 - betas[1] ** k))
        m = _fma(g - m, w1, m)
        v = _fma(w2 * g, g, v * b2)
        denom = _fma(np.sqrt(v), ibc2, eps)
        p = p - step_size * (m / denom)
    return p, m, v


@pytest.mark.parametrize("betas", BETAS)
@pytest.mark.parametrize("t0,steps", [(0, 1), (0, 200), (999, 1), (10 ** 6 - 1, 3)])
def test_restated_update_meets_float64_adam(betas, t0, steps):
    n, lr, eps = 4096, 1e-3, 1e-8
    p0, m0, v0 = adam_state(n, t0, seed=t0 + steps)
    grads = grad_seq(n, steps, seed=steps * 7 + int(betas[1] * 1e4))
    state = (t0, m0, v0) if t0 else None
    r64 = torch_adam(p0, grads, torch.float64, lr, betas, eps, state=state)
    r32 = torch_adam(p0, grads, torch.float32, lr, betas, eps, state=state)
    w1, b2, w2, _ = ctx_consts(betas, eps)
    p, m, v = restated_adam(p0.numpy(), m0.numpy(), v0.numpy(), [g.numpy() for g in grads], t0, lr, betas, eps,
                            (w1, b2, w2))
    ours = (torch.from_numpy(p) - p0, torch.from_numpy(m), torch.from_numpy(v))
    refs = ((r32[0] - p0, r64[0] - p0.double()), (r32[1], r64[1]), (r32[2], r64[2]))
    for what, o, (a, b) in zip(("dP", "M", "V"), ours, refs):
        e_ours, e_ref = rel_err(o, b), rel_err(a, b)
        assert e_ours <= max(RTOL, 3 * e_ref), (what, betas, t0, steps, e_ours, e_ref)

"""The forked MLP-chain backward (weight-gradient GEMMs on a side stream beside the dgrad chain,
functional._WgradFork) against the serial one, eagerly and replayed from a CUDA graph with a batch other than the
captured one: dX bit for bit (the same kernels on the same inputs), dW and db within TOL of their largest magnitude.
Column sums, the head's dW and split-K partials are float atomics in no fixed order, which alone moved the head's
dW (the same kernel on the same stream in both schedules) by 1.4e-6; a backfill wgrad is also split over K
differently.  A gradient read before the side stream wrote it would be off by O(1)."""
import pytest
import torch

from fuxictr_b200 import functional as F2
from fuxictr_b200.arena import ParamArena
from fuxictr_b200._lib import B2_ACT_NONE, B2_ACT_RELU

pytestmark = pytest.mark.gpu

DIMS = [624, 300, 300, 300, 1]
TOL = 1e-5
B = 4096


@pytest.fixture(autouse=True)
def _restore():
    yield
    F2.set_backward_fork(True)
    F2.set_matmul_precision("fp32")


def _mlp(arena):
    torch.manual_seed(0)
    mlp = torch.nn.ModuleList(torch.nn.Linear(DIMS[i], DIMS[i + 1]) for i in range(4)).cuda()
    a = ParamArena(mlp) if arena else None
    layers = [(m.weight, m.bias, B2_ACT_RELU if i < 3 else B2_ACT_NONE) for i, m in enumerate(mlp)]
    return mlp, a, layers


def _inputs(seed):
    gen = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(B, DIMS[0], device="cuda", generator=gen), torch.randn(B, 1, device="cuda", generator=gen) / B


def _grads(mlp, x):
    return [x.grad.clone()] + [p.grad.clone() for p in mlp.parameters()]


def _step(mlp, arena, layers, x, gy):
    if arena is not None:
        arena.G.zero_()
        arena.begin_step(grads_zeroed=True)
    else:
        for p in mlp.parameters():
            p.grad = None
    x.grad = None
    F2.mlp_chain(x, layers).backward(gy)


def _compare(ref, got, tag):
    assert torch.equal(ref[0], got[0]), tag                       # dX
    for r, g in zip(ref[1:], got[1:]):
        err = float((r - g).abs().max()) / max(float(r.abs().max()), 1e-30)
        assert err <= TOL, (tag, tuple(r.shape), err)


def _eager(fork, mode, arena, seed):
    F2.set_matmul_precision(mode)
    F2.set_backward_fork(fork)
    mlp, a, layers = _mlp(arena)
    x, gy = _inputs(seed)
    x.requires_grad_(True)
    _step(mlp, a, layers, x, gy)
    return _grads(mlp, x)          # read right away on the current stream: the backward has joined (or, with an
                                   # arena, nothing defers the join outside fused_train_step)


@pytest.mark.parametrize("mode", ["tf32x3", "tf32", "bf16"])
@pytest.mark.parametrize("arena", [True, False])
def test_forked_backward_matches_serial_eager(mode, arena):
    _compare(_eager(False, mode, arena, 1), _eager(True, mode, arena, 1), (mode, arena))


@pytest.mark.parametrize("mode", ["tf32x3", "tf32", "bf16"])
def test_forked_backward_matches_serial_in_a_graph(mode):
    """Forward + backward captured with the fork (joined at the end of the backward), replayed on a second batch
    copied into the static input."""
    F2.set_matmul_precision(mode)
    ref = _eager(False, mode, True, 2)
    F2.set_backward_fork(True)
    mlp, a, layers = _mlp(True)
    x_static, gy_static = _inputs(1)
    x_static.requires_grad_(True)
    stream = torch.cuda.Stream()
    stream.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(stream):
        for _ in range(2):
            _step(mlp, a, layers, x_static, gy_static)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=stream):
        _step(mlp, a, layers, x_static, gy_static)
    x2, gy2 = _inputs(2)
    with torch.no_grad():
        x_static.copy_(x2)
        gy_static.copy_(gy2)
    g.replay()
    torch.cuda.synchronize()
    _compare(ref, _grads(mlp, x_static), mode)


def test_deferred_join_in_a_graph_keeps_the_operands_alive():
    """A deferred backward and FusedAdam.step captured in one graph, with memory allocated and written between them:
    the activations and dZ the side stream still reads stay allocated until the optimizer's join, so the write
    cannot land in them.  Replayed on a second batch and compared with the serial step from the same state."""
    from fuxictr_b200.arena import FusedAdam
    F2.set_matmul_precision("tf32x3")
    mlp, a, layers = _mlp(True)
    opt = FusedAdam(a, zero_grad_in_step=False)       # G keeps the step's gradients for the comparison
    x_static, gy_static = _inputs(1)

    def step():
        opt.zero_grad()
        a.defer_join = True
        try:
            F2.mlp_chain(x_static, layers).backward(gy_static)
        finally:
            a.defer_join = False
        assert len(a.pending) == (1 if F2._FORK["on"] else 0)
        scratch = torch.empty(B, 2048, device="cuda")      # the size of the freed activations and dZ
        scratch.fill_(1e30)
        opt.step()

    stream = torch.cuda.Stream()
    stream.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(stream):
        for _ in range(2):
            step()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=stream):
        step()
    state = [t.clone() for t in (a.P, opt.M, opt.V, opt.step_dev)]
    x2, gy2 = _inputs(2)
    x_static.copy_(x2)
    gy_static.copy_(gy2)
    g.replay()
    torch.cuda.synchronize()
    got_g = a.G.clone()
    for t, v in zip((a.P, opt.M, opt.V, opt.step_dev), state):
        t.copy_(v)
    F2.set_backward_fork(False)
    with torch.cuda.stream(stream):
        step()
    torch.cuda.synchronize()
    for p in mlp.parameters():
        sl = slice(p._b2_slot.offset, p._b2_slot.offset + p.numel())
        ref = a.G[sl]
        err = float((ref - got_g[sl]).abs().max()) / max(float(ref.abs().max()), 1e-30)
        assert err <= TOL, (tuple(p.shape), err)


def _deepfm(reg):
    from fuxictr_b200 import zoo
    from fuxictr_b200.schema import FeatureMap
    specs = [("C%d" % i, {"type": "categorical", "source": "", "padding_idx": 0, "vocab_size": 1000 + i})
             for i in range(8)]
    fm = FeatureMap.from_specs(specs, embedding_dim=16)
    torch.manual_seed(0)
    model = zoo.DeepFM(fm, gpu=0, embedding_dim=16, hidden_units=[300, 300, 300], net_regularizer=reg)
    model.use_fused_optimizer()
    gen = torch.Generator().manual_seed(1)
    mat = torch.cat([torch.randint(1, s["vocab_size"], (4096, 1), generator=gen).double() for _, s in specs]
                    + [(torch.rand(4096, 1, generator=gen) < 0.25).double()], dim=1)
    return fm, model, mat


def _train_step(fork, reg):
    """One fused_train_step from the same initial state; returns the loss, the gradient arena as the step left it
    (the optimizer is told not to clear it) and how many side-stream joins the optimizer found pending."""
    F2.set_matmul_precision("tf32x3")
    F2.set_backward_fork(fork)
    fm, model, mat = _deepfm(reg)
    opt, seen = model._fused_optimizer, []
    opt.zero_grad_in_step = False
    step_phases = opt.step_phases

    def watched():
        seen.append(len(opt.arena.pending))
        return step_phases()
    opt.step_phases = watched
    loss = model.fused_train_step(fm.batch_dict(mat.cuda()))
    torch.cuda.synchronize()
    return float(loss), opt.arena, seen


@pytest.mark.parametrize("reg", [None, 1e-2])
def test_fused_train_step_forked_matches_serial(reg):
    """fused_train_step with the fork against the serial backward: the same loss, every gradient within TOL.  On
    the fused-logit path the optimizer joins the side stream itself (it finds the join pending).  With a net
    regulariser every MLP weight gets a second gradient, which autograd adds to the chain's on the step's stream:
    there the backward joins before it returns, so the optimizer finds nothing pending and the sum is complete."""
    ref_loss, ref, _ = _train_step(False, reg)
    loss, got, seen = _train_step(True, reg)
    assert seen == [0 if reg else 1], seen
    assert abs(loss - ref_loss) <= 1e-6 * abs(ref_loss)
    for p_ref, p_got in zip(ref.params, got.params):
        sr, sg = p_ref._b2_slot, p_got._b2_slot
        r = ref.G[sr.offset:sr.offset + sr.numel]
        g = got.G[sg.offset:sg.offset + sg.numel]
        err = float((r - g).abs().max()) / max(float(r.abs().max()), 1e-30)
        assert err <= TOL, (tuple(p_ref.shape), err)

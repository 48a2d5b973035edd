"""Dropout in the fused MLP chain on the GPU: the masks the kernels draw (against the numpy restatement of keep()),
the chain's output and every gradient against a float64 restatement with the kernel's masks injected, whole
training steps against the oracle with the same masks (eager and replayed from a CUDA graph), determinism across
processes, and eval mode."""
import os
import subprocess
import sys
from collections import OrderedDict

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from conftest import rel_err, close, ROOT
from test_mlp_dropout_host import keep_mask

sys.path.insert(0, ROOT)
pytestmark = pytest.mark.gpu

RTOL = 1e-5
DEV = torch.device("cuda:0")


@pytest.fixture(scope="module", autouse=True)
def _built():
    import __graft_entry__
    __graft_entry__.build()
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"


@pytest.fixture(autouse=True)
def _restore():
    yield
    from fuxictr_b200 import functional as F2
    F2.set_matmul_precision("fp32")


def snapshot(seed, offset):
    return torch.tensor([seed, offset], dtype=torch.int64, device=DEV)


def kernel_mask(snap, layer, M, N, p):
    """keep * scale as b2_dropout_apply draws it (on ones)."""
    from fuxictr_b200 import functional as F2
    return F2.dropout_apply(torch.ones(M, N, device=DEV), snap, layer, p)


# ------------------------------------------------------------------ 1. the masks
@pytest.mark.parametrize("p", [0.1, 0.2, 0.5])
def test_masks_match_the_restatement_and_the_law(p):
    from fuxictr_b200 import functional as F2
    M, N = 2048, 2053                                   # 4.2 M elements; N % 4 != 0: groups straddle row ends
    seed, off = 0x1D2C3B4A59687706, (3 << 32) + 17
    got = kernel_mask(snapshot(seed, off), 2, M, N, p)
    _, scale = F2.dropout_consts(p)
    kept = got != 0
    assert bool((got[kept] == scale).all())            # kept values are exactly the fp32 scale
    want = torch.from_numpy(keep_mask(seed, off + 2, M, N, p))
    assert torch.equal(kept.cpu(), want)                # bit-equal to the numpy restatement
    n = M * N
    frac = float(kept.double().mean())
    assert abs(frac - (1 - p)) <= 6 * (p * (1 - p) / n) ** 0.5, frac
    # one snapshot gives one mask; consecutive snapshots of the state give independent ones
    state = snapshot(seed, off)
    s1, s2 = torch.empty(2, dtype=torch.int64, device=DEV), torch.empty(2, dtype=torch.int64, device=DEV)
    from fuxictr_b200 import _lib
    _lib.call("b2_dropout_rng_take", F2._ptr(state), F2._ptr(s1), 1, F2._stream())
    _lib.call("b2_dropout_rng_take", F2._ptr(state), F2._ptr(s2), 1, F2._stream())
    assert s1.tolist() == [seed, off] and s2.tolist() == [seed, off + 1] and state.tolist() == [seed, off + 2]
    a, b = kernel_mask(s1, 0, M, N, p) != 0, kernel_mask(s2, 0, M, N, p) != 0
    assert torch.equal(a, kernel_mask(s1, 0, M, N, p) != 0)
    q = (1 - p) ** 2 + p ** 2
    agree = float((a == b).double().mean())
    assert abs(agree - q) <= 6 * (q * (1 - q) / n) ** 0.5, agree


def test_apply_in_place_with_a_leading_dimension():
    from fuxictr_b200 import functional as F2
    M, N, ld = 33, 50, 57
    base = torch.randn(M, ld, device=DEV)
    x = base[:, :N]
    want = x * kernel_mask(snapshot(5, 9), 1, M, N, 0.3)
    tail = base[:, N:].clone()
    F2.dropout_apply(x, snapshot(5, 9), 1, 0.3, out=x)
    assert torch.equal(x, want) and torch.equal(base[:, N:], tail)


# ------------------------------------------------------------------ 2. chain numerics
SHAPES = {"c2": ((624, 300, 300, 300, 1), 4096),          # DeepFM C2: three tensor-core layers and the head
          "dcn_tower": ((624, 500, 500, 500), 2048),       # DCNv2's parallel DNN: ends on act + dropout
          "dlrm_top": ((325, 64, 64, 64, 1), 1000),        # K = 325 is not TMA-aligned: a SIMT-kind first layer
          "off_grid": ((96, 84, 52, 1), 777)}              # M and N off the 128 x BN tile grid
ACTS = {"relu": "relu", "sigmoid": "sigmoid", "none": None}


def _chain_case(shape, act, p, seed):
    dims, B = SHAPES[shape]
    gen = torch.Generator().manual_seed(seed)
    has_head = dims[-1] == 1
    n_hidden = len(dims) - 1 - (1 if has_head else 0)
    x = torch.randn(B, dims[0], generator=gen)
    params = []
    for i in range(len(dims) - 1):
        params.append(torch.randn(dims[i + 1], dims[i], generator=gen) / dims[i] ** 0.5)
        params.append(torch.randn(dims[i + 1], generator=gen) * 0.1)
    if act is None:             # exact zeros among the pre-activations: zero input rows and first-layer bias
        x[::7] = 0.0
        params[1].zero_()
    # an offset keeps the column sums (the last bias gradient) away from cancellation, where the order of the float
    # atomics that form them would decide the last digits
    gout = torch.randn(B, dims[-1], generator=gen) + 0.5
    return dims, B, n_hidden, has_head, x, params, gout


def _restated(dims, n_hidden, has_head, act, p, keeps, gates=None, zs=None):
    """The reference's Linear -> act -> Dropout stack with the kernel's masks (keep in {0, 1}) injected.
    gates: ReLU's branch per hidden layer (z > 0 as the kernel decided it) in place of relu(z) = z * (z > 0), so the
    restatement differentiates the function the kernel took at the few pre-activations within rounding of 0 (the
    caller checks that they are no others); zs collects the pre-activations of the hidden layers."""
    def fn(x, *params):
        h = x
        for i in range(len(dims) - 1):
            h = F.linear(h, params[2 * i], params[2 * i + 1])
            hidden = i < n_hidden
            if hidden and zs is not None:
                zs.append(h.detach())
            if hidden and act == "relu" and gates is not None:
                h = h * gates[i].to(h.dtype)
            elif hidden and act == "relu":
                h = torch.relu(h)
            elif hidden and act == "sigmoid":
                h = torch.sigmoid(h)
            if hidden:
                scale = torch.tensor(1.0 / (1.0 - p), dtype=h.dtype, device=h.device)
                h = h * (keeps[i].to(h.dtype) * scale)
        return h
    return fn


def _fix_state(seed):
    """Put the device's dropout state at {seed, 0}, so a test draws the same masks whatever ran before it."""
    from fuxictr_b200 import functional as F2
    state = F2.dropout_state(DEV)
    state.copy_(snapshot(seed, 0))
    return state


def _grads(fn, inputs, gout, dtype):
    xs = [t.detach().to(device=DEV, dtype=dtype).requires_grad_(True) for t in inputs]
    y = fn(*xs)
    y.backward(gout.to(device=DEV, dtype=dtype))
    return y.detach(), [t.grad for t in xs]


@pytest.mark.parametrize("mode", ["tf32x3", "tf32", "bf16"])
@pytest.mark.parametrize("act", list(ACTS))
@pytest.mark.parametrize("p", [0.1, 0.5])
@pytest.mark.parametrize("shape", list(SHAPES))
def test_chain_matches_float64_with_the_kernel_masks(shape, p, act, mode):
    from fuxictr_b200 import functional as F2
    from fuxictr_b200._lib import B2_ACT_NONE
    a = ACTS[act]
    dims, B, n_hidden, has_head, x, params, gout = _chain_case(shape, a, p, seed=len(shape) * 31 + int(p * 10))
    F2.set_matmul_precision(mode)
    code = F2.ACT_CODE[a]
    xg = x.to(DEV).requires_grad_(True)
    pg = [torch.nn.Parameter(t.to(DEV)) for t in params]
    layers = [(pg[2 * i], pg[2 * i + 1], code if i < n_hidden else B2_ACT_NONE) + ((p,) if i < n_hidden else ())
              for i in range(len(dims) - 1)]
    st = _fix_state(0x5EED0000 + 97 * len(shape) + int(p * 10)).clone()   # the forward snapshots exactly this
    y = F2.mlp_chain(xg, layers)
    assert type(y.grad_fn).__name__.startswith("_MLPChain")
    hs = y.grad_fn.saved_tensors                        # x and every layer's (dropped) output, as the kernels wrote them
    assert len(hs) == len(dims)
    gates = [(hs[i + 1] > 0) for i in range(n_hidden)] if a == "relu" else None
    y.backward(gout.to(DEV))
    keeps = [(kernel_mask(st, i, B, dims[i + 1], p) != 0) for i in range(n_hidden)]
    ours = [xg.grad] + [t.grad for t in pg]
    names = ["x"] + ["%s%d" % (k, i) for i in range(len(dims) - 1) for k in ("W", "b")]
    if mode == "tf32x3":        # the parity arithmetic: the kernel sweep's bar for the output and every gradient
        # ReLU: with ~10^6 pre-activations, some lie within rounding of 0, where two correct fp32 programs take
        # different branches (fp32 torch itself moves dX by up to 0.4 % at C2 that way).  The restatement follows the
        # kernel's branches, and every branch that differs from float64's must sit at such a pre-activation.
        zs = []
        fn = _restated(dims, n_hidden, has_head, a, p, keeps, gates, zs)
        y64, g64 = _grads(fn, [x] + params, gout, torch.float64)
        if gates is not None:
            for i in range(n_hidden):
                z = zs[i]
                flipped = keeps[i] & (gates[i] != (z > 0))
                if bool(flipped.any()):
                    assert float(z[flipped].abs().max()) <= RTOL * float(z.abs().max()), (i, int(flipped.sum()))
        y32, g32 = _grads(fn, [x] + params, gout, torch.float32)
        for what, o, r32, r64 in [("y", y, y32, y64)] + list(zip(names, ours, g32, g64)):
            e_ours, e_ref = rel_err(o, r64), rel_err(r32, r64)
            assert e_ours <= max(RTOL, 3 * e_ref), (what, e_ours, e_ref)
        return
    fn = _restated(dims, n_hidden, has_head, a, p, keeps)
    y64, g64 = _grads(fn, [x] + params, gout, torch.float64)
    # single-pass TF32 / bf16: test_mlp_chain_matches_torch_autograd's bounds (operand rounding and ReLU kinks)
    tol_y, tol = {"tf32": (1e-2, 6e-2), "bf16": (3e-2, 1.5e-1)}[mode]

    def fro(u, v):
        v = v.detach().double().cpu()
        return float((u.detach().double().cpu() - v).norm() / v.norm().clamp_min(1e-30))
    assert fro(y, y64) <= tol_y
    for what, o, r64 in zip(names, ours, g64):
        assert fro(o, r64) <= tol, what


# ------------------------------------------------------------------ 3. training steps
SPECS = [("C%d" % i, {"type": "categorical", "source": "", "padding_idx": 0, "vocab_size": 300 + 7 * i})
         for i in range(8)]
B_STEP, HIDDEN, P_NET = 512, [64, 64, 64], 0.2


def _batches(n):
    gen = torch.Generator().manual_seed(11)
    out = []
    for _ in range(n):
        cols = [torch.randint(1, s["vocab_size"], (B_STEP, 1), generator=gen).double() for _, s in SPECS]
        out.append(torch.cat(cols + [(torch.rand(B_STEP, 1, generator=gen) < 0.3).double()], dim=1))
    return out


def _model(name, p=P_NET):
    from fuxictr_b200 import zoo
    from fuxictr_b200.schema import FeatureMap
    fm = FeatureMap.from_specs(SPECS, embedding_dim=16)
    torch.manual_seed(7)
    if name == "DeepFM":
        model = zoo.DeepFM(fm, gpu=0, embedding_dim=16, hidden_units=HIDDEN, net_dropout=p)
    else:
        model = zoo.DCNv2(fm, gpu=0, embedding_dim=16, parallel_dnn_hidden_units=HIDDEN, num_cross_layers=2,
                          net_dropout=p)
    with torch.no_grad():
        for m in model.modules():
            if isinstance(m, torch.nn.Embedding):
                m.weight[1:].normal_(0, 0.1)
    return fm, model


def _mlp_dropped(x, s, prefix, n_hidden, has_output, masks, p):
    """MLP_Block's Linear -> ReLU -> Dropout children (indices 3 k, 3 k + 1, 3 k + 2) with the masks injected."""
    for k in range(n_hidden):
        x = torch.relu(F.linear(x, s["%smlp.%d.weight" % (prefix, 3 * k)], s["%smlp.%d.bias" % (prefix, 3 * k)]))
        x = x * (masks[k].to(x.dtype) * torch.tensor(1.0 / (1.0 - p), dtype=x.dtype))
    if has_output:
        k = 3 * n_hidden
        x = F.linear(x, s["%smlp.%d.weight" % (prefix, k)], s["%smlp.%d.bias" % (prefix, k)])
    return x


def _oracle_pred(name, spec_map, masks_of_step):
    from oracle import fuxictr_oracle as O
    calls = [0]

    def pred(s, X):
        masks = masks_of_step(calls[0])
        calls[0] += 1
        if name == "DeepFM":
            emb = O.feature_embedding(spec_map, s, "embedding_layer.", X)
            y = O.factorization_machine(spec_map, s, "fm.", X, emb)
            return torch.sigmoid(y + _mlp_dropped(emb.flatten(start_dim=1), s, "mlp.", len(HIDDEN), True, masks, P_NET))
        emb = O.feature_embedding(spec_map, s, "embedding_layer.", X, flatten_emb=True)
        cross = O.crossnet_v2(emb, s, "crossnet.", 2)
        dnn = _mlp_dropped(emb, s, "parallel_dnn.", len(HIDDEN), False, masks, P_NET)
        return torch.sigmoid(F.linear(torch.cat([cross, dnn], dim=-1), s["fc.weight"], s["fc.bias"]))
    return pred


@pytest.mark.parametrize("name", ["DeepFM", "DCNv2"])
def test_fused_train_steps_match_the_oracle_with_the_same_masks(name):
    from fuxictr_b200 import functional as F2
    from oracle import fuxictr_oracle as O
    F2.set_matmul_precision("tf32x3")
    fm, model = _model(name)
    state0 = OrderedDict((k, v.detach().cpu().clone()) for k, v in model.state_dict().items())
    model.use_fused_optimizer()
    seed, off0 = _fix_state(0x5EED1000 + len(name)).tolist()
    mats = _batches(3)
    losses = [float(model.fused_train_step(fm.batch_dict(m.cuda()))) for m in mats]
    n = len(HIDDEN)

    def masks_of_step(k):
        return [torch.from_numpy(keep_mask(seed, off0 + k * n + l, B_STEP, HIDDEN[l], P_NET)) for l in range(n)]
    tr = O.OracleTrainer(state0, _oracle_pred(name, OrderedDict(SPECS), masks_of_step), OrderedDict(SPECS), ["label"])
    ref = [float(tr.train_step(fm.batch_dict(m))) for m in mats]
    assert close(torch.tensor(losses), torch.tensor(ref), RTOL), (losses, ref)
    sd = model.state_dict()
    for k, v in tr.state.items():
        if v.is_floating_point():
            assert close(sd[k], v, 2e-5), (k, rel_err(sd[k], v))
    assert F2.dropout_state(DEV).tolist() == [seed, off0 + 3 * n]


@pytest.mark.parametrize("name", ["DeepFM", "DCNv2"])
def test_graph_replays_draw_the_masks_of_the_eager_steps(name):
    """A captured step reads and advances the device state: replay k draws the masks eager step k would, so a graph
    and an eager run from the same state and weights give the same losses, and replays on one batch differ."""
    from fuxictr_b200 import functional as F2
    from fuxictr_b200.pipeline import TrainPipeline
    F2.set_matmul_precision("tf32x3")
    fm, eager = _model(name)
    _, graphed = _model(name)
    eager.use_fused_optimizer()
    graphed.use_fused_optimizer()
    state = _fix_state(0x5EED2000 + len(name))
    saved = state.clone()
    mat = _batches(1)[0].cuda()
    ref = [float(eager.fused_train_step(fm.batch_dict(mat))) for _ in range(5)]
    state.copy_(saved)
    pipe = TrainPipeline(graphed, B_STEP, mat.shape[1], capture_warmup=3, graph=False)
    pipe.prime(mat)
    pipe.capture(warmup=3)                                  # three eager warm-up steps, then the capture
    got = [float(pipe.step_device(mat)) for _ in range(2)]
    torch.cuda.synchronize()
    assert abs(got[0] - ref[3]) <= 1e-6 * abs(ref[3]) and abs(got[1] - ref[4]) <= 1e-6 * abs(ref[4]), (got, ref)
    assert got[0] != got[1]
    assert state.tolist() == [int(saved[0]), int(saved[1]) + 5 * len(HIDDEN)]


_CHILD = r"""
import sys, torch
sys.path.insert(0, {root!r}); sys.path.insert(0, {tests!r})
import __graft_entry__; __graft_entry__.build()
import test_gpu_mlp_dropout as T
from fuxictr_b200 import functional as F2
F2.set_matmul_precision("tf32x3")
fm, model = T._model("DeepFM")
model.use_fused_optimizer()
torch.manual_seed(1234)
loss = model.fused_train_step(fm.batch_dict(T._batches(1)[0].cuda()))
print("LOSS", float(loss).hex())
"""


def test_same_seed_in_two_processes_gives_bit_equal_first_losses():
    code = _CHILD.format(root=ROOT, tests=os.path.join(ROOT, "tests"))
    out = []
    for _ in range(2):
        r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, r.stderr[-2000:]
        out.append([ln for ln in r.stdout.splitlines() if ln.startswith("LOSS")][-1])
    assert out[0] == out[1], out


# ------------------------------------------------------------------ 4. eval mode
@pytest.mark.parametrize("name", ["DeepFM", "DCNv2"])
def test_eval_forward_is_bit_equal_to_the_model_without_dropout(name):
    from fuxictr_b200 import functional as F2
    F2.set_matmul_precision("tf32x3")
    fm, with_drop = _model(name, P_NET)
    _, plain = _model(name, 0)
    with torch.no_grad():           # the same weights (the Dropout children shift the Linear keys of the state_dict)
        for a, b in zip(plain.parameters(), with_drop.parameters()):
            a.copy_(b)
    with_drop.eval()
    plain.eval()
    batch = fm.batch_dict(_batches(1)[0].cuda())
    with torch.no_grad():
        a = with_drop.forward(batch)["y_pred"]
        b = plain.forward(batch)["y_pred"]
    assert torch.equal(a, b)
    with_drop.train()
    with torch.no_grad():
        c = with_drop.forward(batch)["y_pred"]
    assert not torch.equal(a, c)                             # training mode does drop

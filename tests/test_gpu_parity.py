"""Parity of the sm_90a kernels (called through the C-ABI) against the reference goldens
and the CPU oracle.  Bar (BASELINE.json north_star): index gather bit-exact; logits and
gradients within 1e-5 relative fp32."""
import copy
import ctypes
import os
import sys
from collections import OrderedDict

import numpy as np
import pytest
import torch

from conftest import Golden, rel_err, close, ROOT

sys.path.insert(0, ROOT)
pytestmark = pytest.mark.gpu

RTOL = 1e-5


@pytest.fixture(scope="module", autouse=True)
def _built():
    import __graft_entry__
    __graft_entry__.build()
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from fuxictr_b200 import _lib
    cc = _lib.load().b2_device_cc(0)
    assert cc == 90, "library is sm_90a only (device reports cc %d)" % cc


def fm_from(g, emb_dim=None):
    from fuxictr_b200.schema import FeatureMap
    return FeatureMap.from_specs(g.meta["specs"], labels=g.meta["labels"], embedding_dim=emb_dim)


def cuda_batch(fm, mat, dtype=None):
    mat = mat.cuda()
    if dtype is not None:
        mat = mat.to(dtype)
    batch = fm.batch_dict(mat)
    return batch, OrderedDict((k, v) for k, v in batch.items() if k not in fm.labels)


def load_module(module, g, group="w"):
    module.load_state_dict({k: v for k, v in g[group].items()})
    return module.cuda()


def check_param_grads(module, g, rtol=RTOL):
    """Every parameter gradient within rtol of the reference.  The absolute floor is tied to the
    largest gradient of the module, so a gradient that is mathematically zero (e.g. the last bias
    under a softmax) is compared against rounding noise, not against itself."""
    named = dict(module.named_parameters())
    scale = max(float(ref.abs().max()) for ref in g["g"].values())
    for k, ref in g["g"].items():
        got = named[k].grad
        assert got is not None, k
        assert close(got, ref, rtol, atol=rtol * scale), (k, rel_err(got, ref))


# ------------------------------------------------------------------ embeddings
@pytest.mark.parametrize("idx_dtype", [torch.float64, torch.int64, torch.int32])
def test_feature_embedding_bit_exact(idx_dtype):
    from fuxictr_b200 import layers
    g = Golden("feature_embedding_tiny_npz")
    fm = fm_from(g, 4)
    layer = load_module(layers.FeatureEmbedding(fm, 4), g)
    _, X = cuda_batch(fm, g["in"]["matrix"], idx_dtype)
    out = layer(X)
    assert torch.equal(out.cpu(), g["out"]["stack"])                    # bit-exact gather
    assert torch.equal(layer(X, flatten_emb=True).cpu(), g["out"]["flat"])
    out.backward(g["in"]["gout"].cuda())
    check_param_grads(layer, g)


@pytest.mark.parametrize("tag", ["plain", "avgpool", "sumpool"])
def test_feature_embedding_dict_sequence_shared(tag):
    from fuxictr_b200 import layers
    g = Golden("feature_embedding_dict_tiny_seq_" + tag)
    fm = fm_from(g, 6)
    layer = load_module(layers.FeatureEmbeddingDict(fm, 6), g)
    _, X = cuda_batch(fm, g["in"]["matrix"])
    emb = layer(X)
    assert list(emb.keys()) == [k for k in fm.features.keys()]
    loss = 0
    for k, ref in g["out"].items():
        if tag == "plain" or k != "click_sequence":
            assert torch.equal(emb[k].cpu(), ref), k                    # pure copies stay bit-exact
        else:
            assert close(emb[k], ref, RTOL), k
        loss = loss + (emb[k] * g["gout"][k].cuda()).sum()
    loss.backward()
    check_param_grads(layer, g)


def test_logistic_regression():
    from fuxictr_b200 import layers
    g = Golden("logistic_regression_tiny_seq")
    fm = fm_from(g, 6)
    layer = load_module(layers.LogisticRegression(fm), g)
    _, X = cuda_batch(fm, g["in"]["matrix"])
    out = layer(X)
    assert close(out, g["out"]["y"], RTOL)
    out.backward(g["in"]["gout"].cuda())
    check_param_grads(layer, g)


def test_out_of_range_index_is_flagged_and_empty_batch_ok():
    from fuxictr_b200 import functional as F2, _lib
    table = torch.randn(10, 8, device="cuda")
    plan = F2.GatherPlan([F2.GatherField("a", 0, 8, padding_idx=0)])
    status = torch.zeros(1, dtype=torch.int32, device="cuda")
    idx = torch.tensor([1.0, 12.0, 3.0, -1.0], dtype=torch.float64, device="cuda")
    out = F2.embed_gather(plan, [idx], [table], status=status)
    torch.cuda.synchronize()
    assert int(status.item()) == 1                                      # 1 + field index
    assert torch.equal(out[0], table[1]) and torch.equal(out[2], table[3])
    assert float(out[1].abs().sum()) == 0.0 and float(out[3].abs().sum()) == 0.0
    empty = F2.embed_gather(plan, [idx[:0]], [table])
    assert tuple(empty.shape) == (0, 8)


def test_gather_f64_truncation_matches_long():
    from fuxictr_b200 import functional as F2
    table = torch.arange(40, dtype=torch.float32, device="cuda").view(10, 4)
    idx = torch.tensor([2.9, 3.0, 0.2, 7.999999], dtype=torch.float64, device="cuda")
    plan = F2.GatherPlan([F2.GatherField("a", 0, 4)])
    out = F2.embed_gather(plan, [idx], [table])
    assert torch.equal(out, table[idx.long()])


# ------------------------------------------------------------------ interactions
@pytest.mark.parametrize("name", ["inner_product_B16_F7_D10", "inner_product_B9_F39_D16",
                                  "inner_product_B5_F27_D16"])
def test_inner_product(name):
    from fuxictr_b200 import layers
    g = Golden(name)
    for mode, ref in g["out"].items():
        emb = g["in"]["emb"].cuda().requires_grad_(True)
        layer = layers.InnerProductInteraction(g.meta["F"], output=mode).cuda()
        out = layer(emb)
        assert close(out, ref, RTOL), mode
        out.backward(g["in"]["gout_" + mode].cuda())
        assert close(emb.grad, g["gin"][mode], RTOL), mode


@pytest.mark.parametrize("name", ["crossnet", "crossnet_v2"])
def test_cross(name):
    from fuxictr_b200 import layers
    g = Golden(name)
    cls = layers.CrossNet if name == "crossnet" else layers.CrossNetV2
    layer = load_module(cls(g.meta["input_dim"], g.meta["num_layers"]), g)
    x0 = g["in"]["x0"].cuda().requires_grad_(True)
    out = layer(x0)
    assert close(out, g["out"]["y"], RTOL)
    out.backward(g["in"]["gout"].cuda())
    check_param_grads(layer, g)
    assert close(x0.grad, g["gin"]["x0"], RTOL)


def test_cin():
    from fuxictr_b200 import layers
    g = Golden("cin")
    layer = load_module(layers.CompressedInteractionNet(g.meta["F"], g.meta["cin_hidden_units"]), g)
    emb = g["in"]["emb"].cuda().requires_grad_(True)
    out = layer(emb)
    assert close(out, g["out"]["y"], RTOL)
    out.backward(g["in"]["gout"].cuda())
    check_param_grads(layer, g)
    assert close(emb.grad, g["gin"]["emb"], RTOL)


def test_mlp_relu():
    from fuxictr_b200 import layers
    g = Golden("mlp_relu")
    layer = load_module(layers.MLP_Block(input_dim=20, hidden_units=[16, 12], hidden_activations="ReLU",
                                         output_dim=1), g)
    x = g["in"]["x"].cuda().requires_grad_(True)
    out = layer(x)
    assert close(out, g["out"]["y"], RTOL)
    out.backward(g["in"]["gout"].cuda())
    check_param_grads(layer, g)
    assert close(x.grad, g["gin"]["x"], RTOL)


def test_dice_train_and_eval():
    from fuxictr_b200 import layers
    g = Golden("dice")
    layer = load_module(layers.Dice(12), g)
    layer.train()
    x = g["in"]["x"].cuda().requires_grad_(True)
    out = layer(x)
    assert close(out, g["out"]["train"], RTOL)
    out.backward(g["in"]["gout"].cuda())
    check_param_grads(layer, g)
    assert close(x.grad, g["gin"]["x"], RTOL)
    assert close(layer.bn.running_mean, g["w1"]["bn.running_mean"], RTOL)
    assert close(layer.bn.running_var, g["w1"]["bn.running_var"], RTOL)
    layer.eval()
    assert close(layer(x.detach()), g["out"]["eval"], RTOL)


@pytest.mark.parametrize("softmax", [0, 1])
def test_din_attention(softmax):
    from fuxictr_b200 import layers
    g = Golden("din_attention_softmax%d" % softmax)
    layer = load_module(layers.DIN_Attention(embedding_dim=8, attention_units=[16], hidden_activations="Dice",
                                             use_softmax=bool(softmax)), g)
    layer.train()
    target = g["in"]["target"].cuda().requires_grad_(True)
    hist = g["in"]["history"].cuda().requires_grad_(True)
    out = layer(target, hist, g["in"]["mask"].cuda())
    assert close(out, g["out"]["y"], RTOL)
    out.backward(g["in"]["gout"].cuda())
    check_param_grads(layer, g)
    assert close(target.grad, g["gin"]["target"], RTOL)
    assert close(hist.grad, g["gin"]["history"], RTOL)


# ------------------------------------------------------------------ dense primitives
@pytest.mark.parametrize("M,N,K", [(1, 1, 1), (7, 5, 3), (64, 64, 16), (65, 63, 17), (333, 300, 624),
                                   (4096, 1, 300), (300, 624, 4096), (129, 257, 1000)])
@pytest.mark.parametrize("a_t,b_t", [(False, False), (False, True), (True, False), (True, True)])
def test_gemm_f32_layouts(M, N, K, a_t, b_t):
    from fuxictr_b200 import functional as F2
    gen = torch.Generator().manual_seed(M * 7 + N * 3 + K)
    a = torch.randn((K, M) if a_t else (M, K), generator=gen)
    b = torch.randn((N, K) if b_t else (K, N), generator=gen)
    ref = (a.t() if a_t else a).double() @ (b.t() if b_t else b).double()
    out = torch.empty(M, N, device="cuda")
    F2.gemm_f32(a.cuda(), b.cuda(), out, a_t=a_t, b_t=b_t)
    assert close(out, ref, 2e-6 * max(1, K) ** 0.5, atol=1e-6)


def test_gemm_f32_epilogues_and_accumulate():
    from fuxictr_b200 import functional as F2
    from fuxictr_b200._lib import B2_ACT_RELU, B2_ACT_SIGMOID
    gen = torch.Generator().manual_seed(3)
    M, N, K = 200, 130, 96
    a, b = torch.randn(M, K, generator=gen), torch.randn(N, K, generator=gen)
    bias, mul, add = torch.randn(N, generator=gen), torch.randn(M, N, generator=gen), torch.randn(M, N, generator=gen)
    z = a.double() @ b.double().t() + bias.double()
    out = torch.empty(M, N, device="cuda")
    F2.gemm_f32(a.cuda(), b.cuda(), out, b_t=True, bias=bias.cuda(), act=B2_ACT_RELU)
    assert close(out, torch.relu(z), RTOL)
    F2.gemm_f32(a.cuda(), b.cuda(), out, b_t=True, bias=bias.cuda(), act=B2_ACT_SIGMOID)
    assert close(out, torch.sigmoid(z), RTOL)
    F2.gemm_f32(a.cuda(), b.cuda(), out, b_t=True, bias=bias.cuda(), mul=mul.cuda(), add=add.cuda())
    assert close(out, add.double() + mul.double() * z, RTOL)           # CrossNetV2 epilogue
    base = torch.randn(M, N, generator=gen)
    out = base.cuda().clone()
    F2.gemm_f32(a.cuda(), b.cuda(), out, b_t=True, accumulate=True)
    assert close(out, base.double() + a.double() @ b.double().t(), RTOL)
    # strided output (a column slice of a wider matrix), split-K path (few tiles, long K)
    wide = torch.zeros(40, 100, device="cuda")
    a2, b2 = torch.randn(40, 2048, generator=gen), torch.randn(2048, 30, generator=gen)
    F2.gemm_f32(a2.cuda(), b2.cuda(), wide[:, 10:40])
    assert close(wide[:, 10:40], a2.double() @ b2.double(), RTOL)
    assert float(wide[:, :10].abs().sum()) == 0 and float(wide[:, 40:].abs().sum()) == 0


def test_logit_bce_matches_torch():
    """Fused logit sum + sigmoid + BCE (mean) and its backward against torch."""
    from fuxictr_b200 import functional as F2
    gen = torch.Generator().manual_seed(4)
    B = 513
    t = [torch.randn(B, 1, generator=gen).requires_grad_(True) for _ in range(3)]
    y = (torch.rand(B, 1, generator=gen) < 0.3).float()
    ref_loss = torch.nn.functional.binary_cross_entropy(torch.sigmoid(t[0] + t[1] + t[2]), y)
    ref_loss.backward()
    tc = [v.detach().cuda().requires_grad_(True) for v in t]
    loss, y_pred = F2.logit_bce(y.cuda(), *tc)
    loss.backward()
    assert close(loss, ref_loss, RTOL)
    assert close(y_pred, torch.sigmoid(t[0] + t[1] + t[2]), RTOL)
    for a, b in zip(tc, t):
        assert close(a.grad, b.grad, RTOL)


def test_fused_adam_matches_torch_clip_plus_adam():
    from fuxictr_b200 import zoo, arena
    gen = torch.Generator().manual_seed(5)
    lin = torch.nn.Sequential(torch.nn.Linear(13, 7), torch.nn.Linear(7, 3))
    ref = torch.nn.Sequential(torch.nn.Linear(13, 7), torch.nn.Linear(7, 3))
    ref.load_state_dict(lin.state_dict())
    lin = lin.cuda()
    ar = arena.ParamArena(lin)
    opt = arena.FusedAdam(ar, lr=1e-2, max_norm=0.5)
    ref_opt = torch.optim.Adam(ref.parameters(), lr=1e-2)
    for step in range(4):
        x = torch.randn(20, 13, generator=gen)
        opt.zero_grad()
        ref_opt.zero_grad()
        lin(x.cuda()).pow(2).sum().backward()
        # hand the torch-computed grads to the arena (this test isolates the optimizer kernel)
        for p in ar.params:
            ar.grad_view(p._b2_slot).copy_(p.grad)
        ref(x).pow(2).sum().backward()
        torch.nn.utils.clip_grad_norm_(ref.parameters(), 0.5)
        ref_opt.step()
        opt.step()
        for (k, a), (_, b) in zip(lin.state_dict().items(), ref.state_dict().items()):
            assert close(a, b, RTOL), (step, k)
    assert float(ar.G.abs().sum()) == 0.0  # zero_grad fused into the step


# ------------------------------------------------------------------ whole models vs reference goldens
def build_model(name, g, fused):
    from fuxictr_b200 import zoo
    fm = fm_from(g, g.meta["kwargs"]["embedding_dim"])
    model = getattr(zoo, name)(fm, gpu=-1, **g.meta["kwargs"])
    model.load_state_dict(g["w"])
    model.device = torch.device("cuda:0")
    model.model_to_device()
    model.compile("adam", "binary_crossentropy", 1e-3)  # optimizer over the CUDA parameters
    model.train()
    if fused:
        model.use_fused_optimizer()
    return fm, model


@pytest.mark.parametrize("name", ["DeepFM", "DCNv2", "DLRM", "xDeepFM", "DIN"])
@pytest.mark.parametrize("fused", [False, True])
def test_model_matches_reference_trajectory(name, fused):
    g = Golden("model_" + name)
    fm, model = build_model(name, g, fused)
    B = g.meta["batch"]
    mat = g["in"]["matrix"].cuda()
    batches = [fm.batch_dict(mat[i * B:(i + 1) * B]) for i in range(3)]
    # forward, loss and every gradient on batch 0
    ret = model.forward(batches[0])
    assert close(ret["y_pred"], g["out"]["y_pred"], RTOL)
    loss = model.compute_loss(ret, model.get_labels(batches[0]))
    assert close(loss, g["out"]["loss"], RTOL)
    if fused:
        model._fused_optimizer.zero_grad()
    loss.backward()
    named = dict(model.named_parameters())
    for k, ref in g["g"].items():
        assert close(named[k].grad, ref, RTOL), (k, rel_err(named[k].grad, ref))
    if fused:
        model._arena.zero_grads()
    # three optimisation steps follow the reference's (clip_grad_norm_ + Adam) trajectory
    losses = []
    for i in range(3):
        step = model.fused_train_step if fused else model.train_step
        losses.append(float(step(batches[i])))
        if i == 0:
            sd = model.state_dict()
            for k, ref in g["w1"].items():
                if ref.is_floating_point():
                    assert close(sd[k], ref, RTOL), (k, rel_err(sd[k], ref))
    assert close(torch.tensor(losses), g["out"]["step_losses"], RTOL)
    sd = model.state_dict()
    for k, ref in g["w3"].items():
        if ref.is_floating_point():
            assert close(sd[k], ref, 2e-5), (k, rel_err(sd[k], ref))


# ------------------------------------------------------------------ BASELINE sizes: oracle + properties
def criteo_shape(nf=39, vocab=25641, batch=4096, seed=0, zipf=False):
    from fuxictr_b200.schema import FeatureMap
    specs = [("C%d" % i, {"type": "categorical", "source": "", "padding_idx": 0, "vocab_size": vocab})
             for i in range(nf)]
    fm = FeatureMap.from_specs(specs, embedding_dim=16)
    gen = torch.Generator().manual_seed(seed)
    if zipf:
        u = torch.rand(batch, nf, generator=gen, dtype=torch.float64)
        ids = torch.clamp((u ** -4.0).floor(), 1, vocab - 1)            # heavy head: many duplicates
    else:
        ids = torch.randint(1, vocab, (batch, nf), generator=gen).double()
    label = (torch.rand(batch, 1, generator=gen) < 0.25).double()
    return fm, OrderedDict(specs), torch.cat([ids, label], dim=1)


@pytest.mark.parametrize("zipf", [False, True])
def test_criteo_shape_gather_scatter_vs_oracle(zipf):
    from fuxictr_b200 import layers
    from oracle import fuxictr_oracle as O
    fm, specs, mat = criteo_shape(zipf=zipf)
    torch.manual_seed(1)
    layer = layers.FeatureEmbedding(fm, 16, embedding_initializer="partial(nn.init.normal_, std=0.1)")
    state = OrderedDict((k, v.detach().clone().requires_grad_(True)) for k, v in layer.state_dict().items())
    layer = layer.cuda()
    _, X = cuda_batch(fm, mat)
    out = layer(X)
    Xc = OrderedDict((k, v) for k, v in fm.batch_dict(mat).items() if k != "label")
    ref = O.feature_embedding(specs, state, "", Xc)
    assert torch.equal(out.cpu(), ref)                                   # bit-exact at C2 size
    gout = torch.randn(out.shape, generator=torch.Generator().manual_seed(2))
    out.backward(gout.cuda())
    ref.backward(gout)
    named = dict(layer.named_parameters())
    for k, v in state.items():
        assert close(named[k].grad, v.grad, RTOL), k
    # size-independent properties: total gradient mass is conserved, padding row untouched
    total = sum(float(p.grad.double().sum()) for p in named.values())
    assert abs(total - float(gout.double().sum())) <= 1e-3 * float(gout.double().abs().sum()) ** 0.5 + 1e-3
    for p in named.values():
        assert float(p.grad[0].abs().sum()) == 0.0


@pytest.mark.parametrize("act", ["sigmoid", "relu"])
def test_criteo_shape_deepfm_step_vs_oracle(act):
    """C2 (39 fields x 25,641 rows, D=16, MLP 300-300-300, B=4096): forward, loss, every gradient
    and one optimiser step against the oracle restatement of the reference.

    The oracle is run in float32 (what the reference computes) AND in float64 (the exact answer);
    the bar is "as close to the exact result as the reference's own fp32 arithmetic":
        err(ours, fp64) <= max(1e-5, 3 * err(reference fp32, fp64))       (max-norm, relative)
    * act="sigmoid": a smooth network — the bar applies to predictions, loss and EVERY gradient.
    * act="relu" (the BASELINE config): the loss surface is only piecewise smooth.  With 3.7 M
      pre-activations per step, one of them lies within fp32 rounding of zero with probability
      O(1); two correct fp32 programs then pick different sides, which changes that sample's
      contribution to every weight gradient by ~1e-3 of the gradient (1 sample in 4096, no
      cancellation).  Predictions and loss still meet the bar; gradients are held to 1e-2
      element-wise and 1e-4 in total norm, and the exact element-wise trajectory is pinned by the
      small reference goldens (test_model_matches_reference_trajectory)."""
    from fuxictr_b200 import zoo, functional as F2
    from oracle import fuxictr_oracle as O
    fm, specs, mat = criteo_shape()
    torch.manual_seed(2019)
    model = zoo.DeepFM(fm, gpu=-1, embedding_dim=16, hidden_units=[300, 300, 300], hidden_activations=act)
    with torch.no_grad():
        for m in model.modules():
            if isinstance(m, torch.nn.Embedding):
                m.weight[1:].normal_(0, 0.05)
    state0 = OrderedDict((k, v.detach().clone()) for k, v in model.state_dict().items())
    cpu_batch = fm.batch_dict(mat)
    layout = O.mlp_layout(3, hidden_act=act)

    def logit_fn(s, X):
        emb = O.feature_embedding(specs, s, "embedding_layer.", X)
        y = O.factorization_machine(specs, s, "fm.", X, emb)
        return y + O.mlp_block(emb.flatten(start_dim=1), s, "mlp.", layout)

    def oracle_run(dtype):
        st = OrderedDict((k, v.detach().to(dtype).requires_grad_(True)) for k, v in state0.items())
        X, y = O.split_inputs(specs, ["label"], cpu_batch)
        y_pred = torch.sigmoid(logit_fn(st, X))
        loss = torch.nn.functional.binary_cross_entropy(y_pred, y.to(dtype), reduction="mean")
        loss.backward()
        return y_pred.detach(), loss.detach(), {k: v.grad for k, v in st.items()}
    y64, l64, g64 = oracle_run(torch.float64)
    y32, l32, g32 = oracle_run(torch.float32)

    model.device = torch.device("cuda:0")
    model.model_to_device()
    model.compile("adam", "binary_crossentropy", 1e-3)
    opt = model.use_fused_optimizer()
    batch = fm.batch_dict(mat.cuda())
    opt.zero_grad()
    loss, y_pred = F2.logit_bce(model.get_labels(batch), *model.forward_logits(batch))
    loss.backward()

    def bar(ours, ref32, truth, what):
        e_ours, e_ref = rel_err(ours, truth), rel_err(ref32, truth)
        assert e_ours <= max(RTOL, 3 * e_ref), (what, e_ours, e_ref)
    bar(y_pred, y32, y64, "y_pred")
    bar(loss, l32, l64, "loss")
    named = dict(model.named_parameters())
    if act == "sigmoid":
        for k in g64:
            bar(named[k].grad, g32[k], g64[k], k)
    else:
        for k in g64:
            assert rel_err(named[k].grad, g64[k]) <= 1e-2, (k, rel_err(named[k].grad, g64[k]))
        ours = torch.cat([named[k].grad.flatten().double().cpu() for k in g64])
        truth = torch.cat([g64[k].flatten() for k in g64])
        assert float((ours - truth).norm()) <= 1e-4 * float(truth.norm())
    # one optimiser step, then the next loss (weights feed back through the whole model)
    tr = O.OracleTrainer(state0, lambda s, X: torch.sigmoid(logit_fn(s, X)), specs, ["label"])
    tr.train_step(cpu_batch)
    loss_ref2 = float(O.bce_mean(*tr.forward(cpu_batch)))
    opt.step()
    with torch.no_grad():
        loss2, _ = F2.logit_bce(model.get_labels(batch), *model.forward_logits(batch))
    assert abs(float(loss2) - loss_ref2) <= RTOL * abs(loss_ref2)


def test_scatter_linearity_and_idempotent_gather():
    """Properties that hold at any size: gather(x) twice is identical; scatter(a*g1 + g2) ==
    a*scatter(g1) + scatter(g2) up to fp32 rounding."""
    from fuxictr_b200 import layers
    fm, specs, mat = criteo_shape(nf=26, vocab=100003, batch=8192, seed=9, zipf=True)
    layer = layers.FeatureEmbedding(fm, 16).cuda()
    _, X = cuda_batch(fm, mat)
    o1, o2 = layer(X), layer(X)
    assert torch.equal(o1, o2)
    gen = torch.Generator(device="cuda").manual_seed(3)
    g1 = torch.randn(o1.shape, device="cuda", generator=gen)
    g2 = torch.randn(o1.shape, device="cuda", generator=gen)

    def scat(gout):
        for p in layer.parameters():
            p.grad = None
        layer(X).backward(gout)
        return torch.cat([p.grad.flatten() for p in layer.parameters()])
    lhs = scat(2.5 * g1 + g2)
    rhs = 2.5 * scat(g1) + scat(g2)
    assert close(lhs, rhs, RTOL)


def test_gather_hot_row_staging_is_bit_identical():
    """Shared-memory staging of the leading (most frequent) rows: same bytes out, Zipf-skewed ids that
    mix staged rows, cold rows, the padding row and a table shorter than the staging depth."""
    from fuxictr_b200 import functional as F2
    sys.path.insert(0, ROOT)
    import bench
    D, B = 16, 32768
    vocabs = [4000] * 20 + [9] + [250000] * 18            # one table with fewer rows than hot_rows
    tables = [torch.randn(v, D, device="cuda") for v in vocabs]
    ids = bench.zipf_ids(B, vocabs, 1.05, seed=3, device="cuda")
    ids[::97, 0] = 0                                       # padding rows
    idx = [ids[:, i] for i in range(len(vocabs))]
    plan = F2.GatherPlan([F2.GatherField("C%d" % i, i, D, padding_idx=0) for i in range(len(vocabs))])
    with torch.no_grad():
        base = F2.embed_gather(plan, idx, tables).clone()
        plan.hot_rows = 16
        hot = F2.embed_gather(plan, idx, tables)
    assert torch.equal(base, hot)
    want = torch.cat([t[ids[:, i].long()] for i, t in enumerate(tables)], dim=1)
    assert torch.equal(hot, want)


# ------------------------------------------------------------------ wgmma tensor-core GEMM
TC_SHAPES = [(128, 32, 32), (128, 96, 64), (256, 160, 128), (4096, 300, 624), (4096, 624, 300),
             (300, 624, 4096), (1000, 500, 432), (77, 45, 36), (129, 257, 1000), (8192, 624, 624)]


@pytest.mark.parametrize("M,N,K", TC_SHAPES)
@pytest.mark.parametrize("mode", ["tf32", "tf32x3"])
def test_gemm_tc_vs_fp64(M, N, K, mode):
    from fuxictr_b200 import functional as F2
    gen = torch.Generator().manual_seed(M + 3 * N + 7 * K)
    a = torch.randn(M, K, generator=gen)
    b = torch.randn(N, K, generator=gen)
    bias = torch.randn(N, generator=gen)
    ref = a.double() @ b.double().t() + bias.double()
    out = torch.full((M, N), float("nan"), device="cuda")
    F2.set_matmul_precision(mode)
    try:
        F2.gemm_nt(a.cuda(), b.cuda(), out, bias=bias.cuda())
    finally:
        F2.set_matmul_precision("fp32")
    torch.cuda.synchronize()
    assert not torch.isnan(out).any()
    err = rel_err(out, ref)
    # single-pass TF32 truncates operands to 10 mantissa bits; 3xTF32 must be fp32-class
    assert err <= (3e-3 if mode == "tf32" else 2e-6), err


def test_gemm_tc_epilogues():
    from fuxictr_b200 import functional as F2
    from fuxictr_b200._lib import B2_ACT_RELU
    gen = torch.Generator().manual_seed(8)
    M, N, K = 512, 200, 96
    a, b = torch.randn(M, K, generator=gen), torch.randn(N, K, generator=gen)
    bias, mul, add = torch.randn(N, generator=gen), torch.randn(M, N, generator=gen), torch.randn(M, N, generator=gen)
    z = a.double() @ b.double().t() + bias.double()
    F2.set_matmul_precision("tf32x3")
    try:
        out = torch.empty(M, N, device="cuda")
        F2.gemm_nt(a.cuda(), b.cuda(), out, bias=bias.cuda(), act=B2_ACT_RELU)
        assert close(out, torch.relu(z), RTOL)
        F2.gemm_nt(a.cuda(), b.cuda(), out, bias=bias.cuda(), mul=mul.cuda(), add=add.cuda())
        assert close(out, add.double() + mul.double() * z, RTOL)
        base = torch.randn(M, N, generator=gen)
        out = base.cuda().clone()
        F2.gemm_nt(a.cuda(), b.cuda(), out, accumulate=True)
        assert close(out, base.double() + a.double() @ b.double().t(), RTOL)
    finally:
        F2.set_matmul_precision("fp32")


# MN-major fp32 operands are TMA tensors with rows as the contiguous dimension: rows % 4 == 0 (16-byte pitch)
MN_SHAPES = [(128, 32, 32), (300, 624, 4096), (4096, 624, 300), (624, 300, 8192), (76, 44, 36), (132, 260, 1000),
             (64, 64, 432)]


@pytest.mark.parametrize("M,N,K", MN_SHAPES)
@pytest.mark.parametrize("a_mn,b_mn", [(False, False), (False, True), (True, True), (True, False)])
@pytest.mark.parametrize("mode", ["tf32", "tf32x3", "tf32x3_aux", "bf16"])
def test_gemm_tc_mn_major_operands_vs_fp64(M, N, K, a_mn, b_mn, mode):
    """The contraction reads operands as they lie in memory: A stored (K, M) and/or B stored (K, N)
    (the dgrad / wgrad layouts of nn.Linear) through MN-major matrix descriptors — no transpose."""
    from fuxictr_b200 import functional as F2
    gen = torch.Generator().manual_seed(M + 3 * N + 7 * K + a_mn + 2 * b_mn)
    a = torch.randn(M, K, generator=gen)
    b = torch.randn(N, K, generator=gen)
    ref = a.double() @ b.double().t()
    a_dev = (a.t().contiguous() if a_mn else a).cuda()
    b_dev = (b.t().contiguous() if b_mn else b).cuda()
    out = torch.full((M, N), float("nan"), device="cuda")
    # "tf32x3": small parts derived in shared memory inside the GEMM (default); "tf32x3_aux": read from HBM
    F2.set_x3_inline(mode != "tf32x3_aux")
    mode = mode.replace("_aux", "")
    F2.set_matmul_precision(mode)
    try:
        out_aux = F2.empty_aux(M, N, "cuda") if mode == "bf16" else None
        F2.gemm_ex(a_dev, b_dev, out, a_mn=a_mn, b_mn=b_mn, a_small=F2.make_aux(a_dev), b_small=F2.make_aux(b_dev),
                   out_small=out_aux)
    finally:
        F2.set_matmul_precision("fp32")
        F2.set_x3_inline(True)
    torch.cuda.synchronize()
    assert not torch.isnan(out).any()
    if mode == "bf16":      # checker: the same contraction of the bf16-rounded operands, in float64
        ref = a.bfloat16().double() @ b.bfloat16().double().t()
        assert rel_err(out, ref) <= 3e-5          # fp32 (truncating) accumulation of up to 8192 exact products
        assert torch.equal(out_aux, out.bfloat16())          # the epilogue's bf16 copy is RN(out)
    else:
        err = rel_err(out, ref)
        assert err <= (3e-3 if mode == "tf32" else 2e-6), err


@pytest.mark.parametrize("act_bwd", ["none", "relu", "sigmoid"])
def test_gemm_tc_fused_backward_epilogue(act_bwd):
    """dgrad epilogue = activation backward of the producer + 3xTF32 small part + bias gradient."""
    from fuxictr_b200 import functional as F2
    from fuxictr_b200._lib import B2_ACT_NONE, B2_ACT_RELU, B2_ACT_SIGMOID
    code = {"none": B2_ACT_NONE, "relu": B2_ACT_RELU, "sigmoid": B2_ACT_SIGMOID}[act_bwd]
    gen = torch.Generator().manual_seed(11)
    M, N, K = 700, 200, 96            # dX (M, N) = dZ (M, K) @ W (K, N): W is the MN-major B operand
    dz, w = torch.randn(M, K, generator=gen), torch.randn(K, N, generator=gen)
    y = torch.rand(M, N, generator=gen) - (0.5 if act_bwd == "relu" else 0.0)
    acc = dz.double() @ w.double()
    if act_bwd == "relu":
        want = torch.where(y.double() > 0, acc, torch.zeros_like(acc))
    elif act_bwd == "sigmoid":
        want = acc * ((1 - y.double()) * y.double())
    else:
        want = acc
    dzc, wc = dz.cuda(), w.cuda()
    out = torch.empty(M, N, device="cuda")
    out_small = torch.full((M, N), float("nan"), device="cuda")
    colsum = torch.full((N,), float("nan"), device="cuda")
    F2.gemm_ex(dzc, wc, out, b_mn=True, a_small=F2.split_tf32(dzc), b_small=F2.split_tf32(wc),
               ybwd=y.cuda() if code != B2_ACT_NONE else None, act_bwd=code, out_small=out_small, colsum=colsum)
    assert close(out, want, RTOL)
    assert torch.equal(out_small, F2.split_tf32(out))                       # exactly the consumer's small part
    assert close(colsum, want.sum(dim=0), RTOL, atol=1e-5 * float(want.abs().sum(dim=0).max()))


@pytest.mark.parametrize("mode", ["tf32x3", "tf32x3_aux", "tf32", "bf16"])
@pytest.mark.parametrize("dims,acts,B", [((624, 300, 300, 300, 1), ("relu", "relu", "relu", None), 4096),
                                         ((325, 64, 64, 64, 1), ("relu", "relu", "relu", "sigmoid"), 1000),
                                         ((128, 64, 1), ("sigmoid", None), 777),
                                         ((432, 500, 500, 500), ("relu", "relu", "relu"), 2048),
                                         ((40, 18, 36, 1), ("relu", None, None), 130)])
def test_mlp_chain_matches_torch_autograd(mode, dims, acts, B):
    """MLP_Block as one autograd node (cross-layer fused epilogues, MN-major dgrad/wgrad, fused head)
    against the reference's ops (nn.Linear / ReLU / Sigmoid autograd) in float64."""
    from fuxictr_b200 import layers, functional as F2
    torch.manual_seed(sum(dims) + B)
    hidden = list(dims[1:-1]) if dims[-1] == 1 else list(dims[1:])
    out_dim = 1 if dims[-1] == 1 else None
    hid_acts = [({"relu": "ReLU", "sigmoid": "Sigmoid", None: None}[a]) for a in acts[:len(hidden)]]
    out_act = None
    if out_dim is not None and acts[-1] is not None:
        out_act = {"relu": "ReLU", "sigmoid": "Sigmoid"}[acts[-1]]
    mlp = layers.MLP_Block(input_dim=dims[0], hidden_units=hidden, hidden_activations=hid_acts, output_dim=out_dim,
                           output_activation=out_act)
    ref = copy.deepcopy(mlp).double()
    mlp = mlp.cuda()
    gen = torch.Generator().manual_seed(B)
    x = torch.randn(B, dims[0], generator=gen)
    gout = torch.randn(B, dims[-1], generator=gen)
    xr = x.double().requires_grad_(True)
    yr = ref.mlp(xr)
    yr.backward(gout.double())
    xg = x.cuda().requires_grad_(True)
    F2.set_x3_inline(mode != "tf32x3_aux")
    mode = mode.replace("_aux", "")
    F2.set_matmul_precision(mode)
    try:
        yg = mlp(xg)
        assert type(yg.grad_fn).__name__.startswith("_MLPChain")
        yg.backward(gout.cuda())
    finally:
        F2.set_matmul_precision("fp32")
        F2.set_x3_inline(True)
    if mode == "tf32x3":                    # the parity-grade arithmetic: element-wise, north_star's 1e-5
        assert close(yg, yr, RTOL)
        assert close(xg.grad, xr.grad, RTOL, atol=RTOL * float(xr.grad.abs().max()))
        for (k, pg), (_, pr) in zip(mlp.named_parameters(), ref.named_parameters()):
            assert close(pg.grad, pr.grad, RTOL, atol=RTOL * float(pr.grad.abs().max())), k
        return
    # Single-pass modes truncate (TF32, eps ~1e-3 per contraction) or round (bf16, ~4e-3) every operand, so
    # the fraction ~0.8*eps of pre-activations that sit within eps of zero take the other ReLU branch than
    # in float64; each such unit moves its row of the gradients by that unit's whole contribution, hence a
    # gradient error of ~sqrt(0.8*eps) of the Frobenius norm (3 % TF32, 6-8 % bf16) however exact the GEMMs
    # are (each one is held to its own bar in test_gemm_tc_*; torch's allow_tf32 behaves the same).  These
    # are throughput modes, not parity modes: forward within a few eps, gradients within that kink bound.
    tol_y, tol = {"tf32": (1e-2, 6e-2), "bf16": (3e-2, 1.5e-1)}[mode]

    def fro(a, b):
        b = b.to(torch.float64)
        return float((a.detach().cpu().double() - b.cpu()).norm() / b.norm().clamp_min(1e-30))
    assert fro(yg, yr) <= tol_y
    assert fro(xg.grad, xr.grad) <= tol
    for (k, pg), (_, pr) in zip(mlp.named_parameters(), ref.named_parameters()):
        assert fro(pg.grad, pr.grad) <= tol, k


@pytest.mark.parametrize("name", ["DeepFM", "DCNv2", "DLRM", "xDeepFM", "DIN"])
def test_model_trajectory_tf32x3(name):
    """The tensor-core path in its parity-grade arithmetic (3xTF32) follows the reference too."""
    from fuxictr_b200 import functional as F2
    F2.set_matmul_precision("tf32x3")
    try:
        test_model_matches_reference_trajectory(name, True)
    finally:
        F2.set_matmul_precision("fp32")


def test_criteo_shape_deepfm_step_tf32x3_vs_oracle():
    from fuxictr_b200 import functional as F2
    F2.set_matmul_precision("tf32x3")
    try:
        test_criteo_shape_deepfm_step_vs_oracle("sigmoid")
        test_criteo_shape_deepfm_step_vs_oracle("relu")
    finally:
        F2.set_matmul_precision("fp32")


# ------------------------------------------------------------------ fused sparse front
@pytest.mark.parametrize("want_fm", [True, False])
@pytest.mark.parametrize("dim,nf", [(16, 39), (8, 10), (4, 3), (40, 26), (64, 5)])
def test_fused_front_matches_separate_modules(want_fm, dim, nf):
    """gather+FM+LR in one launch == FeatureEmbedding, InnerProductInteraction, LogisticRegression
    run as separate (already golden-checked) launches: embeddings bit-exact, logits/grads 1e-5."""
    from fuxictr_b200 import layers
    from fuxictr_b200.schema import FeatureMap
    specs = [("C%d" % i, {"type": "categorical", "source": "", "padding_idx": 0, "vocab_size": 50 + 7 * i})
             for i in range(nf)]
    fm = FeatureMap.from_specs(specs, embedding_dim=dim)
    torch.manual_seed(nf * 100 + dim)
    emb_layer = layers.FeatureEmbedding(fm, dim, embedding_initializer="partial(nn.init.normal_, std=0.1)").cuda()
    fmach = layers.FactorizationMachine(fm).cuda()
    with torch.no_grad():
        for p in fmach.parameters():
            p.normal_(0, 0.3)
        for m in fmach.modules():
            if isinstance(m, torch.nn.Embedding):
                m.weight[0].zero_()
    B = 257
    gen = torch.Generator().manual_seed(1)
    ids = torch.cat([torch.randint(0, s["vocab_size"], (B, 1), generator=gen) for _, s in specs], dim=1)
    mat = torch.cat([ids.double(), torch.zeros(B, 1, dtype=torch.float64)], dim=1).cuda()
    X = OrderedDict((k, v) for k, v in fm.batch_dict(mat).items() if k != "label")
    g_emb = torch.randn(B, nf, dim, generator=gen).cuda()
    g_log = torch.randn(B, 1, generator=gen).cuda()

    def run(fused):
        for p in list(emb_layer.parameters()) + list(fmach.parameters()):
            p.grad = None
        if fused:
            emb, logit = layers.fused_front(emb_layer, fmach.lr_layer, X, want_fm)
        else:
            emb = emb_layer(X)
            logit = fmach(X, emb) if want_fm else fmach.lr_layer(X)
        ((emb * g_emb).sum() + (logit * g_log).sum()).backward()
        grads = [p.grad.clone() for p in list(emb_layer.parameters()) + list(fmach.parameters())]
        return emb.detach(), logit.detach(), grads
    e0, l0, g0 = run(False)
    e1, l1, g1 = run(True)
    assert torch.equal(e0, e1)
    assert close(l1, l0, RTOL)
    scale = max(float(g.abs().max()) for g in g0)
    for a, b in zip(g1, g0):
        assert close(a, b, RTOL, atol=RTOL * scale)


@pytest.mark.parametrize("F_,D,units,B", [(39, 16, [16, 16, 16], 130), (26, 10, [32, 8], 77), (5, 4, [3], 9)])
def test_cin_fused_vs_oracle(F_, D, units, B):
    """Fused CIN layers (Hadamard tensor never materialised) at xDeepFM shapes against the oracle's
    einsum + Conv1d restatement (compressed_interaction_net.py:64-76)."""
    from fuxictr_b200 import layers
    from oracle import fuxictr_oracle as O
    torch.manual_seed(F_ + D)
    layer = layers.CompressedInteractionNet(F_, units)
    with torch.no_grad():
        for p in layer.parameters():
            p.normal_(0, 0.2)
    state = OrderedDict((k, v.detach().clone().requires_grad_(True)) for k, v in layer.state_dict().items())
    gen = torch.Generator().manual_seed(B)
    emb = torch.randn(B, F_, D, generator=gen) * 0.5
    gout = torch.randn(B, 1, generator=gen)
    e_ref = emb.clone().requires_grad_(True)
    y_ref = O.compressed_interaction_net(e_ref, state, "", units)
    y_ref.backward(gout)
    layer = layer.cuda()
    e = emb.cuda().requires_grad_(True)
    y = layer(e)
    y.backward(gout.cuda())
    assert close(y, y_ref, RTOL)
    assert close(e.grad, e_ref.grad, RTOL)
    named = dict(layer.named_parameters())
    scale = max(float(v.grad.abs().max()) for v in state.values())
    for k, v in state.items():
        assert close(named[k].grad, v.grad, RTOL, atol=RTOL * scale), k


# ------------------------------------------------------------------ lazy (row-wise) evaluation of dense Adam
def _lazy_pair(name="DeepFM"):
    from fuxictr_b200 import zoo
    from fuxictr_b200.schema import FeatureMap
    specs = [("C%d" % i, {"type": "categorical", "source": "", "padding_idx": 0, "vocab_size": 200 + 17 * i})
             for i in range(9)]
    fm = FeatureMap.from_specs(specs, embedding_dim=8)
    if name == "DeepFM":
        kwargs = dict(embedding_dim=8, hidden_units=[32, 16])
    else:
        kwargs = dict(embedding_dim=8, dnn_hidden_units=[32, 16], cin_hidden_units=[6, 5])

    def build(lazy, max_norm):
        torch.manual_seed(123)
        m = getattr(zoo, name)(fm, gpu=0, **kwargs)
        with torch.no_grad():
            for mod in m.modules():
                if isinstance(mod, torch.nn.Embedding):
                    mod.weight[1:].normal_(0, 0.3)
        m._max_gradient_norm = max_norm
        m.use_fused_optimizer(lazy_tables=lazy)
        return m
    return fm, specs, build


def _batch(specs, gen, B=48):
    ids = torch.cat([torch.randint(0, s["vocab_size"], (B, 1), generator=gen) for _, s in specs], 1)
    return torch.cat([ids.double(), (torch.rand(B, 1, generator=gen) < 0.4).double()], 1).cuda()


def test_lazy_adam_optimizer_is_bit_identical_given_identical_gradients():
    """The reference's Adam moves EVERY table row at every step (zero-gradient rows included).  Lazy
    mode touches only the rows a batch touches and REPLAYS the missed zero-gradient updates on demand.
    Given bit-identical gradients (copied from the dense model: backward atomics make two backward
    passes differ in the last bit) the parameters and both Adam moments after 8 steps with rows idle
    for 0..7 steps must be BIT-identical, and so must the embeddings the fused front reads from the
    not-yet-materialised tables."""
    from fuxictr_b200 import layers
    fm, specs, build = _lazy_pair("DeepFM")
    dense, lazy = build(False, 10.0), build(True, 10.0)
    lz = lazy._lazy
    gen = torch.Generator().manual_seed(9)
    dn, ln = dict(dense.named_parameters()), dict(lazy.named_parameters())
    for step in range(8):
        mat = _batch(specs, gen)
        batch = fm.batch_dict(mat)
        dense._fused_optimizer.zero_grad()
        lazy._fused_optimizer.zero_grad()
        from fuxictr_b200 import functional as F2
        loss, _ = F2.logit_bce(dense.get_labels(batch), *dense.forward_logits(batch))
        loss.backward()
        # hand the dense model's gradients to the lazy arena, parameter by parameter
        for k, p in dn.items():
            q = ln[k]
            lazy._arena.grad_view(q._b2_slot).copy_(dense._arena.grad_view(p._b2_slot))
        # worklist = every (table, row) of this batch except padding rows, exactly once
        rows = []
        for p in lz.tables:
            name = [k for k, q in ln.items() if q is p][0]
            feat = name.split("embedding_layers.")[1].split(".")[0]
            col = fm.get_column_index(feat)
            r = mat[:, col].long().unique()
            rows.append(r[r != 0] + p._b2_grow_base)
        wl = torch.cat(rows).int()
        lz.worklist[:wl.numel()].copy_(wl)
        lz.counter.fill_(wl.numel())
        dense._fused_optimizer.step()
        lazy._fused_optimizer.step()
    torch.cuda.synchronize()
    # the fused front reads stale rows through the replay: must equal the dense tables bit for bit
    probe = _batch(specs, torch.Generator().manual_seed(77), B=256)
    X = OrderedDict((k, v) for k, v in fm.batch_dict(probe).items() if k != "label")
    with torch.no_grad():
        e_dense, l_dense = layers.fused_front(dense.embedding_layer, dense.fm.lr_layer, X, True)
        e_lazy, l_lazy = layers.fused_front(lazy.embedding_layer, lazy.fm.lr_layer, X, True)
    assert torch.equal(e_dense, e_lazy) and torch.equal(l_dense, l_lazy)
    stale = int((lz.last_step < int(lazy._fused_optimizer.step_dev)).sum())
    assert stale > 0                                        # rows really were left behind
    lazy.materialize_tables()
    torch.cuda.synchronize()
    for k, p in dn.items():
        q = ln[k]
        assert torch.equal(p.data, q.data), k
        for a0, a1 in ((dense._fused_optimizer.M, lazy._fused_optimizer.M),
                       (dense._fused_optimizer.V, lazy._fused_optimizer.V)):
            s0, s1 = p._b2_slot, q._b2_slot
            assert torch.equal(a0[s0.offset:s0.offset + s0.numel], a1[s1.offset:s1.offset + s1.numel]), k
    assert float(lazy._arena.G.abs().sum()) == 0.0          # gradient arena left all-zero


@pytest.mark.parametrize("max_norm", [10.0, 0.05])
@pytest.mark.parametrize("name", ["DeepFM", "xDeepFM"])
def test_lazy_adam_training_matches_dense_adam(name, max_norm):
    """End to end (own backward in each model, clipping inactive and active): lazy and dense
    training agree to 1e-6 — the residual is the atomic summation order of the backward kernels and
    of the gradient norm, which also differs between two runs of the SAME mode."""
    fm, specs, build = _lazy_pair(name)
    dense, lazy = build(False, max_norm), build(True, max_norm)
    # seed 9 put an Adam element of DeepFM's C7 table at a near-zero gradient, where the atomic-order residual
    # moved it 3.5e-6 between two DENSE runs as well
    gen = torch.Generator().manual_seed(10)
    for step in range(7):
        mat = _batch(specs, gen)
        l0 = dense.fused_train_step(fm.batch_dict(mat))
        l1 = lazy.fused_train_step(fm.batch_dict(mat))
        assert abs(float(l0) - float(l1)) <= 1e-6 * abs(float(l0)), step
    lazy.materialize_tables()
    torch.cuda.synchronize()
    sd0, sd1 = dense.state_dict(), lazy.state_dict()
    for k in sd0:
        assert close(sd0[k], sd1[k], 1e-6, atol=1e-9), k
    assert float(lazy._arena.G.abs().sum()) == 0.0


# ------------------------------------------------------------------ the other BASELINE configs at full shape
def _taobao_specs():
    specs = [("item_id", {"type": "categorical", "source": "", "padding_idx": 0, "vocab_size": 400000}),
             ("cate_id", {"type": "categorical", "source": "", "padding_idx": 0, "vocab_size": 10000})]
    specs += [("f%d" % i, {"type": "categorical", "source": "", "padding_idx": 0, "vocab_size": 20000}) for i in range(23)]
    specs += [("click_history", {"type": "sequence", "source": "", "padding_idx": 0, "vocab_size": 400000, "max_len": 50,
                                 "share_embedding": "item_id", "feature_encoder": None}),
              ("cate_history", {"type": "sequence", "source": "", "padding_idx": 0, "vocab_size": 10000, "max_len": 50,
                                "share_embedding": "cate_id", "feature_encoder": None})]
    return specs


def _baseline_setup(config):
    """(fm, spec_map, mat, model, pred, state0) of one BASELINE config at full shape: the CPU model with its
    tables initialised like the C2 test, the oracle's y_pred function and the initial state."""
    from fuxictr_b200 import zoo
    from fuxictr_b200.schema import FeatureMap
    from oracle import fuxictr_oracle as O
    gen = torch.Generator().manual_seed(5)
    if config == "C4_DIN":
        specs, B = _taobao_specs(), 2048
    elif config == "C5_DLRM_shape":
        specs, B = [("C%d" % i, {"type": "categorical", "source": "", "padding_idx": 0, "vocab_size": 100000})
                    for i in range(26)], 8192
    else:
        specs = [("C%d" % i, {"type": "categorical", "source": "", "padding_idx": 0, "vocab_size": 25641})
                 for i in range(39)]
        B = 8192 if config == "C3_DCNv2" else 4096
    fm = FeatureMap.from_specs(specs, embedding_dim=16)
    cols = []
    for name, sp in specs:
        if sp["type"] == "sequence":
            ids = torch.randint(1, sp["vocab_size"], (B, 50), generator=gen)
            lens = torch.randint(1, 51, (B, 1), generator=gen)
            cols.append((ids * (torch.arange(50).view(1, -1) < lens)).double())
        else:
            cols.append(torch.randint(1, sp["vocab_size"], (B, 1), generator=gen).double())
    mat = torch.cat(cols + [(torch.rand(B, 1, generator=gen) < 0.25).double()], dim=1)
    torch.manual_seed(2019)
    spec_map = OrderedDict(specs)
    if config == "C3_DCNv2":
        model = zoo.DCNv2(fm, gpu=-1, embedding_dim=16, model_structure="parallel", num_cross_layers=3,
                          parallel_dnn_hidden_units=[500, 500, 500])
        pred = lambda s, X: torch.sigmoid(O.dcnv2_logit(spec_map, s, X, 3, 3))
    elif config == "C4_DIN":
        model = zoo.DIN(fm, gpu=-1, embedding_dim=16, dnn_hidden_units=[500, 500, 500], attention_hidden_units=[64],
                        attention_hidden_activations="Dice")
        pred = lambda s, X: O.din_pred(spec_map, s, X, 16, [("item_id", "cate_id")],
                                       [("click_history", "cate_history")], 1, 3, training=True)
    elif config == "C5_DLRM_shape":
        model = zoo.DLRM(fm, gpu=-1, embedding_dim=16, top_mlp_units=[64, 64, 64], interaction_op="dot")
        pred = lambda s, X: O.dlrm_pred(spec_map, s, X, 3)
    else:
        model = zoo.xDeepFM(fm, gpu=-1, embedding_dim=16, dnn_hidden_units=[400, 400, 400], cin_hidden_units=[16, 16, 16])
        pred = lambda s, X: torch.sigmoid(O.xdeepfm_logit(spec_map, s, X, [16, 16, 16], 3))
    with torch.no_grad():
        for m in model.modules():
            if isinstance(m, torch.nn.Embedding):
                m.weight[1:].normal_(0, 0.05)
    state0 = OrderedDict((k, v.detach().clone()) for k, v in model.state_dict().items())
    return fm, spec_map, mat, model, pred, state0


@pytest.mark.parametrize("config", ["C3_DCNv2", "C4_DIN", "C5_DLRM_shape", "C2_xDeepFM"])
def test_baseline_shapes_forward_and_step(config):
    """BASELINE.json configs[2..4] (and xDeepFM at the C2 shape) at their full batch / field / sequence
    sizes: predictions and loss against the oracle (1e-5), then one fused training step must run and
    lower-bound sanity (finite loss, gradient arena consumed).  C5's 200 M-row vocabulary is reduced to
    26 x 100 k rows so that the CPU oracle can hold it; the shapes that drive the kernels
    (26 fields, D=16, 325 pair products, top MLP 64-64-64, batch 8192) are the real ones."""
    from oracle import fuxictr_oracle as O
    fm, spec_map, mat, model, pred, state0 = _baseline_setup(config)
    tr = O.OracleTrainer(state0, pred, spec_map, ["label"])
    with torch.no_grad():
        y_ref, y_true = tr.forward(fm.batch_dict(mat))
        loss_ref = O.bce_mean(y_ref, y_true)
    model.device = torch.device("cuda:0")
    model.model_to_device()
    model.compile("adam", "binary_crossentropy", 1e-3)
    model.train()
    batch = fm.batch_dict(mat.cuda())
    with torch.no_grad():
        y = model.forward(batch)["y_pred"]
    assert close(y, y_ref, RTOL), rel_err(y, y_ref)
    model.use_fused_optimizer()
    if config == "C4_DIN":      # fresh Dice running statistics for the training step (the forward above updated them)
        model.load_state_dict({k: v.cuda() for k, v in state0.items()})
    loss = model.fused_train_step(batch)
    torch.cuda.synchronize()
    assert close(loss, loss_ref, RTOL), (float(loss), float(loss_ref))
    assert float(model._arena.G.abs().sum()) == 0.0
    assert all(torch.isfinite(p).all() for p in model.parameters())


@pytest.mark.parametrize("config", ["C3_DCNv2", "C4_DIN", "C5_DLRM_shape", "C2_xDeepFM"])
def test_baseline_shapes_gradients_and_step_vs_oracle(config):
    """The configs of test_baseline_shapes_forward_and_step: every parameter gradient, then the loss after
    one fused Adam step, against the oracle — the bar of test_criteo_shape_deepfm_step_vs_oracle.  The
    oracle runs in float32 and float64; predictions and loss must satisfy
        err(ours, fp64) <= max(1e-5, 3 * err(reference fp32, fp64)).
    All four networks have ReLU layers.  One pre-activation within fp32 rounding of zero takes the other branch
    than in float64 and moves its sample's whole contribution (see the C2 test), so every gradient is held to
    1e-2 element-wise (or 3x the fp32 reference's own error, when its kinks land off the float64 side too) and
    to 1e-4 in total norm.  A dense weight sums that contribution over the batch and always meets the
    element-wise bound.  A touched table row is mostly one sample's contribution, which such a flip moves by up
    to ~2 % of the table's largest gradient, so table rows beyond the bound are accepted only when they all
    belong to at most two samples, each of which has a ReLU pre-activation in the float64 oracle within 1e-5
    of its layer's RMS of zero: the kink is shown, not assumed."""
    from fuxictr_b200 import functional as F2
    from oracle import fuxictr_oracle as O
    fm, spec_map, mat, model, pred, state0 = _baseline_setup(config)
    cpu_batch = fm.batch_dict(mat)

    pre = []            # the float64 oracle's ReLU inputs, (batch, units) per layer

    def oracle_run(dtype):
        st = OrderedDict((k, v.to(dtype) if v.is_floating_point() else v) for k, v in state0.items())
        tr = O.OracleTrainer(st, pred, spec_map, ["label"])
        relu = torch.relu
        if dtype == torch.float64:
            torch.relu = lambda x: (pre.append(x.detach()), relu(x))[1]
        try:
            y_pred, y = tr.forward(cpu_batch)
        finally:
            torch.relu = relu
        loss = O.bce_mean(y_pred, y.to(dtype))
        loss.backward()
        return y_pred.detach(), loss.detach(), tr.state
    y64, l64, s64 = oracle_run(torch.float64)
    y32, l32, s32 = oracle_run(torch.float32)

    model.device = torch.device("cuda:0")
    model.model_to_device()
    model.compile("adam", "binary_crossentropy", 1e-3)
    model.train()
    opt = model.use_fused_optimizer()
    batch = fm.batch_dict(mat.cuda())
    opt.zero_grad()
    if hasattr(model, "forward_logits"):
        loss, y_pred = F2.logit_bce(model.get_labels(batch), *model.forward_logits(batch))
    else:
        y_pred = model.forward(batch)["y_pred"]
        loss = model.compute_loss({"y_pred": y_pred}, model.get_labels(batch))
    loss.backward()

    def bar(ours, ref32, truth, what):
        e_ours, e_ref = rel_err(ours, truth), rel_err(ref32, truth)
        assert e_ours <= max(RTOL, 3 * e_ref), (what, e_ours, e_ref)
    bar(y_pred, y32, y64, "y_pred")
    bar(loss, l32, l64, "loss")
    named = OrderedDict((k, p) for k, p in model.named_parameters() if p.requires_grad)
    assert len(named) > 0
    B = mat.shape[0]
    bad = []            # (table, row) beyond the element-wise bound
    for k, p in named.items():
        assert p.grad is not None, k
        g, g64 = p.grad.double().cpu(), s64[k].grad
        e_ours, e_ref = rel_err(g, g64), rel_err(s32[k].grad, g64)
        lim = max(1e-2, 3 * e_ref)
        if ".embedding_layers." not in k:
            assert e_ours <= lim, (k, e_ours, e_ref)
            continue
        rows = torch.nonzero((g - g64).abs().amax(dim=1) > lim * float(g64.abs().max())).view(-1)
        bad += [(k, int(r)) for r in rows]

    def samples_of(k, row):
        """Samples whose ids (of any feature reading table k) include `row`."""
        feat = k.rsplit(".embedding_layers.", 1)[1][:-len(".weight")]
        feats = [f for f, sp in spec_map.items()
                 if f == feat or ("lr_layer." not in k and sp.get("share_embedding") == feat)]
        return torch.stack([(cpu_batch[f].long().view(B, -1) == row).any(1) for f in feats]).any(0)
    covers, kinks = [samples_of(k, r) for k, r in bad], []
    assert all(bool(c.any()) for c in covers), ("gradient in a row no sample reads", bad[:10])
    while covers:
        s = int(torch.stack(covers).sum(0).argmax())
        kinks.append(s)
        covers = [c for c in covers if not c[s]]
    assert len(kinks) <= 2, (kinks, bad[:10])
    for s in kinks:
        margin = min(float(z[s].abs().min()) / float(z.pow(2).mean().sqrt()) for z in pre)
        assert margin <= 1e-5, ("table rows off without a ReLU kink", s, margin, bad[:10])
    ours = torch.cat([p.grad.flatten().double().cpu() for p in named.values()])
    truth = torch.cat([s64[k].grad.flatten() for k in named])
    assert float((ours - truth).norm()) <= 1e-4 * float(truth.norm())
    # one optimiser step, then the next loss (weights feed back through the whole model)
    tr = O.OracleTrainer(state0, pred, spec_map, ["label"])
    tr.train_step(cpu_batch)
    loss_ref2 = float(O.bce_mean(*tr.forward(cpu_batch)))
    opt.step()
    with torch.no_grad():
        loss2 = model.compute_loss(model.forward(batch), model.get_labels(batch))
    assert abs(float(loss2) - loss_ref2) <= RTOL * abs(loss_ref2), (float(loss2), loss_ref2)


# ------------------------------------------------------------------ C5 at its full shape, by properties
def test_c5_full_shape_lookup_properties():
    """BASELINE configs C5: 26 sparse fields, 200 M rows x 16 fp32 (12.8 GB of tables), batch 65,536.  No CPU
    oracle finishes at this size, so the bar is properties: the fused gather equals the reference's own op
    on every field (`F.embedding` on the same device tensors — feature_embedding.py:284-285 — bit for bit),
    is idempotent, and its backward conserves gradient mass, leaves padding rows untouched and matches an
    index_add_ of the same rows."""
    free, _ = torch.cuda.mem_get_info()
    if free < 60e9:
        pytest.skip("needs ~40 GB of free HBM")
    from fuxictr_b200 import layers
    from fuxictr_b200.schema import FeatureMap
    if ROOT not in sys.path:
        sys.path.insert(0, ROOT)
    import bench
    vocabs = bench.DLRM_VOCABS
    assert len(vocabs) == 26 and sum(vocabs) == 200_000_000
    specs = [("C%d" % i, {"type": "categorical", "source": "", "padding_idx": 0, "vocab_size": v})
             for i, v in enumerate(vocabs)]
    fm = FeatureMap.from_specs(specs, embedding_dim=16)
    B = 65536
    with torch.device("cuda"):
        layer = layers.FeatureEmbedding(fm, 16, embedding_initializer="partial(nn.init.normal_, std=0.05)")
    gen = torch.Generator().manual_seed(5)
    cols = []
    for i, v in enumerate(vocabs):      # half the fields uniform, half Zipf(1.05)-skewed (SURVEY 8d), some padding ids
        if i % 2:
            ids = bench.zipf_ids(B, [v], seed=100 + i)[:, 0]
        else:
            ids = torch.randint(1, v, (B,), generator=gen).double()
        ids[torch.rand(B, generator=gen) < 0.01] = 0
        cols.append(ids)
    mat = torch.stack(cols, dim=1).cuda()
    X = OrderedDict(("C%d" % i, mat[:, i]) for i in range(26))
    out = layer(X)
    assert tuple(out.shape) == (B, 26, 16)
    tables = dict(layer.named_parameters())
    names = list(tables.keys())
    assert len(names) == 26
    for i, k in enumerate(names):
        want = torch.nn.functional.embedding(mat[:, i].long(), tables[k], padding_idx=0)
        assert torch.equal(out[:, i, :], want), k
    assert torch.equal(layer(X), out)                                           # idempotent
    gout = torch.randn(out.shape, device="cuda", generator=torch.Generator(device="cuda").manual_seed(6))
    out.backward(gout)
    mass_in = 0.0
    for i, k in enumerate(names):
        g = tables[k].grad
        assert float(g[0].abs().sum()) == 0.0, k                               # padding row: no gradient
        idx = mat[:, i].long()
        live = idx != 0
        mass_in = float(gout[:, i, :][live].double().sum())
        assert abs(float(g.double().sum()) - mass_in) <= 1e-6 * float(gout[:, i, :].double().abs().sum()) + 1e-6, k
        if i in (0, 11, 25):        # three fields in full: the rows the batch touched, against index_add_
            rows = torch.unique(idx[live])
            ref = torch.zeros(tables[k].shape[0], 16, device="cuda", dtype=torch.float64)
            ref.index_add_(0, idx[live], gout[:, i, :][live].double())
            assert close(g[rows], ref[rows], RTOL, atol=1e-6), k
            del ref
        tables[k].grad = None

"""FinalNet on the H100: FinalBlock and FeatureGating against the reference's goldens in every matmul mode; the
factorized-interaction row kernels against float64 over their launch-plan branches (float4 and scalar widths, both
residuals, batch norm on and off, each activation, train and eval); running statistics against torch's BatchNorm1d;
the operand copies bit for bit; eval against dropout 0; the 2B loss against float64; zoo.FinalNet with the fused
optimizer along the reference's training trajectories; a CUDA-graph-captured step against the eager one; and two
virtual ranks with row-sharded tables against the unsharded model."""
import pytest
import torch

from conftest import Golden, close, rel_err

pytestmark = pytest.mark.gpu

RTOL = 1e-5
# single-pass modes: Frobenius bars on a block's output and gradients (the row kernels are fp32 in every mode; the
# GEMMs round their operands, and batch norm over 8 rows amplifies that)
FRO = {"tf32": (2e-2, 1e-1), "bf16": (6e-2, 3e-1)}
# ... and on a whole model's y_pred, loss and gradients the larger of a floor and four times the error that the
# reference's ops make in the same precision (torch eager with TF32 matmuls, or under bf16 autocast) on the same inputs
MODEL_FLOOR = {"tf32": 2e-4, "bf16": 2e-3}


@pytest.fixture(scope="module", autouse=True)
def _built():
    import __graft_entry__
    __graft_entry__.build()
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"


@pytest.fixture
def mode_of():
    from fuxictr_b200 import functional as F2
    yield F2.set_matmul_precision
    F2.set_matmul_precision("fp32")
    F2.set_x3_inline(True)


def fro(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


# ------------------------------------------------------------------ the reference's goldens
@pytest.mark.parametrize("mode", ["fp32", "tf32x3", "tf32", "bf16"])
@pytest.mark.parametrize("c", ["concat_bn_train", "sum_bn_train", "concat_nobn", "sum_nobn", "concat_bn_eval"])
def test_block_matches_reference_golden(c, mode, mode_of):
    from fuxictr_b200 import layers
    g = Golden("next_FinalBlock")
    _, din, units, acts, bn, res, training = [q for q in g.meta["cases"] if q[0] == c][0]
    block = layers.FinalBlock(din, units, acts, 0, bn, res)
    block.load_state_dict(g["w_" + c])
    block = block.cuda().train(training)
    mode_of(mode)
    x = g["in"]["x_" + c].cuda().requires_grad_(True)
    out = block(x)
    out.backward(g["in"]["gout_" + c].cuda())
    named = dict(block.named_parameters())
    want = g["g_" + c]
    sd = block.state_dict()
    for key, ref in g["s_" + c].items():           # running statistics after the forward
        if "running" in key or "num_batches" in key:
            assert close(sd[key], ref, 1e-5, atol=1e-6), (key, rel_err(sd[key], ref))
    if mode in ("fp32", "tf32x3"):
        assert close(out, g["out"]["y_" + c], RTOL), rel_err(out, g["out"]["y_" + c])
        assert close(x.grad, g["gin"]["x_" + c], RTOL, atol=RTOL * float(g["gin"]["x_" + c].abs().max()))
        scale = max(float(v.abs().max()) for v in want.values())
        for key, ref in want.items():
            assert close(named[key].grad, ref, 2 * RTOL, atol=RTOL * scale), (key, rel_err(named[key].grad, ref))
        return
    tol_y, tol = FRO[mode]
    assert fro(out, g["out"]["y_" + c]) <= tol_y
    assert fro(x.grad, g["gin"]["x_" + c]) <= tol
    for key, ref in want.items():
        assert fro(named[key].grad, ref) <= tol, key


@pytest.mark.parametrize("c", ["f5_d4", "f7_d3"])
def test_gating_matches_reference_golden(c):
    from fuxictr_b200 import layers
    g = Golden("next_FeatureGating")
    _, nf, D = [q for q in g.meta["cases"] if q[0] == c][0]
    gate = layers.FeatureGating(nf)
    gate.load_state_dict(g["w_" + c])
    gate = gate.cuda()
    x = g["in"]["x_" + c].cuda().requires_grad_(True)
    out = gate(x)
    out.backward(g["in"]["gout_" + c].cuda())
    assert close(out, g["out"]["y_" + c], RTOL), rel_err(out, g["out"]["y_" + c])
    assert close(x.grad, g["gin"]["x_" + c], RTOL), rel_err(x.grad, g["gin"]["x_" + c])
    named = dict(gate.named_parameters())
    for key, ref in g["g_" + c].items():
        assert close(named[key].grad, ref, RTOL), (key, rel_err(named[key].grad, ref))


# ------------------------------------------------------------------ float64 over the launch-plan branches
def _fi64(x, W, b, residual, norm, training, act):
    h = x @ W.t() + b
    m = h.shape[1] // 2
    h2, h1 = h[:, :m], h[:, m:]
    z = torch.cat([h2, h1 * h2], 1) if residual == "concat" else h2 + h1 * h2
    if norm is not None:
        if training:
            mu, var = z.mean(0), z.var(0, unbiased=False)
        else:
            mu, var = norm.running_mean.double(), norm.running_var.double()
        z = (z - mu) / torch.sqrt(var + norm.eps) * norm.weight.double() + norm.bias.double()
    if act == "ReLU":
        z = torch.relu(z)
    elif act == "Sigmoid":
        z = torch.sigmoid(z)
    return z


SWEEP = [(B, K, n, res, bn, act, tr)
         for (B, K, n) in [(2, 12, 8), (37, 20, 6), (1000, 16, 64), (4096, 40, 12), (129, 7, 10)]
         for res in ("concat", "sum") for bn in (True, False) for act in (None, "ReLU", "Sigmoid")
         for tr in (True, False)] + [(0, 8, 8, "concat", True, None, False), (1, 8, 8, "sum", True, "ReLU", False)]


@pytest.mark.parametrize("case", SWEEP, ids=lambda c: "B%d_K%d_n%d_%s_bn%d_%s_tr%d" % (c[0], c[1], c[2], c[3],
                                                                                        c[4], c[5], c[6]))
def test_layer_matches_float64(case):
    from fuxictr_b200 import layers
    B, K, n, res, bn, act, training = case
    torch.manual_seed(B + K + n)
    block = layers.FinalBlock(K, [n], act, 0, bn, res).cuda()
    with torch.no_grad():
        block.layer[0].linear.weight.normal_(0, 0.5)
        block.layer[0].linear.bias.normal_(0, 0.3)
        if bn:
            block.norm[0].weight.uniform_(0.5, 1.5)
            block.norm[0].bias.uniform_(-0.3, 0.3)
            block.norm[0].running_mean.normal_(0, 0.3)
            block.norm[0].running_var.uniform_(0.5, 1.5)
    block.train(training)
    norm64 = None
    if bn:
        norm64 = torch.nn.BatchNorm1d(n).double().cuda()
        norm64.load_state_dict(block.norm[0].state_dict())
    x = torch.randn(B, K, device="cuda").requires_grad_(True)
    gout = torch.randn(B, n, device="cuda")
    out = block(x)
    out.backward(gout)
    x64 = x.detach().double().requires_grad_(True)
    W64 = block.layer[0].linear.weight.detach().double().requires_grad_(True)
    b64 = block.layer[0].linear.bias.detach().double().requires_grad_(True)
    if bn:
        norm64.weight.requires_grad_(True)
        norm64.bias.requires_grad_(True)
    y64 = _fi64(x64, W64, b64, res, norm64, training, act)
    if B == 0:
        assert out.shape == (0, n)
        return
    y64.backward(gout.double())
    assert close(out, y64, 2e-5, atol=1e-6), rel_err(out, y64)
    # The batch-statistics backward subtracts terms of the size of g gamma rstd (1 + |h|) from each other; at B = 2 the
    # input gradient vanishes but for eps.  The bars' absolute part follows the size of those terms, dh_scale.
    with torch.no_grad():
        h64 = x64 @ W64.t() + b64
        m = h64.shape[1] // 2
        z64 = torch.cat([h64[:, :m], h64[:, m:] * h64[:, :m]], 1) if res == "concat" else h64[:, :m] * (1 + h64[:, m:])
        gain = 1.0
        if bn:
            var = z64.var(0, unbiased=False) if training else norm64.running_var
            gain = float((norm64.weight.abs() / torch.sqrt(var + norm64.eps)).max())
        dh_scale = float(gout.abs().max()) * gain * (1 + float(h64.abs().max()))
    lin = block.layer[0].linear
    for got, ref, terms in ((x.grad, x64.grad, float(W64.detach().abs().sum(0).max())),
                            (lin.weight.grad, W64.grad, float(x64.detach().abs().sum(0).max())),
                            (lin.bias.grad, b64.grad, float(B))):
        assert close(got, ref, 5e-5, atol=2e-6 * dh_scale * terms + 1e-6), rel_err(got, ref)
    if bn:
        for got, ref in ((block.norm[0].weight.grad, norm64.weight.grad), (block.norm[0].bias.grad, norm64.bias.grad)):
            assert close(got, ref, 5e-5, atol=1e-6), rel_err(got, ref)


@pytest.mark.parametrize("F,D,B", [(1, 1, 3), (5, 4, 33), (39, 40, 257), (128, 64, 9), (128, 1, 5), (3, 128, 2)])
def test_gating_matches_float64(F, D, B):
    from fuxictr_b200 import layers
    torch.manual_seed(F * D)
    gate = layers.FeatureGating(F).cuda()
    with torch.no_grad():
        gate.linear.weight.normal_(0, 0.3)
        gate.linear.bias.uniform_(0.5, 1.5)
    e = torch.randn(B, F, D, device="cuda").requires_grad_(True)
    gout = torch.randn(B, 2 * F, D, device="cuda")
    out = gate(e)
    out.backward(gout)
    e64 = e.detach().double().requires_grad_(True)
    W64 = gate.linear.weight.detach().double().requires_grad_(True)
    b64 = gate.linear.bias.detach().double().requires_grad_(True)
    g64 = (e64.transpose(1, 2) @ W64.t() + b64).transpose(1, 2)
    y64 = torch.cat([e64, e64 * g64], 1)
    y64.backward(gout.double())
    assert close(out, y64, 1e-5), rel_err(out, y64)
    for got, ref in ((e.grad, e64.grad), (gate.linear.weight.grad, W64.grad), (gate.linear.bias.grad, b64.grad)):
        assert close(got, ref, 2e-5, atol=1e-6), rel_err(got, ref)


def test_running_statistics_follow_torch_batchnorm():
    """Five training forwards of a concat and a sum block: running_mean, running_var and num_batches_tracked as
    torch's BatchNorm1d in float32 on the same z."""
    from fuxictr_b200 import layers
    for res in ("concat", "sum"):
        torch.manual_seed(5)
        block = layers.FinalBlock(24, [16], None, 0, True, res).cuda().train()
        ref = torch.nn.BatchNorm1d(16).cuda().train()
        lin = block.layer[0].linear
        for step in range(5):
            x = torch.randn(300 + step, 24, device="cuda")
            block(x)
            with torch.no_grad():
                h = torch.nn.functional.linear(x, lin.weight, lin.bias)
                h2, h1 = h.chunk(2, 1)
                ref(torch.cat([h2, h1 * h2], 1) if res == "concat" else h2 + h1 * h2)
        norm = block.norm[0]
        assert int(norm.num_batches_tracked) == 5
        assert close(norm.running_mean, ref.running_mean, 1e-5), rel_err(norm.running_mean, ref.running_mean)
        assert close(norm.running_var, ref.running_var, 1e-5), rel_err(norm.running_var, ref.running_var)


@pytest.mark.parametrize("mode", ["bf16", "tf32x3"])
def test_operand_copies_are_bit_exact(mode, mode_of):
    from fuxictr_b200 import functional as F2
    mode_of(mode)
    F2.set_x3_inline(False)
    torch.manual_seed(3)
    # half 32: the float4 path; half 10 and 18: the scalar one, where the second halves of h and of a concat output
    # start at columns that are no multiple of 4
    for H in (64, 20, 36):
        for res in ("concat", "sum"):
            x = torch.randn(100, 32, device="cuda")
            W = torch.randn(H, 32, device="cuda") * 0.2
            b = torch.randn(H, device="cuda") * 0.1
            out = F2.factorized_interaction(x, W, b, res, want_aux=True)
            aux = out._b2_aux[1]
            want = F2.make_aux(out.clone())
            assert torch.equal(aux.float(), want.float()), (H, res)
            # the backward's copy of dh, against the copy of dh itself
            xg = x.clone().requires_grad_(True)
            Wg = W.clone().requires_grad_(True)
            seen = {}
            real = F2._linear_dgrad

            def spy(tc, gz, gz_aux, W_, gx, w_aux=None, **kw):
                seen["dh"], seen["aux"] = gz.clone(), None if gz_aux is None else gz_aux.clone()
                return real(tc, gz, gz_aux, W_, gx, w_aux, **kw)
            F2._linear_dgrad = spy
            try:
                F2.factorized_interaction(xg, Wg, b, res).backward(torch.randn(out.shape, device="cuda"))
            finally:
                F2._linear_dgrad = real
            assert seen["aux"] is not None
            assert torch.equal(seen["aux"].float(), F2.make_aux(seen["dh"]).float()), (H, res)
    e = torch.randn(50, 6, 8, device="cuda")
    out = F2.feature_gating(e, torch.randn(6, 6, device="cuda"), torch.randn(6, device="cuda"), want_aux=True)
    assert torch.equal(out._b2_aux[1].float(), F2.make_aux(out.clone()).float())


def test_eval_mode_is_bit_equal_to_dropout_zero():
    from fuxictr_b200 import layers
    torch.manual_seed(8)
    a = layers.FinalBlock(20, [16, 8], "ReLU", 0.3, True, "concat").cuda()
    b = layers.FinalBlock(20, [16, 8], "ReLU", 0.0, True, "concat").cuda()
    b.load_state_dict(a.state_dict())
    x = torch.randn(64, 20, device="cuda")
    a.train()
    a(x)                                             # dropout draws in training ...
    b.load_state_dict(a.state_dict())
    a.eval()
    b.eval()
    assert torch.equal(a(x), b(x))                   # ... and none in eval


def test_two_block_loss_matches_float64():
    from fuxictr_b200 import functional as F2
    torch.manual_seed(9)
    for B in (1, 7, 1000, 70000):
        y1 = (torch.randn(B, 1, device="cuda") * 3).requires_grad_(True)
        y2 = (torch.randn(B, 1, device="cuda") * 3).requires_grad_(True)
        y = (torch.rand(B, 1, device="cuda") < 0.3).float()
        loss, y_pred = F2.finalnet_loss(y, y1, y2)
        loss.backward()
        a, c = y1.detach().double().requires_grad_(True), y2.detach().double().requires_grad_(True)
        p = torch.sigmoid(0.5 * (a + c))
        bce = torch.nn.functional.binary_cross_entropy
        l64 = bce(p, y.double()) + bce(torch.sigmoid(a), p.detach()) + bce(torch.sigmoid(c), p.detach())
        l64.backward()
        assert abs(float(loss) - float(l64)) <= 1e-5 * abs(float(l64)), (float(loss), float(l64))
        assert close(y_pred, p, 1e-6)
        assert close(y1.grad, a.grad, 1e-5, atol=1e-9), rel_err(y1.grad, a.grad)
        assert close(y2.grad, c.grad, 1e-5, atol=1e-9), rel_err(y2.grad, c.grad)


# ------------------------------------------------------------------ zoo.FinalNet
def eager_same_precision_errors(g, mode, batch):
    """Relative Frobenius errors against the reference's goldens of the reference's ops (the float64 oracle's code)
    run in fp32 on the GPU with TF32 matmuls (mode "tf32") or under bf16 autocast (mode "bf16"): y_pred, the loss and
    each parameter gradient on `batch`."""
    import finalnet_oracle as FO
    from oracle import fuxictr_oracle as O
    st = {k: (v.float().cuda().requires_grad_("running" not in k) if v.is_floating_point() else v.cuda())
          for k, v in g["w"].items()}
    X, y = O.split_inputs(g.specs(), g.meta["labels"], {k: v.cuda() for k, v in batch.items()})
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = mode == "tf32"
    try:
        with torch.autocast("cuda", dtype=torch.bfloat16, enabled=mode == "bf16"):
            y1, y2 = FO.finalnet_logits(g.specs(), st, X, g.meta["kwargs"])
        loss, y_pred = FO.finalnet_loss(y1.float(), None if y2 is None else y2.float(), y.float())
        loss.backward()
    finally:
        torch.backends.cuda.matmul.allow_tf32 = prev
    errs = {"y_pred": fro(y_pred, g["out"]["y_pred"]), "loss": fro(loss.view(1), g["out"]["loss"].view(1))}
    for key, ref in g["g"].items():
        errs[key] = fro(st[key].grad, ref)
    return errs


def build_golden_model(g):
    from fuxictr_b200 import zoo
    from fuxictr_b200.schema import FeatureMap
    fm = FeatureMap.from_specs(g.meta["specs"], labels=g.meta["labels"], embedding_dim=g.meta["kwargs"]["embedding_dim"])
    model = zoo.FinalNet(fm, gpu=-1, **g.meta["kwargs"])
    model.load_state_dict(g["w"])
    model.device = torch.device("cuda:0")
    model.model_to_device()
    model.compile("adam", "binary_crossentropy", 1e-3)
    model.train()
    model.use_fused_optimizer()
    return fm, model


@pytest.mark.parametrize("mode", ["fp32", "tf32x3", "tf32", "bf16"])
@pytest.mark.parametrize("name", ["2B", "1B_sum", "nobn"])
def test_model_with_fused_adam_matches_reference_trajectory(name, mode, mode_of):
    """y_pred, loss and every gradient on batch 0, then three fused_train_steps (the fused 2B loss, arena clip + Adam)
    against the reference's train_step()s: losses, gradients and the state after three steps (running statistics
    included) to 1e-5 in fp32 and 3xTF32.  In TF32 and bf16 the bars follow the error of the reference's ops in the
    same precision (MODEL_FLOOR); the parameters after three steps may differ by at most Adam's step bound, and the
    running statistics by the bar of y_pred."""
    mode_of(mode)
    g = Golden("model_FinalNet_" + name)
    fm, model = build_golden_model(g)
    B = g.meta["batch"]
    mat = g["in"]["matrix"].cuda()
    batches = [fm.batch_dict(mat[i * B:(i + 1) * B]) for i in range(3)]
    exact = mode in ("fp32", "tf32x3")
    if not exact:
        e = eager_same_precision_errors(g, mode, batches[0])
        bar = {k: max(MODEL_FLOOR[mode], 4 * v) for k, v in e.items()}
    ret = model.forward(batches[0])
    if exact:
        assert close(ret["y_pred"], g["out"]["y_pred"], RTOL), rel_err(ret["y_pred"], g["out"]["y_pred"])
    else:
        assert fro(ret["y_pred"], g["out"]["y_pred"]) <= bar["y_pred"], (fro(ret["y_pred"], g["out"]["y_pred"]), bar)
    loss = model.compute_loss(ret, model.get_labels(batches[0]))
    model._fused_optimizer.zero_grad()
    loss.backward()
    assert abs(float(loss) - float(g["out"]["loss"])) <= (RTOL if exact else bar["loss"]) * abs(float(g["out"]["loss"]))
    named = dict(model.named_parameters())
    for key, ref in g["g"].items():
        if exact:
            assert close(named[key].grad, ref, 2 * RTOL, atol=RTOL * float(ref.abs().max()) + 1e-9), \
                (key, rel_err(named[key].grad, ref))
        else:
            assert fro(named[key].grad, ref) <= bar[key], (key, fro(named[key].grad, ref), e[key])
    model._arena.zero_grads()
    # the running statistics now hold the forward above, as the reference's do before its train_step()s
    losses = [float(model.fused_train_step(b)) for b in batches]
    want = g["out"]["step_losses"]
    if exact:
        assert close(torch.tensor(losses), want, RTOL)
    else:
        assert fro(torch.tensor(losses), want) <= bar["loss"], (losses, want)
    sd = model.state_dict()
    for key, ref in g["w3"].items():
        if exact:
            assert close(sd[key], ref, 2e-5, atol=1e-7), (key, rel_err(sd[key], ref))
        elif key in named:
            # Adam moves a parameter by about lr per step whatever the gradient's size: two runs whose gradients
            # differ by rounding are at most 2 lr apart per step
            assert float((sd[key].cpu() - ref).abs().max()) <= 3 * 2 * 1e-3 * 1.01, key
        elif ref.is_floating_point():
            assert fro(sd[key], ref) <= 10 * bar["y_pred"], (key, fro(sd[key], ref))
        else:
            assert torch.equal(sd[key].cpu(), ref), key


def _fm_and_batches(n, B, seed, dim):
    import test_gpu_sharded_models as S
    from fuxictr_b200.schema import FeatureMap
    fm = FeatureMap.from_specs(S._CAT, embedding_dim=dim)
    gen = torch.Generator().manual_seed(seed)
    mats = []
    for _ in range(n):
        ids = torch.cat([torch.randint(0, s["vocab_size"], (B, 1), generator=gen) for _, s in S._CAT], 1)
        mats.append(torch.cat([ids.double(), (torch.rand(B, 1, generator=gen) < 0.4).double()], 1).cuda())
    return fm, mats


def make_model(fm, kw, seed=123):
    from fuxictr_b200 import zoo
    torch.manual_seed(seed)
    m = zoo.FinalNet(fm, gpu=0, **kw)
    with torch.no_grad():
        for mod in m.modules():
            if isinstance(mod, torch.nn.Embedding):
                mod.weight[1:].normal_(0, 0.3)
    return m


DEFAULT = dict(embedding_dim=40, block_type="2B", batch_norm=True, use_feature_gating=True,
               block1_hidden_units=[64, 64, 64], block2_hidden_units=[64, 64, 64], residual_type="concat")


@pytest.mark.parametrize("mode", ["fp32", "tf32x3", "tf32", "bf16"])
def test_default_config_trains_and_evaluates(mode, mode_of):
    """FinalNet_default's hyperparameters: ten fused_train_steps on one batch give finite, falling losses, and
    evaluate() returns logloss and AUC."""
    mode_of(mode)
    fm, mats = _fm_and_batches(1, 512, seed=3, dim=40)
    model = make_model(fm, DEFAULT)
    model.train()
    model.use_fused_optimizer()
    losses = [float(model.fused_train_step(fm.batch_dict(mats[0]))) for _ in range(10)]
    assert all(l == l for l in losses) and losses[-1] < losses[0], losses
    model.eval()
    res = model.evaluate([fm.batch_dict(mats[0])])
    assert set(res) >= {"logloss", "AUC"} and res["AUC"] > 0.5, res


@pytest.mark.parametrize("drop", [0.0, 0.2])
@pytest.mark.parametrize("mode", ["tf32x3", "bf16"])
def test_graph_captured_step_matches_eager(drop, mode, mode_of):
    """Five eager fused_train_steps against three warm-up steps and two replays of the captured step, running
    statistics included (the kernels update them inside the graph)."""
    from fuxictr_b200.pipeline import TrainPipeline
    from fuxictr_b200 import functional as F2
    mode_of(mode)
    kw = dict(DEFAULT, embedding_dim=16, block1_hidden_units=[32, 16], block2_hidden_units=[32, 16],
              block1_dropout=drop, block2_dropout=drop)
    fm, mats = _fm_and_batches(1, 512, seed=4, dim=16)
    mat = mats[0]
    eager, graphed = make_model(fm, kw), make_model(fm, kw)
    for m in (eager, graphed):
        m.train()
        m.use_fused_optimizer()
    torch.manual_seed(11)
    F2._DROPOUT.clear()
    F2.dropout_state(mat.device)
    ref = [float(eager.fused_train_step(fm.batch_dict(mat))) for _ in range(5)]
    torch.manual_seed(11)
    F2._DROPOUT.clear()
    F2.dropout_state(mat.device)
    pipe = TrainPipeline(graphed, mat.shape[0], mat.shape[1], graph=False)
    pipe.prime(mat)
    pipe.capture(warmup=3)
    got = [float(pipe.step_device(mat)) for _ in range(2)]
    torch.cuda.synchronize()
    tol = 5e-5 if mode == "tf32x3" else 2e-3
    for a, b in zip(got, ref[3:]):
        assert abs(a - b) <= tol * abs(b), (got, ref)
    if drop:
        assert ref[3] != ref[4]
    sd, want = graphed.state_dict(), eager.state_dict()
    for key, v in want.items():
        if key.endswith("num_batches_tracked"):
            assert int(sd[key]) == int(v) == 5, key
        elif mode == "tf32x3":
            assert close(sd[key], v, 1e-4, atol=1e-7), (key, rel_err(sd[key], v))
        else:
            assert fro(sd[key], v) <= 2e-2, (key, fro(sd[key], v))


def test_two_sharded_ranks_train_like_the_unsharded_model():
    """test_gpu_sharded_models.py's lock-step harness: two virtual ranks on one GPU, each with half of every table's
    rows, three fused_train_steps against the unsharded model with torch's clip + Adam on the global batches.  Batch
    norm is off: each rank's batch statistics would cover its own rows only."""
    import test_gpu_sharded_models as S
    from fuxictr_b200.schema import FeatureMap
    world = 2
    fm = FeatureMap.from_specs(S._CAT, embedding_dim=S.D)
    kw = dict(embedding_dim=S.D, block_type="2B", batch_norm=False, use_feature_gating=True,
              block1_hidden_units=[16, 8], block2_hidden_units=[8], residual_type="concat")

    def make():
        return make_model(fm, kw)
    ref = make()
    ref.fm_ = fm
    models = S._ranks(make, world, fm)
    gen = torch.Generator().manual_seed(21)
    batches = []
    for _ in range(3):
        ids = torch.cat([torch.randint(0, s["vocab_size"], (S.B_L * world, 1), generator=gen) for _, s in S._CAT], 1)
        batches.append(torch.cat([ids.double(), (torch.rand(S.B_L * world, 1, generator=gen) < 0.4).double()],
                                 1).cuda())
    losses = []
    for mat in batches:
        mats = [mat[r * S.B_L:(r + 1) * S.B_L].contiguous() for r in range(world)]
        losses.append(sum(S._lockstep_train_step(models, mats, fm)) / world)
    ref_losses = S._reference_steps(ref, batches, world, False)
    for a, b in zip(losses, ref_losses):
        assert abs(a - b) <= 1e-5 * abs(b), (losses, ref_losses)
    S._check_states(models, ref, world)

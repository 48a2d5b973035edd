"""DIEN on the H100: the interest stack (extractor GRU, attention, evolution GRU) against the reference's goldens in
every matmul mode; b2_gru_fwd / _bwd and the score kernels against the float64 oracle over the kernels' launch-plan
branches; zoo.DIEN with the fused optimizer along the reference's training trajectories and in the single-pass modes;
DIEN_test and DIEN_default training in every mode; a CUDA-graph-captured training step against the eager one;
evaluate / predict against forward; and two virtual ranks with row-sharded tables against the unsharded model."""
import sys

import pytest
import torch

from conftest import Golden, ROOT, close, rel_err

sys.path.insert(0, ROOT)
import dien_oracle as DO  # noqa: E402
from oracle import fuxictr_oracle as O  # noqa: E402

pytestmark = pytest.mark.gpu

RTOL = 1e-5
FRO = {"tf32": (1e-2, 5e-2), "bf16": (5e-2, 2e-1)}
MODES = ["fp32", "tf32x3", "tf32", "bf16"]
CASES = ["augru_bilinear", "agru_dot", "augru_din_sumpool", "gru_dice_bn"]


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


def fro(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def inert(g):
    """Parameters with an exact gradient of zero (a DNN bias ahead of a BatchNorm, attn_mlp's last bias under the
    softmax): their Adam steps follow rounding noise and are not compared; nor are the running statistics after them."""
    return set(k for k, v in g["g"].items() if float(v.abs().max()) < 1e-6)


def build_golden_model(g):
    from fuxictr_b200 import zoo
    from fuxictr_b200.schema import FeatureMap
    fm = FeatureMap.from_specs(g.meta["specs"], labels=g.meta["labels"], embedding_dim=g.meta["kwargs"]["embedding_dim"])
    model = zoo.DIEN(fm, gpu=-1, **g.meta["kwargs"])
    model.load_state_dict(g["w"], strict=False)
    model.device = torch.device("cuda:0")
    model.model_to_device()
    model.compile("adam", "binary_crossentropy", 1e-3)
    model.train()
    model.use_fused_optimizer()
    return fm, model


# ------------------------------------------------------------------ the reference's goldens
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("c", CASES)
def test_stack_matches_reference_golden(c, mode, mode_of):
    """h_out, the sequence's and the target's gradients and every stack parameter's gradient.  The recurrences are
    fp32 in every mode; only din_attention's MLP follows the mode."""
    mode_of(mode)
    g = Golden("next_DIEN_" + c)
    from fuxictr_b200 import zoo
    from fuxictr_b200.schema import FeatureMap
    specs = [("item_id", {"type": "categorical", "source": "", "padding_idx": 0, "vocab_size": 5}),
             ("click_history", {"type": "sequence", "source": "", "padding_idx": 0, "vocab_size": 5,
                                "max_len": g.meta["L"], "share_embedding": "item_id", "feature_encoder": None})]
    kw = dict(g.meta["kwargs"], embedding_dim=g.meta["H"], dien_target_field="item_id",
              dien_sequence_field="click_history", enable_sum_pooling=False)
    model = zoo.DIEN(FeatureMap.from_specs(specs, embedding_dim=g.meta["H"]), gpu=0, **kw)
    model.load_state_dict(g["w"], strict=False)
    model.train()
    seq = g["in"]["seq"].cuda().requires_grad_(True)
    tgt = g["in"]["target"].cuda().requires_grad_(True)
    out = model.interest(0, seq, tgt, g["in"]["mask"].cuda().contiguous())
    (out * g["in"]["gout"].cuda()).sum().backward()
    named = dict(model.named_parameters())
    tgrad = tgt.grad if tgt.grad is not None else torch.zeros_like(tgt)
    got = [out, seq.grad, tgrad] + [named[k].grad for k in g["g"]]
    want = [g["out"]["h_out"], g["gin"]["seq"], g["gin"]["target"]] + list(g["g"].values())
    names = ["h_out", "gin.seq", "gin.target"] + list(g["g"])
    tc_mlp = c == "augru_din_sumpool" and mode in FRO
    for n, a, b in zip(names, got, want):
        if n.startswith("attention_modules.0.attn_mlp") and float(b.abs().max()) < 1e-6:
            assert float(a.abs().max()) < 1e-5, n          # the last bias under the softmax: exact gradient zero
        elif tc_mlp:
            assert fro(a, b) <= FRO[mode][1], (n, fro(a, b))
        else:
            assert close(a, b, 2 * RTOL, atol=2 * RTOL * float(b.abs().max()) + 1e-9), (n, rel_err(a, b))


@pytest.mark.parametrize("mode", ["tf32", "bf16"])
@pytest.mark.parametrize("name", CASES)
def test_model_matches_reference_golden_single_pass(name, mode, mode_of):
    """y_pred and loss on batch 0 in the single-pass modes within the Frobenius bars; in TF32 all the gradients as one
    vector."""
    mode_of(mode)
    g = Golden("model_DIEN_" + name)
    fm, model = build_golden_model(g)
    batch = fm.batch_dict(g["in"]["matrix"].cuda()[:g.meta["batch"]])
    ret = model.forward(batch)
    loss = model.compute_loss(ret, model.get_labels(batch))
    model._fused_optimizer.zero_grad()
    loss.backward()
    fy, fg = FRO[mode]
    named = dict(model.named_parameters())
    skip = inert(g)
    got = torch.cat([named[k].grad.double().cpu().flatten() for k in g["g"] if k not in skip])
    ref = torch.cat([r.double().flatten() for k, r in g["g"].items() if k not in skip])
    worst = float((got - ref).norm() / ref.norm())
    print("measured %s %s: y_pred %.2e, loss %.2e, gradients %.2e" % (
        mode, name, fro(ret["y_pred"], g["out"]["y_pred"]), fro(loss, g["out"]["loss"]), worst))
    assert fro(ret["y_pred"], g["out"]["y_pred"]) <= fy and fro(loss, g["out"]["loss"]) <= fy
    assert worst <= fg


@pytest.mark.parametrize("mode", ["fp32", "tf32x3"])
@pytest.mark.parametrize("name", CASES)
def test_model_with_fused_adam_matches_reference_trajectory(name, mode, mode_of):
    """y_pred, loss and every gradient on batch 0, then three fused_train_steps against the reference's
    train_step()s."""
    mode_of(mode)
    g = Golden("model_DIEN_" + name)
    fm, model = build_golden_model(g)
    B = g.meta["batch"]
    mat = g["in"]["matrix"].cuda()
    batches = [fm.batch_dict(mat[i * B:(i + 1) * B]) for i in range(3)]
    ret = model.forward(batches[0])
    assert close(ret["y_pred"], g["out"]["y_pred"], RTOL)
    loss = model.compute_loss(ret, model.get_labels(batches[0]))
    assert close(loss, g["out"]["loss"], RTOL)
    model._fused_optimizer.zero_grad()
    loss.backward()
    named = dict(model.named_parameters())
    skip = inert(g)
    for k, ref in g["g"].items():
        got = named[k].grad
        if k in skip:
            assert float(got.abs().max()) <= 1e-6, k
            continue
        assert close(got, ref, 2 * RTOL, atol=2 * RTOL * float(ref.abs().max()) + 1e-9), (k, rel_err(got, ref))
    model._arena.zero_grads()
    losses = []
    for i in range(3):
        losses.append(float(model.fused_train_step(batches[i])))
        if i == 0:
            sd = model.state_dict()
            for k, ref in g["w1"].items():
                if k not in skip and not k.endswith("num_batches_tracked"):
                    assert close(sd[k], ref, RTOL, atol=1e-7), (k, rel_err(sd[k], ref))
    assert close(torch.tensor(losses), g["out"]["step_losses"], RTOL)
    sd = model.state_dict()
    for k, ref in g["w3"].items():
        if k not in skip and "running_" not in k and not k.endswith("num_batches_tracked"):
            assert close(sd[k], ref, 2e-5, atol=1e-7), (k, rel_err(sd[k], ref))


# ------------------------------------------------------------------ float64 oracle sweep of the kernels
def _mask(B, L, gen):
    """Rows: empty, full, length 1, a zero inside the history, then random post-padded lengths."""
    lens = torch.randint(0, L + 1, (B,), generator=gen)
    lens[:3] = torch.tensor([0, L, 1])[:B]
    m = torch.arange(L).view(1, -1) < lens.view(-1, 1)
    if B > 3 and L > 2:
        m[3] = True
        m[3, L // 2] = False
    return m


# (cell, B, L, H): H 1, every group width the kernels choose (1, 2, 4, 8, 16, 32, 64), odd H and the maximum 64;
# L 1, 2, 50 and the maximum 1024; B 0, 1 and across several CTAs
SWEEP = [("GRU", 5, 1, 1), ("AUGRU", 6, 2, 2), ("AGRU", 7, 50, 3), ("AUGRU", 300, 50, 16), ("GRU", 33, 50, 16),
         ("AGRU", 130, 50, 32), ("AUGRU", 9, 50, 33), ("GRU", 20, 50, 64), ("AUGRU", 17, 50, 64),
         ("AGRU", 4, 1024, 8), ("AUGRU", 3, 1024, 64), ("GRU", 0, 7, 4), ("AUGRU", 1, 7, 5)]


@pytest.mark.parametrize("cell, B, L, H", SWEEP)
def test_gru_kernels_match_float64(cell, B, L, H):
    """b2_gru_fwd / _bwd through functional.gru_sequence: h_seq, h_last, dx, da and every weight gradient, with
    gradients on both outputs (dh_seq and dh_last)."""
    from fuxictr_b200 import functional as F2
    gen = torch.Generator().manual_seed(B * 1000 + L * 10 + H)
    mask = _mask(B, L, gen)
    x = torch.randn(B, L, H, generator=gen, dtype=torch.float64) * 0.8
    W = [torch.randn(3 * H, H, generator=gen, dtype=torch.float64) * (0.9 / H ** 0.5),
         torch.randn(3 * H, generator=gen, dtype=torch.float64) * 0.3,
         torch.randn(3 * H, H, generator=gen, dtype=torch.float64) * (0.9 / H ** 0.5),
         torch.randn(3 * H, generator=gen, dtype=torch.float64) * 0.3]
    att = torch.rand(B, L, generator=gen, dtype=torch.float64) if cell != "GRU" else None
    gs = torch.randn(B, L, H, generator=gen, dtype=torch.float64)
    gl = torch.randn(B, H, generator=gen, dtype=torch.float64)
    ref_in = [t.clone().requires_grad_(True) for t in [x] + W + ([att] if att is not None else [])]
    hs, hl = DO.gru_sequence(ref_in[0], mask, *ref_in[1:5], cell=cell, att=ref_in[5] if att is not None else None)
    ((hs * gs).sum() + (hl * gl).sum()).backward()
    dev_in = [t.float().cuda().requires_grad_(True) for t in [x] + W + ([att] if att is not None else [])]
    mask_u8 = mask.to(torch.uint8).cuda()
    a = dev_in[5] if att is not None else None
    hs2, hl2 = F2.gru_sequence(dev_in[0], mask_u8, *dev_in[1:5], cell=cell, att=a)
    ((hs2 * gs.float().cuda()).sum() + (hl2 * gl.float().cuda()).sum()).backward()
    if B == 0:      # no launch: empty outputs and zero weight gradients
        assert hs2.shape == (0, L, H) and hl2.shape == (0, H)
        assert all(d.grad is None or d.grad.numel() == 0 or float(d.grad.abs().max()) == 0 for d in dev_in)
        return
    tol = 2e-5 if L <= 50 else 1e-4
    assert close(hs2, hs, tol), rel_err(hs2, hs)
    assert close(hl2, hl, tol), rel_err(hl2, hl)
    for n, r, d in zip(["dx", "dW_ih", "db_ih", "dW_hh", "db_hh", "da"], ref_in, dev_in):
        assert close(d.grad, r.grad, tol, atol=1e-6), (n, rel_err(d.grad, r.grad))


@pytest.mark.parametrize("kind", ["bilinear", "dot"])
@pytest.mark.parametrize("B, L, H", [(1, 1, 1), (37, 50, 16), (5, 9, 33), (300, 7, 64), (0, 4, 4)])
def test_scores_and_sum_pool_match_float64(kind, B, L, H):
    from fuxictr_b200 import functional as F2
    gen = torch.Generator().manual_seed(B + L + H)
    mask = _mask(B, L, gen)
    h = torch.randn(B, L, H, generator=gen, dtype=torch.float64)
    t = torch.randn(B, H, generator=gen, dtype=torch.float64)
    W = torch.randn(H, H, generator=gen, dtype=torch.float64) if kind == "bilinear" else None
    gs = torch.randn(B, L, generator=gen, dtype=torch.float64)
    gp = torch.randn(B, 2 * H, generator=gen, dtype=torch.float64)
    ref = [v.clone().requires_grad_(True) for v in (h, t) + ((W,) if W is not None else ())]
    st = {"attention_modules.0.W_kernel": ref[2]} if W is not None else {}
    s = DO.attention(ref[0], ref[1], mask, st, "attention_modules.0.",
                     {"attention_type": kind + "_attention", "use_attention_softmax": False})
    p = ref[0].sum(dim=1)
    pool = torch.cat([p, ref[1] * p], dim=-1)
    ((s * gs).sum() + (pool * gp).sum()).backward()
    dev = [v.float().cuda().requires_grad_(True) for v in (h, t) + ((W,) if W is not None else ())]
    mu = mask.to(torch.uint8).cuda()
    s2 = F2.dien_scores(dev[0], dev[1], mu, dev[2] if W is not None else None)
    pool2 = F2.dien_sum_pool(dev[0], dev[1])
    ((s2 * gs.float().cuda()).sum() + (pool2 * gp.float().cuda()).sum()).backward()
    if B == 0:
        assert s2.shape == (0, L) and pool2.shape == (0, 2 * H)
        return
    assert close(s2, s, 1e-5) and close(pool2, pool, 1e-5)
    for r, d in zip(ref, dev):
        assert close(d.grad, r.grad, 1e-5), rel_err(d.grad, r.grad)


# ------------------------------------------------------------------ the YAML shapes, graph capture, evaluate
def _seq_fm(max_len, dim, n_cat=3):
    from fuxictr_b200.schema import FeatureMap
    specs = [("C%d" % i, {"type": "categorical", "source": "", "padding_idx": 0, "vocab_size": 50 + i})
             for i in range(n_cat)]
    specs += [("adgroup_id", {"type": "categorical", "source": "", "padding_idx": 0, "vocab_size": 500}),
              ("click_sequence", {"type": "sequence", "source": "", "padding_idx": 0, "vocab_size": 500,
                                  "max_len": max_len, "share_embedding": "adgroup_id", "feature_encoder": None})]
    return FeatureMap.from_specs(specs, embedding_dim=dim)


def _matrix(fm, B, gen):
    cols = []
    for name, spec in fm.features.items():
        if spec["type"] == "sequence":
            L_ = spec["max_len"]
            ids = torch.randint(1, spec["vocab_size"], (B, L_), generator=gen)
            lens = torch.randint(0, L_ + 1, (B, 1), generator=gen)
            cols.append((ids * (torch.arange(L_).view(1, -1) < lens)).double())
        else:
            cols.append(torch.randint(0, spec["vocab_size"], (B, 1), generator=gen).double())
    cols.append((torch.rand(B, 1, generator=gen) < 0.3).double())
    return torch.cat(cols, dim=1)


CONFIGS = {
    "DIEN_test": dict(max_len=5, embedding_dim=4, dnn_hidden_units=[64, 32], batch=128),
    "DIEN_default": dict(max_len=50, embedding_dim=16, dnn_hidden_units=[1024, 512, 256], batch=1024),
}
MODEL_KW = dict(dien_target_field="adgroup_id", dien_sequence_field="click_sequence", dien_neg_seq_field=[],
                gru_type="AUGRU", attention_type="bilinear_attention", dnn_activations="Dice", batch_norm=True)


def _model(fm, cfg, **kw):
    from fuxictr_b200 import zoo
    torch.manual_seed(1)
    args = dict(MODEL_KW, embedding_dim=cfg["embedding_dim"], dnn_hidden_units=cfg["dnn_hidden_units"])
    args.update(kw)
    model = zoo.DIEN(fm, gpu=0, **args)
    with torch.no_grad():
        for m in model.modules():
            if isinstance(m, torch.nn.Embedding):
                m.weight[1:].normal_(0, 0.1)
    return model


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("name", ["DIEN_test", "DIEN_default"])
def test_yaml_configs_train_in_every_mode(name, mode, mode_of):
    """Three fused_train_steps from the same state as the float64 oracle's clip + Adam steps: the losses within the
    mode's bar."""
    mode_of(mode)
    cfg = CONFIGS[name]
    fm = _seq_fm(cfg["max_len"], cfg["embedding_dim"])
    model = _model(fm, cfg)
    kw = dict(MODEL_KW, dnn_hidden_units=cfg["dnn_hidden_units"])
    tr = O.OracleTrainer({k: v.detach().cpu().double() for k, v in model.state_dict().items()},
                         lambda s, X: torch.sigmoid(DO.dien_logit(fm.features, s, X, kw)), fm.features, fm.labels)
    model.use_fused_optimizer()
    gen = torch.Generator().manual_seed(9)
    losses, ref = [], []
    for _ in range(3):
        mat = _matrix(fm, cfg["batch"], gen)
        losses.append(float(model.fused_train_step(fm.batch_dict(mat.cuda()))))
        ref.append(float(tr.train_step(fm.batch_dict(mat)).detach()))
    bar = {"fp32": 1e-5, "tf32x3": 1e-5, "tf32": 1e-3, "bf16": 5e-3}[mode]
    for a, b in zip(losses, ref):
        assert abs(a - b) <= bar * abs(b), (losses, ref)


@pytest.mark.parametrize("mode", ["tf32x3", "bf16"])
@pytest.mark.parametrize("kw", [dict(), dict(gru_type="GRU"),
                                dict(attention_type="din_attention", attention_hidden_units=[16, 8],
                                     attention_activation="ReLU", enable_sum_pooling=True)])
def test_graph_captured_step_matches_eager(kw, mode, mode_of):
    from fuxictr_b200.pipeline import TrainPipeline
    mode_of(mode)
    cfg = dict(CONFIGS["DIEN_test"], dnn_hidden_units=[32, 16], embedding_dim=8)
    fm = _seq_fm(9, 8)
    mat = _matrix(fm, 512, torch.Generator().manual_seed(4)).cuda()
    eager, graphed = _model(fm, cfg, **kw), _model(fm, cfg, **kw)
    for m in (eager, graphed):
        m.train()
        m.use_fused_optimizer()
    ref = [float(eager.fused_train_step(fm.batch_dict(mat))) for _ in range(5)]
    pipe = TrainPipeline(graphed, mat.shape[0], mat.shape[1], graph=False)
    pipe.prime(mat)
    pipe.capture(warmup=3)
    got = [float(pipe.step_device(mat)) for _ in range(2)]
    torch.cuda.synchronize()
    # the GRU weight-gradient and split-K sums are float atomics: two runs differ in the last bits
    for a, b in zip(got, ref[3:]):
        assert abs(a - b) <= (1e-4 if mode == "bf16" else 1e-5) * abs(b), (got, ref)


def test_evaluate_and_predict_match_forward():
    cfg = CONFIGS["DIEN_test"]
    fm = _seq_fm(cfg["max_len"], cfg["embedding_dim"])
    model = _model(fm, cfg)
    model.eval()
    mat = _matrix(fm, 700, torch.Generator().manual_seed(5)).cuda()
    batches = [fm.batch_dict(mat[i:i + 256]) for i in range(0, 700, 256)]
    with torch.no_grad():
        y = torch.cat([model(b)["y_pred"].view(-1) for b in batches]).double().cpu()
    pred = torch.from_numpy(model.predict(batches))
    assert close(pred, y, 1e-6)
    res = model.evaluate(batches, ["logloss", "AUC"])
    labels = mat[:, -1].cpu().numpy()
    want = O.evaluate_metrics(labels, y.numpy(), ["logloss", "AUC"])
    assert abs(res["logloss"] - want["logloss"]) <= 1e-5 and abs(res["AUC"] - want["AUC"]) <= 1e-5, (res, want)


# ------------------------------------------------------------------ row-sharded tables, two virtual ranks
@pytest.mark.parametrize("kw", [dict(gru_type="AUGRU"), dict(gru_type="GRU", enable_sum_pooling=True)])
def test_two_sharded_ranks_train_like_the_unsharded_model(kw):
    """test_gpu_sharded_models.py's lock-step harness: two virtual ranks, each with half of every table's rows and its
    own lengths and mask from its local ids, three fused_train_steps against the unsharded model."""
    import test_gpu_sharded_models as S
    from fuxictr_b200 import zoo, sharded as SH
    world = 2
    fm = S._din_fm()

    def make():
        torch.manual_seed(3)
        m = zoo.DIEN(fm, gpu=0, embedding_dim=S.D, dnn_hidden_units=[16, 8], batch_norm=False,
                     dnn_activations="ReLU", dien_target_field=[("item_id", "cate_id")],
                     dien_sequence_field=[("click_history", "cate_history")], dien_neg_seq_field=[], **kw)
        with torch.no_grad():
            for mod in m.modules():
                if isinstance(mod, torch.nn.Embedding):
                    mod.weight[1:].normal_(0, 0.1)
        return m
    ref = make()
    ref.fm_ = fm
    models = S._ranks(make, world, fm)
    gen = torch.Generator().manual_seed(21)
    batches = [S._din_batch(gen, S.B_L * world) for _ in range(3)]
    losses = []
    for mat in batches:
        mats = [mat[r * S.B_L:(r + 1) * S.B_L].contiguous() for r in range(world)]
        losses.append(sum(S._lockstep_train_step(models, mats, fm)) / world)
    ref_losses = S._reference_steps(ref, batches, world, False)
    for a, b in zip(losses, ref_losses):
        assert abs(a - b) <= 1e-5 * abs(b), (losses, ref_losses)
    sd_ref = ref.state_dict()
    for r, m in enumerate(models):
        for k, v in m.state_dict().items():
            want = sd_ref[k]
            if "embedding_layers" in k:
                want = SH.shard_rows(want, r, world)
            assert close(v, want, 1e-4), (r, k, rel_err(v, want))

"""ETA and SDIM on the H100: b2_eta_retrieve_fwd, b2_sdim_pool_fwd and the two gradient assemblies against the float64
oracle over the kernels' launch-plan branches (hash_bits across the code-word boundary, L below, at and above topk and
up to 4096, shared and per-sample rotations, boundary ties); the interest blocks against the reference's goldens in
every matmul mode; zoo.ETA and zoo.SDIM with the fused optimizer along the reference's training trajectories;
ETA_default and SDIM_default training in every mode; a CUDA-graph-captured step against the eager one; evaluate /
predict against forward."""
import sys

import pytest
import torch

from conftest import Golden, ROOT, close, rel_err

sys.path.insert(0, ROOT)
import longctr_oracle as LO  # noqa: E402
from oracle import fuxictr_oracle as O  # noqa: E402

pytestmark = pytest.mark.gpu

RTOL = 1e-5
FRO = {"tf32": (1e-2, 5e-2), "bf16": (5e-2, 2e-1)}
MODES = ["fp32", "tf32x3", "tf32", "bf16"]
ETA_CASES = ["reuse_b32", "perbatch_b64_Lbelowk", "reuse_b7_one_field"]
SDIM_CASES = ["l2_h3_b3", "noqkvo_h1_b2", "perbatch_l2_h2_b4"]
ATT = ("W_q", "W_k", "W_v", "W_o")


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


# ------------------------------------------------------------------ float64 oracle sweep of the kernels
def _quarter(shape, gen, lo=-4, hi=5):
    """Multiples of 1/4 in [-1, 1]: every projection is exact in fp32 and in float64, so both hash alike, exact zeros
    (bit 0) and many equal distances included."""
    return torch.randint(lo, hi, shape, generator=gen).double() / 4


def _hist_mask(B, L, gen):
    """Rows: empty, full, length 1, then random pre-padded lengths."""
    lens = torch.randint(0, L + 1, (B,), generator=gen)
    lens[0], lens[1 % B] = 0, L
    if B > 2:
        lens[2] = 1
    return (torch.arange(L).view(1, -1) >= (L - lens).view(-1, 1)).double()


def _run_eta(x, mask, R, S, topk, Ws, Wl, heads=2):
    from fuxictr_b200 import functional as F2
    xd = x.float().cuda().requires_grad_(True)
    ws = [w.float().cuda().requires_grad_(True) for w in Ws]
    wl = [w.float().cuda().requires_grad_(True) for w in Wl]
    out = F2.eta_interest(xd, mask.float().cuda(), R.float().cuda(), S, topk, heads, True, ws, wl)
    return out, xd, ws, wl


@pytest.mark.parametrize("bits", [1, 31, 32, 33, 64])
@pytest.mark.parametrize("L,topk", [(7, 50), (50, 50), (300, 50), (4096, 256)])
@pytest.mark.parametrize("per_sample", [False, True])
def test_eta_retrieval_matches_float64(bits, L, topk, per_sample):
    """Chosen positions exactly (ascending (distance, position), so every boundary tie goes to the lower position),
    the compact rows, and the block's forward and gradients."""
    from fuxictr_b200 import functional as F2
    F2.set_matmul_precision("fp32")
    gen = torch.Generator().manual_seed(bits * 7 + L)
    B, d = (6 if L == 4096 else 13), 12
    x = _quarter((B, L + 1, d), gen)
    x[:, :L // 3] = x[:, L // 3:2 * (L // 3)].clone() if L >= 3 else x[:, :L // 3]    # repeated rows: many ties
    mask = _hist_mask(B, L, gen)
    x[:, :L] *= mask.unsqueeze(-1)                       # padding rows are zero, as padding_idx embeddings are
    R = _quarter((B if per_sample else 1, d, bits), gen)
    Ws = [torch.randn(8, d, generator=gen, dtype=torch.float64) * 0.3 for _ in range(3)] + \
        [torch.randn(d, 8, generator=gen, dtype=torch.float64) * 0.3]
    Wl = [w * 0.7 for w in Ws]
    S = 4
    (target, short, long, pos), xd, ws, wl = _run_eta(x, mask, R, S, topk, Ws, Wl)
    xr = x.clone().requires_grad_(True)
    wsr = [w.clone().requires_grad_(True) for w in Ws]
    wlr = [w.clone().requires_grad_(True) for w in Wl]
    rt, rs, rl, rpos = LO.eta_block(xr, mask, R, S, topk, 2, True, wsr, wlr)
    assert torch.equal(pos.cpu().long(), rpos)
    assert close(short, rs, RTOL) and close(long, rl, RTOL), (rel_err(short, rs), rel_err(long, rl))
    gen2 = torch.Generator().manual_seed(3)
    gs = [torch.randn(B, d, generator=gen2, dtype=torch.float64) for _ in range(3)]
    sum((o * g.float().cuda()).sum() for o, g in zip((target, short, long), gs)).backward()
    sum((o * g).sum() for o, g in zip((rt, rs, rl), gs)).backward()
    assert close(xd.grad, xr.grad, RTOL), rel_err(xd.grad, xr.grad)
    for a, b in zip(ws + wl, wsr + wlr):
        assert close(a.grad, b.grad, RTOL), rel_err(a.grad, b.grad)


@pytest.mark.parametrize("nh,bits", [(1, 1), (2, 4), (3, 7), (32, 2), (4, 24)])
@pytest.mark.parametrize("L", [5, 64, 1000, 4096])
@pytest.mark.parametrize("l2_norm", [False, True])
@pytest.mark.parametrize("d", [4, 12, 96])
def test_sdim_pooling_matches_float64(nh, bits, L, l2_norm, d):
    """The block's forward and every gradient (the collision-weighted rows with the normalize Jacobian), with shared
    and per-sample rotations, zero rows, empty histories and no-collision samples."""
    from fuxictr_b200 import functional as F2
    F2.set_matmul_precision("fp32")
    if L == 4096 and d == 96:
        pytest.skip("covered at d 4 and 12")
    gen = torch.Generator().manual_seed(nh * 31 + bits + L + d)
    B = 7
    x = _quarter((B, L + 1, d), gen)
    mask = _hist_mask(B, L, gen)
    x[:, :L] *= mask.unsqueeze(-1)
    x[3, L] = 0                                         # a zero target: bucket 0, collides with the zero rows it meets
    R = _quarter((B if nh == 3 else 1, d, nh, bits), gen)
    S = 2
    Ws = [torch.randn(8, d, generator=gen, dtype=torch.float64) * 0.3 for _ in range(3)] + \
        [torch.randn(d, 8, generator=gen, dtype=torch.float64) * 0.3]
    xd = x.float().cuda().requires_grad_(True)
    ws = [w.float().cuda().requires_grad_(True) for w in Ws]
    target, short, long = F2.sdim_interest(xd, mask.float().cuda(), R.float().cuda(), S + 1, l2_norm, 2, True, ws)
    xr = x.clone().requires_grad_(True)
    wsr = [w.clone().requires_grad_(True) for w in Ws]
    rt, rs, rl = LO.sdim_block(xr, mask, R, S + 1, l2_norm, 2, True, wsr)
    assert close(long, rl, RTOL) and close(short, rs, RTOL), (rel_err(long, rl), rel_err(short, rs))
    gen2 = torch.Generator().manual_seed(5)
    gs = [torch.randn(B, d, generator=gen2, dtype=torch.float64) for _ in range(3)]
    sum((o * g.float().cuda()).sum() for o, g in zip((target, short, long), gs)).backward()
    sum((o * g).sum() for o, g in zip((rt, rs, rl), gs)).backward()
    assert close(xd.grad, xr.grad, RTOL, atol=1e-5), rel_err(xd.grad, xr.grad)
    for a, b in zip(ws, wsr):
        assert close(a.grad, b.grad, RTOL), rel_err(a.grad, b.grad)


# ------------------------------------------------------------------ the reference's goldens
def _golden_block(name, g):
    from fuxictr_b200 import functional as F2
    kw = g.meta["kwargs"]
    x = g["in"]["x"].float().cuda().requires_grad_(True)
    w = {k: v.float().cuda().requires_grad_(True) for k, v in g["w"].items()}
    att = lambda p: [w["%s.%s.weight" % (p, n)] for n in ATT] if "%s.W_q.weight" % p in w else []   # noqa: E731
    mask, R = g["in"]["mask"].cuda(), g["in"]["R"].float().cuda()
    if name == "ETA":
        out = F2.eta_interest(x, mask, R, kw["short_seq_len"], kw["topk"], kw["num_heads"], kw["use_scale"],
                              att("short_attention"), att("long_attention"))
    else:
        out = F2.sdim_interest(x, mask, R, kw["short_seq_len"], kw["l2_norm"], kw["num_heads"], kw["use_scale"],
                               att("short_attention"))
    return out, x, w


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("name,c", [("ETA", c) for c in ETA_CASES] + [("SDIM", c) for c in SDIM_CASES])
def test_block_matches_reference_golden(name, c, mode, mode_of):
    mode_of(mode)
    g = Golden("next_%s_%s" % (name, c))
    out, x, w = _golden_block(name, g)
    target, short, long = out[:3]
    if name == "ETA":
        assert torch.equal(out[3].sort(dim=1).values.cpu(), g["out"]["pos"])
    gi = g["in"]
    ((target * gi["g_target"].cuda()).sum() + (short * gi["g_short"].cuda()).sum()
     + (long * gi["g_long"].cuda()).sum()).backward()
    pairs = [(short, g["out"]["short"]), (long, g["out"]["long"]), (x.grad, g["gin"]["x"])] + \
        [(w[k].grad, ref) for k, ref in g["g"].items()]
    for got, ref in pairs:
        if mode in FRO:
            assert fro(got, ref) <= FRO[mode][1], fro(got, ref)
        else:
            assert close(got, ref, RTOL, atol=RTOL * float(ref.abs().max()) + 1e-9), rel_err(got, ref)


def _triples(g, device="cuda"):
    out = []
    for i in range(3):
        ins = g["in"]
        bd = {"user_id": ins["%d/user_id" % i].to(device), "label": ins["%d/label" % i].to(device)}
        items = {k: ins["%d/%s" % (i, k)].to(device) for k in g.meta["item_fields"]}
        out.append((bd, items, ins["%d/mask" % i].to(device)))
    return out


def _golden_model(name, g):
    from fuxictr_b200 import zoo
    from fuxictr_b200.schema import FeatureMap
    fm = FeatureMap.from_specs(g.meta["specs"], labels=g.meta["labels"], embedding_dim=g.meta["kwargs"]["embedding_dim"])
    model = getattr(zoo, name)(fm, gpu=-1, **g.meta["kwargs"])
    model.load_state_dict(g["w"])
    model.device = torch.device("cuda:0")
    model.model_to_device()
    model.compile("adam", "binary_crossentropy", 1e-3)
    model.train()
    model.use_fused_optimizer()
    return fm, model


MODEL_CASES = [("ETA", "reuse_b32"), ("ETA", "reuse_b7_one_field"), ("SDIM", "l2_h3_b3"), ("SDIM", "noqkvo_h1_b2")]


@pytest.mark.parametrize("mode", ["fp32", "tf32x3"])
@pytest.mark.parametrize("name,c", MODEL_CASES)
def test_model_with_fused_adam_matches_reference_trajectory(name, c, mode, mode_of):
    mode_of(mode)
    g = Golden("model_%s_%s" % (name, c))
    fm, model = _golden_model(name, g)
    batches = _triples(g)
    ret = model.forward(batches[0])
    assert close(ret["y_pred"], g["out"]["y_pred"], RTOL), rel_err(ret["y_pred"], g["out"]["y_pred"])
    loss = model.compute_loss(ret, model.get_labels(batches[0]))
    assert close(loss, g["out"]["loss"], RTOL)
    model._fused_optimizer.zero_grad()
    loss.backward()
    named = dict(model.named_parameters())
    for k, ref in g["g"].items():
        assert close(named[k].grad, ref, 2 * RTOL, atol=2 * RTOL * float(ref.abs().max()) + 1e-9), \
            (k, rel_err(named[k].grad, ref))
    model._arena.zero_grads()
    losses = []
    for i in range(3):
        losses.append(float(model.fused_train_step(batches[i])))
        if i == 0:
            sd = model.state_dict()
            for k, ref in g["w1"].items():
                assert close(sd[k], ref, RTOL, atol=1e-7), (k, rel_err(sd[k], ref))
    assert close(torch.tensor(losses), g["out"]["step_losses"], RTOL)
    sd = model.state_dict()
    for k, ref in g["w3"].items():
        assert close(sd[k], ref, 2e-5, atol=1e-7), (k, rel_err(sd[k], ref))
    assert torch.equal(sd["random_rotations"].cpu(), g["w"]["random_rotations"])


@pytest.mark.parametrize("mode", ["tf32", "bf16"])
@pytest.mark.parametrize("name,c", MODEL_CASES)
def test_model_matches_reference_golden_single_pass(name, c, mode, mode_of):
    mode_of(mode)
    g = Golden("model_%s_%s" % (name, c))
    fm, model = _golden_model(name, g)
    batch = _triples(g)[0]
    ret = model.forward(batch)
    loss = model.compute_loss(ret, model.get_labels(batch))
    model._fused_optimizer.zero_grad()
    loss.backward()
    named = dict(model.named_parameters())
    got = torch.cat([named[k].grad.double().cpu().flatten() for k in g["g"]])
    ref = torch.cat([r.double().flatten() for r in g["g"].values()])
    fy, fg = FRO[mode]
    assert fro(ret["y_pred"], g["out"]["y_pred"]) <= fy and fro(loss, g["out"]["loss"]) <= fy
    assert float((got - ref).norm() / ref.norm()) <= fg


# ------------------------------------------------------------------ the YAML defaults
CONFIGS = {
    "ETA_default": dict(batch=8192, embedding_dim=4, dnn_hidden_units=[64, 32], attention_dim=64, num_heads=2,
                        use_scale=True, attention_dropout=0, reuse_hash=True, hash_bits=32, topk=50, short_seq_len=50,
                        net_dropout=0, batch_norm=False, max_len=50),
    "SDIM_default": dict(batch=10000, embedding_dim=32, dnn_hidden_units=[64, 32], attention_dim=64, use_qkvo=True,
                         num_heads=2, use_scale=True, attention_dropout=0, reuse_hash=True, num_hashes=2, hash_bits=4,
                         net_dropout=0, batch_norm=False, l2_norm=False, short_seq_len=50, max_len=50),
}


def _fm(dim, items=2):
    from fuxictr_b200.schema import FeatureMap
    specs = [("user_id", {"type": "categorical", "source": "user", "padding_idx": 0, "vocab_size": 500}),
             ("item_id", {"type": "categorical", "source": "item", "padding_idx": 0, "vocab_size": 3000}),
             ("cate_id", {"type": "categorical", "source": "item", "padding_idx": 0, "vocab_size": 60}),
             ("brand_id", {"type": "categorical", "source": "item", "padding_idx": 0, "vocab_size": 200})]
    return FeatureMap.from_specs(specs[:1 + items], embedding_dim=dim)


def _triple(fm, B, L, gen, device="cuda"):
    lens = torch.randint(0, L + 1, (B,), generator=gen)
    lens[1] = L
    hist = torch.randint(1, 3000, (B, L), generator=gen) * (torch.arange(L).view(1, -1) >= (L - lens).view(-1, 1))
    items = torch.cat([hist, torch.randint(1, 3000, (B, 1), generator=gen)], dim=1).flatten()
    idict = {"item_id": items}
    for f, v in (("cate_id", 60), ("brand_id", 200)):
        if f in fm.features:
            idict[f] = torch.where(items > 0, items % (v - 1) + 1, torch.zeros_like(items))
    bd = {"user_id": torch.randint(1, 500, (B,), generator=gen),
          "label": (torch.rand(B, generator=gen) < 0.3).double()}
    return ({k: v.to(device) for k, v in bd.items()}, {k: v.to(device) for k, v in idict.items()},
            (hist > 0).float().to(device))


def _model(name, fm, cfg, **kw):
    from fuxictr_b200 import zoo
    torch.manual_seed(1)
    args = {k: v for k, v in cfg.items() if k not in ("batch", "max_len")}
    args.update(kw)
    model = getattr(zoo, name)(fm, gpu=0, **args)
    with torch.no_grad():
        for m in model.modules():
            if isinstance(m, torch.nn.Embedding):
                m.weight[1:].normal_(0, 0.1)
    return model


class _Oracle(O.OracleTrainer):
    def __init__(self, name, model, fm, cfg):
        state = {k: v.detach().cpu().double() for k, v in model.state_dict().items()}
        super(_Oracle, self).__init__(state, None, fm.features, fm.labels)
        self.name, self.fm, self.cfg = name, fm, cfg

    def forward(self, triple):
        bd, idict, mask = [({k: v.cpu() for k, v in t.items()} if isinstance(t, dict) else t.cpu()) for t in triple]
        logit = LO.model_logit(self.name, self.state, self.fm, (bd, idict, mask.double()), self.cfg)
        return torch.sigmoid(logit), bd["label"].double().view(-1, 1)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("name", ["ETA_default", "SDIM_default"])
def test_yaml_configs_train_in_every_mode(name, mode, mode_of):
    """Three fused_train_steps from the same state as the float64 oracle's clip + Adam steps: the losses within the
    mode's bar.  The hash codes of the fp32 kernel and the float64 oracle agree on these draws unless a projection
    falls within rounding of a hyperplane; the bars leave room for that."""
    mode_of(mode)
    cfg = CONFIGS[name]
    model_name = name.split("_")[0]
    fm = _fm(cfg["embedding_dim"])
    model = _model(model_name, fm, cfg)
    tr = _Oracle(model_name, model, fm, cfg)
    model.use_fused_optimizer()
    gen = torch.Generator().manual_seed(9)
    losses, ref = [], []
    for _ in range(3):
        t = _triple(fm, cfg["batch"], cfg["max_len"], gen)
        losses.append(float(model.fused_train_step(t)))
        ref.append(float(tr.train_step(t).detach()))
    bar = {"fp32": 1e-4, "tf32x3": 1e-4, "tf32": 1e-3, "bf16": 5e-3}[mode]
    for a, b in zip(losses, ref):
        assert abs(a - b) <= bar * abs(b), (losses, ref)


def _capture(model, triple, warmup=3):
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(warmup):
            model.fused_train_step(triple)
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        loss = model.fused_train_step(triple).detach()
    return graph, loss


@pytest.mark.parametrize("mode", ["tf32x3", "bf16"])
@pytest.mark.parametrize("name,kw", [("ETA", dict()), ("ETA", dict(reuse_hash=False)), ("SDIM", dict()),
                                     ("SDIM", dict(l2_norm=True, num_hashes=3))])
def test_graph_captured_step_matches_eager(name, kw, mode, mode_of):
    from fuxictr_b200 import functional as F2
    mode_of(mode)
    cfg = dict(CONFIGS[name + "_default"], embedding_dim=8)
    fm = _fm(8)
    triple = _triple(fm, 512, 60, torch.Generator().manual_seed(4))
    eager, graphed = _model(name, fm, cfg, **kw), _model(name, fm, cfg, **kw)
    for m in (eager, graphed):
        m.train()
        m.use_fused_optimizer()
    torch.manual_seed(11)
    torch.cuda.manual_seed(11)
    ref = [float(eager.fused_train_step(triple)) for _ in range(5)]
    torch.manual_seed(11)
    torch.cuda.manual_seed(11)
    graph, loss_dev = _capture(graphed, triple)
    got = []
    for _ in range(2):
        graphed._fused_optimizer.count_step()
        F2.bump_weight_epoch()
        graph.replay()
        got.append(float(loss_dev))
    tol = 1e-4 if mode == "bf16" else 1e-5
    if kw.get("reuse_hash", True):
        for a, b in zip(got, ref[3:]):
            assert abs(a - b) <= tol * abs(b), (got, ref)
    else:   # fresh rotations every step: the graph's draws advance like the eager ones, the losses stay finite
        assert all(torch.isfinite(torch.tensor(got))) and len(set(got)) == 2, got


@pytest.mark.parametrize("name", ["ETA", "SDIM"])
def test_evaluate_and_predict_match_forward(name):
    cfg = CONFIGS[name + "_default"]
    fm = _fm(cfg["embedding_dim"], items=3)
    model = _model(name, fm, cfg)
    model.eval()
    gen = torch.Generator().manual_seed(5)
    batches = [_triple(fm, 300, 50, gen) for _ in range(3)]
    with torch.no_grad():
        y = torch.cat([model(b)["y_pred"].view(-1) for b in batches]).double().cpu()
    pred = torch.from_numpy(model.predict(batches))
    assert close(pred, y, 1e-6)
    res = model.evaluate(batches, ["logloss", "AUC"])
    labels = torch.cat([b[0]["label"].cpu() for b in batches]).numpy()
    want = O.evaluate_metrics(labels, y.numpy(), ["logloss", "AUC"])
    assert abs(res["logloss"] - want["logloss"]) <= 1e-5 and abs(res["AUC"] - want["AUC"]) <= 1e-5, (res, want)

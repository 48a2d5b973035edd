"""MIRRN on the H100: b2_mirrn_retrieve_fwd, the filter, mean and assembly kernels against the float64 oracle over the
launch-plan branches (hash_bits across the code-word boundary, L below, at and above topk, empty histories, shared and
per-call rotations, k up to 256); the interest block against the reference's goldens in every matmul mode; zoo.MIRRN
with the fused optimizer along the reference's trajectories; filter dropout against the host Philox; graph capture,
evaluate / predict, bit-identical backward runs, B = 0 and MIRRN_default training in every mode."""
import sys

import pytest
import torch

from conftest import Golden, ROOT, close, rel_err

sys.path.insert(0, ROOT)
import mirrn_oracle as MO  # noqa: E402
from oracle import fuxictr_oracle as O  # noqa: E402

pytestmark = pytest.mark.gpu

RTOL = 1e-5
FRO = {"tf32": (1e-2, 5e-2), "bf16": (5e-2, 2e-1)}
MODES = ["fp32", "tf32x3", "tf32", "bf16"]
CASES = ["k5_L8_reuse_b16", "k4_L20_percall_b64", "k2_L20_reuse_b48_one_field", "k1_L8_percall_b7",
         "k12_L6_reuse_b33"]
MODEL_CASES = ["k5_L8_reuse_b16", "k2_L20_reuse_b48_one_field", "k12_L6_reuse_b33"]


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


def _quarter(shape, gen, lo=-4, hi=5):
    """Multiples of 1/4 in [-1, 1]: projections are exact in fp32 and float64, so both hash alike (ties included)."""
    return torch.randint(lo, hi, shape, generator=gen).double() / 4


def _hist_mask(B, L, gen):
    lens = torch.randint(0, L + 1, (B,), generator=gen)
    lens[0], lens[1 % B] = 0, L
    if B > 2:
        lens[2] = 1
    return (torch.arange(L).view(1, -1) >= (L - lens).view(-1, 1)).double()


def _params(d, L, gen, heads=2):
    Ws = [torch.randn(8, d, generator=gen, dtype=torch.float64) * 0.3 for _ in range(3)] + \
        [torch.randn(d, 8, generator=gen, dtype=torch.float64) * 0.3]
    Wl = [w * 0.7 for w in Ws]
    P = torch.randn(L + 3, d, generator=gen, dtype=torch.float64)
    cws = [torch.randn(4, d // 4, d // 4, 2, generator=gen, dtype=torch.float64) * 0.5 for _ in range(3)]
    gam = [1 + 0.2 * torch.randn(d, generator=gen, dtype=torch.float64) for _ in range(3)]
    bet = [0.1 * torch.randn(d, generator=gen, dtype=torch.float64) for _ in range(3)]
    return Ws, Wl, P, cws, gam, bet


def _run(x, mask, R, S1, topk, params, heads=2, dropout=0.0):
    from fuxictr_b200 import functional as F2
    Ws, Wl, P, cws, gam, bet = params
    leaf = lambda t: t.float().cuda().requires_grad_(True)       # noqa: E731
    xd = leaf(x)
    ws, wl, Pd = [leaf(w) for w in Ws], [leaf(w) for w in Wl], leaf(P)
    cd, gd, bd = [leaf(w) for w in cws], [leaf(w) for w in gam], [leaf(w) for w in bet]
    out = F2.mirrn_interest(xd, mask.float().cuda(), R.float().cuda(), S1, topk, heads, True, ws, wl, Pd, cd, gd, bd,
                            dropout)
    return out, [xd] + ws + wl + [Pd] + cd + gd + bd


def _oracle(x, mask, R, S1, topk, params, heads=2):
    Ws, Wl, P, cws, gam, bet = params
    leaves = [t.clone().requires_grad_(True) for t in [x] + list(Ws) + list(Wl) + [P] + cws + gam + bet]
    xr, ws, wl, Pr = leaves[0], leaves[1:5], leaves[5:9], leaves[9]
    cr, gr, br = leaves[10:13], leaves[13:16], leaves[16:19]
    out = MO.mirrn_block(xr, mask, R, S1, topk, heads, True, ws, wl, Pr, cr, gr, br)
    return out, leaves


def _check(x, mask, R, S1, topk, params, seed, heads=2):
    (t, s, lg, pos), leaves = _run(x, mask, R, S1, topk, params, heads)
    (rt, rs, rl, rpos, _), rleaves = _oracle(x, mask, R, S1, topk, params, heads)
    assert torch.equal(pos.cpu().long(), rpos)
    assert close(s, rs, RTOL) and close(lg, rl, RTOL), (rel_err(s, rs), rel_err(lg, rl))
    gen = torch.Generator().manual_seed(seed)
    gs = [torch.randn(rt.shape, generator=gen, dtype=torch.float64) for _ in range(3)]
    sum((o * g.float().cuda()).sum() for o, g in zip((t, s, lg), gs)).backward()
    sum((o * g).sum() for o, g in zip((rt, rs, rl), gs)).backward()
    for i, (a, b) in enumerate(zip(leaves, rleaves)):
        assert close(a.grad, b.grad, 2e-5, atol=2e-5 * float(b.grad.abs().max()) + 1e-9), (i, rel_err(a.grad, b.grad))


@pytest.mark.parametrize("bits", [7, 32, 64])
@pytest.mark.parametrize("L,topk", [(7, 50), (50, 50), (300, 50)])
@pytest.mark.parametrize("per_call", [False, True])
def test_block_matches_float64(bits, L, topk, per_call):
    """Positions exactly (ties to the lower position, ascending), outputs and every gradient, with empty, full and
    one-item histories and repeated rows."""
    from fuxictr_b200 import functional as F2
    F2.set_matmul_precision("fp32")
    gen = torch.Generator().manual_seed(bits * 7 + L + per_call)
    B, d = 11, 12
    x = _quarter((B, L + 1, d), gen)
    if L >= 3:
        x[:, :L // 3] = x[:, L // 3:2 * (L // 3)].clone()
    mask = _hist_mask(B, L, gen)
    x[:, :L] *= mask.unsqueeze(-1)
    R = _quarter((3, d, bits) if per_call else (d, bits), gen)
    _check(x, mask, R, 5, topk, _params(d, L, gen), bits)


@pytest.mark.parametrize("k,d", [(1, 4), (2, 8), (3, 12), (16, 48), (64, 16), (256, 8)])
def test_filter_matches_float64_up_to_k_256(k, d):
    from fuxictr_b200 import functional as F2
    F2.set_matmul_precision("fp32")
    gen = torch.Generator().manual_seed(k + d)
    B, L = 5, max(k, 20)
    x = torch.randn(B, L + 1, d, generator=gen, dtype=torch.float64)
    mask = torch.ones(B, L, dtype=torch.float64)
    R = torch.randn(d, 32, generator=gen, dtype=torch.float64)
    _check(x, mask, R, 3, k, _params(d, L, gen), k)


def test_empty_batch():
    from fuxictr_b200 import functional as F2
    gen = torch.Generator().manual_seed(1)
    d, L = 8, 10
    (t, s, lg, pos), leaves = _run(torch.zeros(0, L + 1, d, dtype=torch.float64), torch.zeros(0, L),
                                   torch.randn(d, 16, generator=gen), 3, 4, _params(d, L, gen))
    assert t.shape == (0, d) and pos.shape == (0, 3, 4)
    (t.sum() + s.sum() + lg.sum()).backward()
    assert leaves[0].grad.shape == (0, L + 1, d)
    assert F2.mirrn_bound(d, L, 4, 16, 0) is None


def test_backward_is_bit_identical_across_runs():
    gen = torch.Generator().manual_seed(2)
    B, L, d = 64, 300, 16
    x = torch.randn(B, L + 1, d, generator=gen, dtype=torch.float64)
    mask = _hist_mask(B, L, gen)
    R = torch.randn(d, 32, generator=gen, dtype=torch.float64)
    params = _params(d, L, gen)
    grads = []
    for _ in range(2):
        (t, s, lg, _), leaves = _run(x, mask, R, 5, 50, params)
        (t.sum() + 2 * s.sum() + 3 * lg.sum()).backward()
        grads.append(leaves[0].grad.clone())
    assert torch.equal(grads[0], grads[1])


@pytest.mark.parametrize("ps", [(0.1, 0.1, 0.1), (0.1, 0.0, 0.3)])
def test_dropout_masks_match_host_philox(ps):
    """The add-norm of block q draws layer q of the forward's snapshot with block q's own probability: rerunning each
    block's LayerNorm on the host with the mask b2_dropout_apply writes for those offsets reproduces the interests."""
    from fuxictr_b200 import functional as F2
    gen = torch.Generator().manual_seed(4)
    B, L, d, k = 16, 30, 8, 6
    x = torch.randn(B, L + 1, d, generator=gen, dtype=torch.float64)
    mask = torch.ones(B, L)
    R = torch.randn(d, 16, generator=gen, dtype=torch.float64)
    params = _params(d, L, gen)
    state = F2.dropout_state(torch.device("cuda:0")).clone()     # the device key the block uses
    (t, s, lg, pos), _ = _run(x, mask, R, 3, k, params, dropout=ps)
    snap = state.clone()
    (rt, rs, rl, rpos, _), _ = _oracle(x, mask, R, 3, k, params)
    assert torch.equal(pos.cpu().long(), rpos)
    Ws, Wl, P, cws, gam, bet = params
    hist = x[:, :-1]
    ints = []
    for q in range(3):
        idx = rpos[:, q]
        u = torch.gather(hist, 1, idx.unsqueeze(-1).expand(-1, -1, d)) + P[L - idx] * 0.02
        spec = torch.fft.rfft(u, dim=1, norm="ortho").view(B, k // 2 + 1, 4, d // 4)
        spec = torch.einsum("blnd,ndd->blnd", spec, torch.view_as_complex(cws[q].contiguous()))
        A = torch.fft.irfft(spec.reshape(B, k // 2 + 1, d), n=k, dim=1, norm="ortho")
        ones = torch.ones(B * k, d, device="cuda")
        keep = F2.dropout_apply(ones, snap.cuda(), q, ps[q]) if ps[q] > 0 else ones
        keep = keep.cpu().double().view(B, k, d)
        z = A * keep + u
        mu = z.mean(-1, keepdim=True)
        var = (z - mu).pow(2).mean(-1, keepdim=True)
        ints.append((gam[q] * (z - mu) / torch.sqrt(var + 1e-12) + bet[q]).mean(1))
    ref_long = MO.mhta(x[:, -1], torch.stack(ints, 1), torch.ones(B, 3), 2, True, Wl)
    assert close(lg, ref_long, 1e-4), rel_err(lg, ref_long)



def test_each_filter_block_keeps_its_own_dropout():
    """zoo.MIRRN passes every block's out_dropout.p: with all three at 0 a training forward matches the evaluation
    one (the same kernels up to the training path's launch choices), and dropout on block 1 alone changes it."""
    fm = _fm(CONFIG["embedding_dim"])
    model = _model(fm, CONFIG)
    batch = _triple(fm, 256, 50, torch.Generator().manual_seed(6))
    with torch.no_grad():
        model.eval()
        ref = model(batch)["y_pred"]
        model.train()
        for blk in model.MHFT_block:
            blk.out_dropout.p = 0.0
        assert close(model(batch)["y_pred"], ref, 1e-6), rel_err(model(batch)["y_pred"], ref)
        model.MHFT_block[1].out_dropout.p = 0.5
        assert rel_err(model(batch)["y_pred"], ref) > 1e-4

# ------------------------------------------------------------------ the reference's goldens
def _golden_block(g):
    from fuxictr_b200 import functional as F2
    kw = g.meta["kwargs"]
    x = g["in"]["x"].float().cuda().requires_grad_(True)
    w = {k: v.float().cuda().requires_grad_(True) for k, v in g["w"].items()}
    Ws, Wl, P, cws, gam, bet = MO.block_params(w)
    out = F2.mirrn_interest(x, g["in"]["mask"].cuda(), g["in"]["R"].float().cuda(), kw["short_seq_len"], kw["topk"],
                            kw["num_heads"], kw["use_scale"], Ws, Wl, P, cws, gam, bet)
    return out, x, w


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("c", CASES)
def test_block_matches_reference_golden(c, mode, mode_of):
    mode_of(mode)
    g = Golden("next_MIRRN_%s" % c)
    out, x, w = _golden_block(g)
    target, short, long, pos = out
    assert torch.equal(pos.cpu(), g["out"]["pos"])
    gi = g["in"]
    ((target * gi["g_target"].cuda()).sum() + (short * gi["g_short"].cuda()).sum()
     + (long * gi["g_long"].cuda()).sum()).backward()
    pairs = [(short, g["out"]["short"]), (long, g["out"]["long"]), (x.grad, g["gin"]["x"])] + \
        [(w[k].grad, ref) for k, ref in g["g"].items()]
    for got, ref in pairs:
        if mode in FRO:
            assert fro(got, ref) <= FRO[mode][1], fro(got, ref)
        else:
            assert close(got, ref, 2e-5, atol=2e-5 * float(ref.abs().max()) + 1e-9), rel_err(got, ref)


def _triples(g, device="cuda"):
    out = []
    for i in range(3):
        ins = g["in"]
        bd = {"user_id": ins["%d/user_id" % i].to(device), "label": ins["%d/label" % i].to(device)}
        items = {k: ins["%d/%s" % (i, k)].to(device) for k in g.meta["item_fields"]}
        out.append((bd, items, ins["%d/mask" % i].to(device)))
    return out


def _golden_model(g):
    from fuxictr_b200 import zoo
    from fuxictr_b200.schema import FeatureMap
    fm = FeatureMap.from_specs(g.meta["specs"], labels=g.meta["labels"], embedding_dim=g.meta["kwargs"]["embedding_dim"])
    model = zoo.MIRRN(fm, gpu=-1, **g.meta["kwargs"])
    for blk in model.MHFT_block:
        blk.out_dropout.p = 0.0
    model.load_state_dict(g["w"])
    model.device = torch.device("cuda:0")
    model.model_to_device()
    model.compile("adam", "binary_crossentropy", 1e-3)
    model.train()
    model.use_fused_optimizer()
    return fm, model


@pytest.mark.parametrize("mode", ["fp32", "tf32x3"])
@pytest.mark.parametrize("c", MODEL_CASES)
def test_model_with_fused_adam_matches_reference_trajectory(c, mode, mode_of):
    mode_of(mode)
    g = Golden("model_MIRRN_%s" % c)
    fm, model = _golden_model(g)
    batches = _triples(g)
    ret = model.forward(batches[0])
    assert close(ret["y_pred"], g["out"]["y_pred"], RTOL), rel_err(ret["y_pred"], g["out"]["y_pred"])
    loss = model.compute_loss(ret, model.get_labels(batches[0]))
    assert close(loss, g["out"]["loss"], RTOL)
    model._fused_optimizer.zero_grad()
    loss.backward()
    named = dict(model.named_parameters())
    for k, ref in g["g"].items():
        assert close(named[k].grad, ref, 1e-4, atol=1e-4 * float(ref.abs().max()) + 1e-9), \
            (k, rel_err(named[k].grad, ref))
    model._arena.zero_grads()
    losses = []
    for i in range(3):
        losses.append(float(model.fused_train_step(batches[i])))
        if i == 0:
            sd = model.state_dict()
            for k, ref in g["w1"].items():
                assert close(sd[k], ref, RTOL, atol=1e-6), (k, rel_err(sd[k], ref))
    assert close(torch.tensor(losses), g["out"]["step_losses"], RTOL)
    sd = model.state_dict()
    for k, ref in g["w3"].items():
        assert close(sd[k], ref, 5e-5, atol=1e-6), (k, rel_err(sd[k], ref))
    assert torch.equal(sd["random_rotations"].cpu(), g["w"]["random_rotations"])


# ------------------------------------------------------------------ the YAML default
CONFIG = dict(batch=8192, embedding_dim=16, dnn_hidden_units=[64, 32], attention_dim=32, num_heads=4,
              use_scale=True, attention_dropout=0, reuse_hash=True, hash_bits=32, topk=4, max_len=50,
              short_seq_len=50, net_dropout=0, batch_norm=False)


def _fm(dim, items=3):
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


def _model(fm, cfg, **kw):
    from fuxictr_b200 import zoo
    torch.manual_seed(1)
    args = {k: v for k, v in cfg.items() if k != "batch"}
    args.update(kw)
    model = zoo.MIRRN(fm, gpu=0, **args)
    with torch.no_grad():
        for m in model.modules():
            if isinstance(m, torch.nn.Embedding) and m is not model.pos:
                m.weight[1:].normal_(0, 0.1)
    return model


class _Oracle(O.OracleTrainer):
    def __init__(self, model, fm, cfg):
        state = {k: v.detach().cpu().double() for k, v in model.state_dict().items()}
        super(_Oracle, self).__init__(state, None, fm.features, fm.labels)
        self.fm, self.cfg = fm, cfg

    def forward(self, triple):
        bd, idict, mask = [({k: v.cpu() for k, v in t.items()} if isinstance(t, dict) else t.cpu()) for t in triple]
        logit = MO.model_logit(self.state, self.fm, (bd, idict, mask.double()), self.cfg)
        return torch.sigmoid(logit), bd["label"].double().view(-1, 1)


@pytest.mark.parametrize("mode", MODES)
def test_yaml_config_trains_in_every_mode(mode, mode_of):
    """MIRRN_default (with attention_dropout 0 and the filter dropout off, so the float64 oracle can follow): three
    fused_train_steps against the oracle's clip + Adam steps, the losses within the mode's bar."""
    mode_of(mode)
    fm = _fm(CONFIG["embedding_dim"])
    model = _model(fm, CONFIG)
    for blk in model.MHFT_block:
        blk.out_dropout.p = 0.0
    tr = _Oracle(model, fm, CONFIG)
    model.use_fused_optimizer()
    gen = torch.Generator().manual_seed(9)
    losses, ref = [], []
    for _ in range(3):
        t = _triple(fm, CONFIG["batch"], CONFIG["max_len"], gen)
        losses.append(float(model.fused_train_step(t)))
        ref.append(float(tr.train_step(t).detach()))
    bar = {"fp32": 1e-4, "tf32x3": 1e-4, "tf32": 1e-3, "bf16": 5e-3}[mode]
    for a, b in zip(losses, ref):
        assert abs(a - b) <= bar * abs(b), (losses, ref)


@pytest.mark.parametrize("mode", MODES)
def test_yaml_config_trains_with_filter_dropout(mode, mode_of):
    mode_of(mode)
    fm = _fm(CONFIG["embedding_dim"])
    model = _model(fm, CONFIG)
    model.use_fused_optimizer()
    gen = torch.Generator().manual_seed(10)
    t = _triple(fm, CONFIG["batch"], CONFIG["max_len"], gen)
    losses = [float(model.fused_train_step(t)) for _ in range(4)]
    assert all(torch.isfinite(torch.tensor(losses))) and losses[-1] < losses[0], losses


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
@pytest.mark.parametrize("kw", [dict(), dict(reuse_hash=False)])
def test_graph_captured_step_matches_eager(kw, mode, mode_of):
    """Filter dropout on: the graph's Philox offsets advance like the eager steps', so replays 1 and 2 follow eager
    steps 4 and 5."""
    from fuxictr_b200 import functional as F2
    mode_of(mode)
    cfg = dict(CONFIG, embedding_dim=8, max_len=60)
    fm = _fm(8, items=2)
    triple = _triple(fm, 512, 60, torch.Generator().manual_seed(4))
    eager, graphed = _model(fm, cfg, **kw), _model(fm, cfg, **kw)
    for m in (eager, graphed):
        m.train()
        m.use_fused_optimizer()
    torch.manual_seed(11)
    torch.cuda.manual_seed(11)
    state = F2.dropout_state(torch.device("cuda:0"))
    saved = state.clone()
    ref = [float(eager.fused_train_step(triple)) for _ in range(5)]
    torch.manual_seed(11)
    torch.cuda.manual_seed(11)
    state.copy_(saved)                  # the same seed leaves the state where the eager steps left it
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
    else:
        assert all(torch.isfinite(torch.tensor(got))) and len(set(got)) == 2, got


def test_evaluate_and_predict_match_forward():
    """In eval mode the filter dropout is off: forward equals the float64 oracle without it."""
    fm = _fm(CONFIG["embedding_dim"])
    model = _model(fm, CONFIG)
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
    tr = _Oracle(model, fm, CONFIG)
    ref = tr.forward(batches[0])[0].view(-1)
    assert close(y[:300], ref, 1e-4), rel_err(y[:300], ref)

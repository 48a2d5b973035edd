"""SIM and TWIN on the H100: b2_sim_retrieve_fwd, b2_twin_topk_fwd and their backwards against the float64 oracle
over L below, at and above topk up to 4096, 1 to 4 heads, quarter-grid scores with many deliberate ties, empty
histories, histories with fewer valid rows than k and signed-zero SIM scores; the interest blocks against the
reference's goldens in every matmul mode; zoo.SIM and zoo.TWIN with the fused optimizer along the reference's training
trajectories; SIM_default and TWIN_default training in every mode; a CUDA-graph-captured step against the eager one;
evaluate / predict against forward."""
import sys

import pytest
import torch

from conftest import Golden, ROOT, close, rel_err

sys.path.insert(0, ROOT)
import sim_twin_oracle as SO  # noqa: E402
from oracle import fuxictr_oracle as O  # noqa: E402
from test_gpu_longctr import (_built, mode_of, fro, _quarter, _hist_mask, _triples, _golden_model, _fm,  # noqa
                              _triple, _model, _capture, FRO, MODES, RTOL)

pytestmark = pytest.mark.gpu

CASES = ["h2_k5", "h1_k8_one_field", "h2_k12"]
MHTA = ("W_q", "W_k", "W_v", "W_o")
TOPK = ("W_q", "W_h", "W_v", "W_o")


def _weights(gen, d, A=8, scale=0.3):
    return [torch.randn(A, d, generator=gen, dtype=torch.float64) * scale for _ in range(3)] + \
        [torch.randn(d, A, generator=gen, dtype=torch.float64) * scale]


def _leaves(ts):
    return [t.float().cuda().requires_grad_(True) for t in ts]


def _inputs(B, L, d, gen):
    """Quarter-grid rows (every fp32 score is exact, so positions compare exactly), repeated rows for ties, zero
    padding rows, and pre-padded masks: empty, full, length 1, random."""
    x = _quarter((B, L + 1, d), gen)
    if L >= 3:
        x[:, :L // 3] = x[:, L // 3:2 * (L // 3)].clone()
    mask = _hist_mask(B, L, gen)
    x[:, :L] *= mask.unsqueeze(-1)
    return x, mask


def _check_grads(outs, refs, leaves, rleaves, gen):
    """Gradients within fp32 bounds: relative, and absolute at RTOL of the O(1) gradient scale, where a single
    chosen row (k = 1) makes a softmax gradient that vanishes in float64 and is rounding in fp32."""
    gs = [torch.randn(r.shape, generator=gen, dtype=torch.float64) for r in refs]
    sum((o * g.float().cuda()).sum() for o, g in zip(outs, gs)).backward()
    sum((r * g).sum() for r, g in zip(refs, gs)).backward()
    for a, b in zip(leaves, rleaves):
        assert close(a.grad, b.grad, RTOL, atol=RTOL * max(1.0, float(b.grad.abs().max()))), rel_err(a.grad, b.grad)


@pytest.mark.parametrize("L", [2, 7, 50, 300, 4096])
@pytest.mark.parametrize("topk", [1, 50, 256])
@pytest.mark.parametrize("heads", [1, 2, 4])
def test_sim_matches_float64(L, topk, heads):
    """Positions exactly (descending score, ties to the lower position, -0.0 == +0.0), values and gradients."""
    from fuxictr_b200 import functional as F2
    F2.set_matmul_precision("fp32")
    if L == 4096 and heads != 2:
        pytest.skip("covered at 2 heads")
    gen = torch.Generator().manual_seed(L * 13 + topk + heads)
    B, d = (5 if L == 4096 else 11), 12
    x, mask = _inputs(B, L, d, gen)
    Ws, Wl = _weights(gen, d), _weights(gen, d)
    Wa = _quarter((8, d), gen)
    Wb = torch.eye(8, d, dtype=torch.float64)          # W_b^T W_a t on the quarter grid: every score exact in fp32
    S = 2 if L < 4 else 4
    leaves = _leaves([x, Wa, Wb] + Ws + Wl)
    out = F2.sim_interest(leaves[0], mask.float().cuda(), S, topk, heads, leaves[1], leaves[2], leaves[3:7],
                          leaves[7:])
    rleaves = [t.clone().requires_grad_(True) for t in [x, Wa, Wb] + Ws + Wl]
    ref = SO.sim_block(rleaves[0], mask, S, topk, heads, rleaves[1], rleaves[2], rleaves[3:7], rleaves[7:])
    assert torch.equal(out[4].cpu().long(), ref[4])
    for o, r in zip(out[:4], ref[:4]):
        assert close(o, r, RTOL, atol=1e-6), rel_err(o, r)
    _check_grads(out[:4], ref[:4], leaves, rleaves, gen)


@pytest.mark.parametrize("L", [2, 7, 50, 300, 4096])
@pytest.mark.parametrize("topk", [1, 50, 256])
@pytest.mark.parametrize("heads", [1, 2, 4])
def test_twin_matches_float64(L, topk, heads):
    """Per-head positions exactly (masked scores are exactly -1e9 and tie), values and gradients; an all-masked head
    weights its k chosen rows uniformly."""
    from fuxictr_b200 import functional as F2
    F2.set_matmul_precision("fp32")
    if L == 4096 and heads != 2:
        pytest.skip("covered at 2 heads")
    gen = torch.Generator().manual_seed(L * 17 + topk + heads)
    B, d = (5 if L == 4096 else 11), 12
    x, mask = _inputs(B, L, d, gen)
    A = 4 * heads
    Ws = _weights(gen, d, A)
    # W_q = I-like rows and W_h on the quarter grid scaled by sqrt(head_dim) = 2: every fp32 score is exact
    Wq = torch.zeros(A, d, dtype=torch.float64)
    Wq[torch.arange(A), torch.arange(A) % d] = 1.0
    Wt = [Wq, _quarter((A, d), gen) * 2, torch.randn(A, d, generator=gen, dtype=torch.float64) * 0.3,
          torch.randn(d, A, generator=gen, dtype=torch.float64) * 0.3]
    S = 2 if L < 4 else 4
    leaves = _leaves([x] + Ws + Wt)
    out = F2.twin_interest(leaves[0], mask.float().cuda(), S, topk, heads, leaves[1:5], leaves[5:])
    rleaves = [t.clone().requires_grad_(True) for t in [x] + Ws + Wt]
    ref = SO.twin_block(rleaves[0], mask, S, topk, heads, rleaves[1:5], rleaves[5:])
    assert torch.equal(out[3].cpu().long(), ref[3])
    for o, r in zip(out[:3], ref[:3]):
        assert close(o, r, RTOL, atol=1e-6), rel_err(o, r)
    _check_grads(out[:3], ref[:3], leaves, rleaves, gen)


def test_sim_signed_zero_scores_tie():
    """A masked row with a negative product scores -0.0 in the reference ((u . x) * 0); it ties with the +0.0 of the
    other zero scores, and the tie goes to the lower position."""
    from fuxictr_b200 import functional as F2
    F2.set_matmul_precision("fp32")
    B, L, d = 2, 6, 4
    x = torch.zeros(B, L + 1, d, dtype=torch.float64)
    x[:, -1, 0] = 1.0                       # target: u = W_b^T W_a t = e_0
    x[:, 2, 0] = -0.25
    x[:, 3, 0] = 0.5
    x[:, 4, 0] = -0.5
    mask = torch.tensor([[0, 1, 0, 1, 1, 1], [1, 1, 1, 1, 1, 1]], dtype=torch.float64)
    W = torch.eye(4, d, dtype=torch.float64)
    Ws = _weights(torch.Generator().manual_seed(1), d)
    leaves = _leaves([x, W, W] + Ws + Ws)
    out = F2.sim_interest(leaves[0], mask.float().cuda(), 2, 4, 1, leaves[1], leaves[2], leaves[3:7], leaves[7:])
    ref = SO.sim_block(x, mask, 2, 4, 1, W, W, Ws, Ws)
    assert out[4].cpu().tolist() == [[3, 0, 1, 2], [3, 0, 1, 5]] == ref[4].tolist()


# ------------------------------------------------------------------ the reference's goldens
def _golden_block(name, g):
    from fuxictr_b200 import functional as F2
    kw = g.meta["kwargs"]
    x = g["in"]["x"].float().cuda().requires_grad_(True)
    w = {k: v.float().cuda().requires_grad_(True) for k, v in g["w"].items()}
    att = lambda p, n=MHTA: [w["%s.%s.weight" % (p, m)] for m in n]     # noqa: E731
    mask = g["in"]["mask"].cuda()
    if name == "SIM":
        out = F2.sim_interest(x, mask, kw["short_seq_len"], kw["topk"], kw["num_heads"], w["W_a.weight"],
                              w["W_b.weight"], att("short_attention"), att("long_attention"))
        return out, ("target", "short", "long", "pooled"), x, w
    out = F2.twin_interest(x, mask, kw["short_seq_len"], kw["topk"], kw["num_heads"], att("short_attention"),
                           att("long_attention", TOPK))
    return out, ("target", "short", "long"), x, w


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("name", ["SIM", "TWIN"])
@pytest.mark.parametrize("c", CASES)
def test_block_matches_reference_golden(name, c, mode, mode_of):
    mode_of(mode)
    g = Golden("next_%s_%s" % (name, c))
    out, names, x, w = _golden_block(name, g)
    assert torch.equal(out[-1].sort(dim=-1).values.cpu(), g["out"]["pos"])
    sum((o * g["in"]["g_" + n].cuda()).sum() for o, n in zip(out, names)).backward()
    pairs = [(o, g["out"][n]) for o, n in zip(out, names)] + [(x.grad, g["gin"]["x"])] + \
        [(w[k].grad, ref) for k, ref in g["g"].items()]
    for got, ref in pairs:
        if mode in FRO:
            assert fro(got, ref) <= FRO[mode][1], fro(got, ref)
        else:
            assert close(got, ref, RTOL, atol=RTOL * float(ref.abs().max()) + 1e-9), rel_err(got, ref)


@pytest.mark.parametrize("mode", ["fp32", "tf32x3"])
@pytest.mark.parametrize("name", ["SIM", "TWIN"])
@pytest.mark.parametrize("c", CASES)
def test_model_with_fused_adam_matches_reference_trajectory(name, c, mode, mode_of):
    mode_of(mode)
    g = Golden("model_%s_%s" % (name, c))
    fm, model = _golden_model(name, g)
    batches = _triples(g)
    ret = model.forward(batches[0])
    assert close(ret["y_pred"], g["out"]["y_pred"], RTOL), rel_err(ret["y_pred"], g["out"]["y_pred"])
    if name == "SIM":
        assert close(ret["y_aux"], g["out"]["y_aux"], RTOL), rel_err(ret["y_aux"], g["out"]["y_aux"])
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


# ------------------------------------------------------------------ the YAML defaults
CONFIGS = {
    "SIM_default": dict(batch=8192, embedding_dim=4, dnn_hidden_units=[64, 32], attention_dim=64, num_heads=2,
                        attention_dropout=0, gsu_type="soft", topk=50, short_seq_len=50, alpha=1, beta=1,
                        net_dropout=0, batch_norm=False, max_len=50),
    "TWIN_default": dict(batch=8192, embedding_dim=4, dnn_hidden_units=[64, 32], attention_dim=64, num_heads=2,
                         attention_dropout=0, topk=50, short_seq_len=50, Kc_cross_features=0, net_dropout=0,
                         batch_norm=False, max_len=50),
}


class _Oracle(O.OracleTrainer):
    def __init__(self, name, model, fm, cfg):
        state = {k: v.detach().cpu().double() for k, v in model.state_dict().items()}
        super(_Oracle, self).__init__(state, None, fm.features, fm.labels)
        self.name, self.fm, self.cfg = name, fm, cfg

    def train_step(self, triple):
        bd, idict, mask = [({k: v.cpu() for k, v in t.items()} if isinstance(t, dict) else t.cpu()) for t in triple]
        self.optimizer.zero_grad()
        logits = SO.model_logits(self.name, self.state, self.fm, (bd, idict, mask.double()), self.cfg)
        y = bd["label"].double().view(-1, 1)
        bce = lambda z: O.bce_mean(torch.sigmoid(z), y)           # noqa: E731
        loss = bce(logits[0]) if self.name == "TWIN" else \
            self.cfg["alpha"] * bce(logits[1]) + self.cfg["beta"] * bce(logits[0])
        loss.backward()
        torch.nn.utils.clip_grad_norm_(self.params, self.max_norm)
        self.optimizer.step()
        return loss


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("name", ["SIM_default", "TWIN_default"])
def test_yaml_configs_train_in_every_mode(name, mode, mode_of):
    """Three fused_train_steps from the same state as the float64 oracle's clip + Adam steps: the losses within the
    mode's bar.  The fp32 scores and the float64 ones select alike unless two scores fall within rounding of each other
    at the k boundary; the bars leave room for that."""
    mode_of(mode)
    cfg = CONFIGS[name]
    model_name = name.split("_")[0]
    fm = _fm(cfg["embedding_dim"], items=3)
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


@pytest.mark.parametrize("mode", ["tf32x3", "bf16"])
@pytest.mark.parametrize("name", ["SIM", "TWIN"])
def test_graph_captured_step_matches_eager(name, mode, mode_of):
    from fuxictr_b200 import functional as F2
    mode_of(mode)
    cfg = dict(CONFIGS[name + "_default"], embedding_dim=8)
    fm = _fm(8)
    triple = _triple(fm, 512, 60, torch.Generator().manual_seed(4))
    eager, graphed = _model(name, fm, cfg), _model(name, fm, cfg)
    for m in (eager, graphed):
        m.train()
        m.use_fused_optimizer()
    ref = [float(eager.fused_train_step(triple)) for _ in range(5)]
    graph, loss_dev = _capture(graphed, triple)
    got = []
    for _ in range(2):
        graphed._fused_optimizer.count_step()
        F2.bump_weight_epoch()
        graph.replay()
        got.append(float(loss_dev))
    tol = 1e-4 if mode == "bf16" else 1e-5
    for a, b in zip(got, ref[3:]):
        assert abs(a - b) <= tol * abs(b), (got, ref)


@pytest.mark.parametrize("name", ["SIM", "TWIN"])
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

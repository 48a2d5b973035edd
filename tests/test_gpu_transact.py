"""TransAct on the H100: the token, attention and output kernels against float64 over their launch-plan branches (L
around the 32-row tile and up to 256, head widths 1 to 256, 1 to 16 heads, empty, full and ragged histories padded
on either side, B = 0, max-pool ties); the TransActTransformer module against the reference's goldens in every matmul
mode; zoo.TransAct against the reference's trajectories (single pass in TF32 and bf16, fused Adam in fp32 and 3xTF32);
the dropout masks against the host Philox and eval against dropout 0; a CUDA-graph-captured step against the eager
one; bit-identical backward runs; the TransAct_test and TransAct_default shapes training in every mode; and two
virtual ranks with row-sharded tables against the unsharded model."""
import sys

import pytest
import torch

from conftest import Golden, ROOT, close, rel_err

sys.path.insert(0, ROOT)
import transact_oracle as TO  # noqa: E402
from oracle import fuxictr_oracle as O  # noqa: E402
from test_transact_host import stable_part  # noqa: E402

pytestmark = pytest.mark.gpu

RTOL = 1e-5
FRO = {"tf32": (1e-2, 5e-2), "bf16": (5e-2, 2e-1)}
MODES = ["fp32", "tf32x3", "tf32", "bf16"]


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


def _ids(B, L, kind, gen):
    """(B, L) int64 ids: "empty", "full", "ragged" (padded on the right), "left" (padded on the left, TransAct's
    layout) or "mixed" (both, with an empty and a full row)."""
    ids = torch.randint(1, 100, (B, L), generator=gen)
    pos = torch.arange(L).view(1, -1)
    if kind == "empty":
        return ids * 0
    if kind == "full":
        return ids
    lens = torch.randint(0, L + 1, (B,), generator=gen)
    if kind == "mixed" and B >= 2:
        lens[0], lens[1] = 0, L
    right = pos < lens.view(-1, 1)
    left = pos >= (L - lens).view(-1, 1)
    if kind == "ragged":
        keep = right
    elif kind == "left":
        keep = left
    else:
        keep = torch.where((torch.arange(B) % 2 == 1).view(-1, 1), left, right)
    return ids * keep


# ------------------------------------------------------------------ kernels against float64
# (B, L, md, H, histories): L 1, 2, tile - 1, tile, tile + 1, 50, 100, 256; head widths 1, 3, 8, 64, 65, 128, 256;
# 1 to 16 heads; B 0
ATTN_CASES = [
    (5, 1, 8, 8, "mixed"),
    (7, 2, 3, 1, "mixed"),
    (9, 31, 64, 1, "left"),
    (9, 32, 130, 2, "mixed"),
    (9, 33, 128, 1, "ragged"),
    (6, 50, 128, 1, "left"),
    (4, 100, 256, 1, "mixed"),
    (3, 256, 256, 1, "mixed"),
    (3, 256, 512, 16, "full"),
    (4, 40, 256, 4, "empty"),
    (11, 17, 48, 16, "mixed"),
    (2, 70, 512, 2, "left"),
    (0, 50, 128, 1, "mixed"),
]


def _attn64(qkv, pad, H, gout, keep=None, p=0.0):
    B, L, md3 = qkv.shape
    md = md3 // 3
    dh = md // H
    qkv = qkv.double().requires_grad_(True)
    q, k, v = (t.reshape(B, L, H, dh).transpose(1, 2) for t in qkv.split(md, dim=-1))
    s = torch.matmul(q * (1.0 / dh) ** 0.5, k.transpose(-1, -2)).masked_fill(pad.view(B, 1, 1, L), float("-inf"))
    a = s.softmax(dim=-1)
    if keep is not None:
        a = a * keep.double() / (1.0 - p)
    ctx = torch.matmul(a, v).transpose(1, 2).reshape(B, L, md)
    (ctx * gout.double()).sum().backward()
    return ctx, qkv.grad


@pytest.mark.parametrize("case", ATTN_CASES)
def test_attention_matches_float64(case):
    """ctx at the live rows and the whole dQKV, with dO zero at the padded rows (the model's zeroing): the padded rows'
    dQ and the padded keys' dK, dV are then exactly 0 in float64 too."""
    from fuxictr_b200 import functional as F2
    B, L, md, H, kind = case
    gen = torch.Generator().manual_seed(L * 31 + md + H)
    ids = _ids(B, L, kind, gen)
    pad = TO.adjusted_padding(ids.clone())
    valid = (~pad).to(torch.uint8)
    qkv = torch.randn(B, L, 3 * md, generator=gen)
    gout = torch.randn(B, L, md, generator=gen) * (~pad).unsqueeze(-1)
    qg = qkv.cuda().view(B * L, 3 * md).requires_grad_(True)
    ctx = F2.transact_attention(qg, valid.cuda().contiguous(), B, L, H)
    ctx.backward(gout.cuda().view(B * L, md))
    if B == 0:
        assert ctx.shape == (0, md) and qg.grad.shape == (0, 3 * md)
        return
    ref, dref = _attn64(qkv, pad, H, gout)
    live = ~pad
    got = ctx.view(B, L, md).cpu()
    assert close(got[live], ref[live], RTOL, atol=RTOL), rel_err(got[live], ref[live])
    assert torch.equal(got[pad], torch.zeros_like(got[pad]))
    gq = qg.grad.view(B, L, 3 * md).cpu()
    assert close(gq, dref, 2 * RTOL, atol=2 * RTOL * float(dref.abs().max())), rel_err(gq, dref)


@pytest.mark.parametrize("B, L, D, ns, nt, kind", [(0, 5, 4, 1, 1, "mixed"), (1, 1, 3, 1, 1, "empty"),
                                                   (37, 50, 64, 1, 1, "mixed"), (9, 33, 8, 3, 5, "left"),
                                                   (4099, 7, 16, 2, 2, "ragged")])
def test_tokens_match_float64(B, L, D, ns, nt, kind):
    """The tokens, the adjusted valid bytes (ids as float64 column views and as int64) and the gradients: each sequence
    view's, and each target view's sum over the slots."""
    from fuxictr_b200 import functional as F2
    gen = torch.Generator().manual_seed(B + L + D)
    ids = _ids(B, L, kind, gen)
    seqs = [torch.randn(B, L, D, generator=gen) for _ in range(ns)]
    tgts = [torch.randn(B, D, generator=gen) for _ in range(nt)]
    md = D * (ns + nt)
    g = torch.randn(B * L, md, generator=gen)
    mat = torch.cat([torch.zeros(B, 2, dtype=torch.float64), ids.double()], dim=1).cuda()
    for ids_dev in (mat[:, 2:], ids.cuda()):
        vs = [t.cuda().requires_grad_(True) for t in seqs + tgts]
        x, valid = F2.transact_tokens(vs[:ns], vs[ns:], ids_dev)
        x.backward(g.cuda())
        if B == 0:
            assert x.shape == (0, md) and valid.shape == (0, L) and vs[0].grad.shape == (0, L, D)
            continue
        want = torch.cat([torch.cat(seqs, -1), torch.cat(tgts, -1).unsqueeze(1).expand(B, L, nt * D)], -1)
        assert torch.equal(x.cpu().view(B, L, md), want)
        assert torch.equal(valid.cpu().bool(), ~TO.adjusted_padding(ids.clone()))
        gv = g.view(B, L, md)
        for f in range(ns):
            assert torch.equal(vs[f].grad.cpu(), gv[:, :, f * D:(f + 1) * D])
        for f in range(nt):
            ref = gv[:, :, (ns + f) * D:(ns + f + 1) * D].double().sum(dim=1)
            assert close(vs[ns + f].grad, ref, 1e-6, atol=1e-5)


@pytest.mark.parametrize("B, L, md, k, pool", [(0, 5, 8, 1, True), (1, 1, 3, 1, True), (37, 50, 128, 1, True),
                                               (9, 33, 256, 33, True), (4099, 7, 16, 3, False), (6, 256, 512, 2, True)])
def test_output_matches_float64_with_ties(B, L, md, k, pool):
    """Last k slots and the masked max over L on a tensor with repeated rows (exact ties, gradient to the first slot),
    empty, full and ragged histories."""
    from fuxictr_b200 import functional as F2
    gen = torch.Generator().manual_seed(B + L + md)
    ids = _ids(B, L, "mixed", gen)
    pad = TO.adjusted_padding(ids.clone())
    y = torch.randn(B, L, md, generator=gen)
    if L >= 3:
        y[:, 2] = y[:, 1]                           # ties between slots 1 and 2
        y[:, :, 0] = 0.5                            # a column tied over every slot
    yg = y.cuda().view(B * L, md).requires_grad_(True)
    out = F2.transact_output(yg, (~pad).to(torch.uint8).cuda(), B, L, k, max_pool=pool)
    last, maxv = out if pool else (out, None)
    gl = torch.randn(B, k * md, generator=gen)
    gm = torch.randn(B, md, generator=gen)
    loss = (last * gl.cuda()).sum() + ((maxv * gm.cuda()).sum() if pool else 0)
    loss.backward()
    y64 = y.double().requires_grad_(True)
    z = y64.masked_fill(pad.unsqueeze(-1), 0.0)
    rl = z[:, L - k:].flatten(start_dim=1)
    ref = (rl * gl.double()).sum()
    if pool:
        rm = z.masked_fill(pad.unsqueeze(-1), -1e9).max(dim=1).values
        ref = ref + (rm * gm.double()).sum()
        assert torch.equal(maxv.cpu().double(), rm.detach())
    if B == 0:
        assert yg.grad.shape == (0, md)
        return
    ref.backward()
    assert torch.equal(last.cpu().double(), rl.detach())
    assert close(yg.grad.view(B, L, md), y64.grad, 1e-6, atol=1e-6)


# ------------------------------------------------------------------ the module against the reference's goldens
def _module(g):
    from fuxictr_b200 import layers
    _, L, D, ns, nt, H, n, ffn, k, pool = g.meta["case"]
    mod = layers.TransActTransformer(D * (ns + nt), dim_feedforward=ffn, num_heads=H, transformer_layers=n,
                                     first_k_cols=k, concat_max_pool=pool)
    mod.load_state_dict(g["w"])
    return mod.cuda().train()


def _run_module(mod, g, seq, tgt):
    _, L, D, ns, nt, H, n, ffn, k, pool = g.meta["case"]
    return mod.run(list(seq.split(D, dim=-1)), list(tgt.split(D, dim=-1)), g["in"]["ids"].cuda())


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("c", ["h1_k1_pool", "h2_l2_k3_pool_tuple", "h4_k2_nopool", "h1_l2_k1_pool_ties"])
def test_module_matches_reference_golden(c, mode, mode_of):
    g = Golden("next_TransActTransformer_" + c)
    mod = _module(g)
    mode_of(mode)
    seq = g["in"]["seq"].cuda().requires_grad_(True)
    tgt = g["in"]["tgt"].cuda().requires_grad_(True)
    y = _run_module(mod, g, seq, tgt)
    y.backward(g["in"]["gout"].cuda())
    named = dict(mod.named_parameters())
    if mode in ("fp32", "tf32x3"):
        assert close(y, g["out"]["y"], RTOL, atol=RTOL), rel_err(y, g["out"]["y"])
        for got, ref in ((seq.grad, g["gin"]["seq"]), (tgt.grad, g["gin"]["tgt"])):
            assert close(got, ref, RTOL, atol=RTOL * float(ref.abs().max())), rel_err(got, ref)
        scale = max(float(v.abs().max()) for v in g["g"].values())
        for k, ref in g["g"].items():
            assert close(named[k].grad, ref, 2 * RTOL, atol=2 * RTOL * scale), (k, rel_err(named[k].grad, ref))
        return
    fy, fg = FRO[mode]
    print("measured %s %s: y %.2e, dseq %.2e" % (mode, c, fro(y, g["out"]["y"]), fro(seq.grad, g["gin"]["seq"])))
    assert fro(y, g["out"]["y"]) <= fy
    assert fro(seq.grad, g["gin"]["seq"]) <= fg and fro(tgt.grad, g["gin"]["tgt"]) <= fg
    got = torch.cat([named[k].grad.double().cpu().flatten() for k in g["g"]])
    ref = torch.cat([v.double().flatten() for v in g["g"].values()])
    assert float((got - ref).norm() / ref.norm()) <= fg


def test_two_backward_runs_are_bit_identical(mode_of):
    """The attention, token and output backward write without float atomics: two runs give the same bits."""
    g = Golden("next_TransActTransformer_h2_l2_k3_pool_tuple")
    mode_of("tf32x3")
    grads = []
    for _ in range(2):
        mod = _module(g)
        seq = g["in"]["seq"].cuda().requires_grad_(True)
        tgt = g["in"]["tgt"].cuda().requires_grad_(True)
        _run_module(mod, g, seq, tgt).backward(g["in"]["gout"].cuda())
        grads.append([seq.grad.clone(), tgt.grad.clone()] +
                     [p.grad.clone() for n, p in mod.named_parameters() if "in_proj" in n])
    for a, b in zip(*grads):
        assert torch.equal(a, b)


def test_dropout_masks_match_the_host_philox(mode_of):
    """One layer in training mode with dropout against the float64 oracle given the masks the host Philox draws: the
    attention weights' at snapshot layer 0 over (B H L, L), dropout1's at layer 1 over (B L, md), then the FFN chain's
    own snapshot: the inner dropout at the next offset over (B L, ffn), dropout2 at the one after over (B L, md)."""
    from fuxictr_b200 import functional as F2, layers
    from test_mlp_dropout_host import keep_mask
    mode_of("fp32")
    B, L, md, H, ffn, p = 7, 37, 64, 2, 48, 0.2
    gen = torch.Generator().manual_seed(5)
    torch.manual_seed(5)
    mod = layers.TransActTransformer(md, dim_feedforward=ffn, num_heads=H, dropout=p).cuda().train()
    st = {k: v.detach().cpu().double().requires_grad_(True) for k, v in mod.state_dict().items()}
    ids = _ids(B, L, "mixed", gen)
    pad = TO.adjusted_padding(ids.clone())
    x = torch.randn(B, L, md, generator=gen)
    gout = torch.randn(B, L, md, generator=gen) * (~pad).unsqueeze(-1)
    xg = x.cuda().requires_grad_(True)
    seed, off = [int(v) for v in F2.dropout_state(xg.device).cpu()]
    y = mod.run_layers(xg.view(B * L, md), (~pad).to(torch.uint8).cuda(), B, L)
    y.backward(gout.cuda().view(B * L, md))

    def keep(o, M, N):
        return torch.from_numpy(keep_mask(seed, off + o, M, N, p))
    x64 = x.double().requires_grad_(True)
    y64 = TO.encoder_layer(x64, pad, st, "transformer_encoder.layers.0.", H,
                           attn_keep=keep(0, B * H * L, L).view(B, H, L, L), p_attn=p,
                           keep1=keep(1, B * L, md).view(B, L, md), keep0=keep(2, B * L, ffn).view(B, L, ffn),
                           keep2=keep(3, B * L, md).view(B, L, md), p=p)
    (y64 * gout.double()).sum().backward()
    live = ~pad
    got = y.view(B, L, md).cpu()
    assert close(got[live], y64[live], RTOL, atol=RTOL), rel_err(got[live], y64[live])
    assert close(xg.grad, x64.grad, 2 * RTOL, atol=2 * RTOL * float(x64.grad.abs().max())), rel_err(xg.grad, x64.grad)
    named = dict(mod.named_parameters())
    for k, p_ in st.items():
        if p_.grad is None or k.endswith("in_proj_bias"):
            continue
        ref, got_g = p_.grad, named[k].grad
        assert close(got_g, ref, 5 * RTOL, atol=5 * RTOL * float(ref.abs().max()) + 1e-9), (k, rel_err(got_g, ref))


# ------------------------------------------------------------------ models
def build_golden_model(g):
    from fuxictr_b200 import zoo
    from fuxictr_b200.schema import FeatureMap
    fm = FeatureMap.from_specs(g.meta["specs"], labels=g.meta["labels"], embedding_dim=g.meta["kwargs"]["embedding_dim"])
    model = zoo.TransAct(fm, gpu=-1, **g.meta["kwargs"])
    model.load_state_dict(g["w"])
    model.device = torch.device("cuda:0")
    model.model_to_device()
    model.compile("adam", "binary_crossentropy", 1e-3)
    model.train()
    model.use_fused_optimizer()
    return fm, model


MODEL_CASES = ["tuple_k1_pool", "two_pairs_k2_nopool", "h4_k3_bn"]


@pytest.mark.parametrize("name", MODEL_CASES)
def test_model_matches_reference_golden_single_pass(name, mode_of):
    """The golden models' y_pred, loss and gradients (as one vector) on batch 0 in TF32 and bf16, in one pass each."""
    g = Golden("model_TransAct_" + name)
    kw = g.meta["kwargs"]
    for mode in ("tf32", "bf16"):
        mode_of(mode)
        fm, model = build_golden_model(g)
        batch = fm.batch_dict(g["in"]["matrix"].cuda()[:g.meta["batch"]])
        ret = model.forward(batch)
        loss = model.compute_loss(ret, model.get_labels(batch))
        model._fused_optimizer.zero_grad()
        loss.backward()
        fy, fg = FRO[mode]
        named = dict(model.named_parameters())
        keys = [k for k in g["g"] if stable_part(k, g["g"][k], kw).numel()]
        got = torch.cat([stable_part(k, named[k].grad, kw).double().cpu().flatten() for k in keys])
        ref = torch.cat([stable_part(k, g["g"][k], kw).double().flatten() for k in keys])
        worst = float((got - ref).norm() / ref.norm())
        print("measured %s %s: y_pred %.2e, loss %.2e, gradients %.2e" % (
            mode, name, fro(ret["y_pred"], g["out"]["y_pred"]), fro(loss, g["out"]["loss"]), worst))
        assert fro(ret["y_pred"], g["out"]["y_pred"]) <= fy and fro(loss, g["out"]["loss"]) <= fy
        assert worst <= fg


@pytest.mark.parametrize("mode", ["fp32", "tf32x3"])
@pytest.mark.parametrize("name", MODEL_CASES)
def test_model_with_fused_adam_matches_reference_trajectory(name, mode, mode_of):
    """y_pred, loss and every gradient on batch 0, then three fused_train_steps (fused logit + BCE, arena clip + Adam)
    against the reference's train_step()s.  The parts whose exact gradient is zero (test_transact_host.stable_part)
    are held to an absolute bound and their Adam steps, driven by rounding noise, are not compared."""
    mode_of(mode)
    g = Golden("model_TransAct_" + name)
    kw = g.meta["kwargs"]
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
    for k, ref in g["g"].items():
        got = named[k].grad
        if stable_part(k, ref, kw).numel() == 0:
            assert float(got.abs().max()) <= 1e-6, k
            continue
        got, ref = stable_part(k, got, kw), stable_part(k, ref, kw)
        assert close(got, ref, 2 * RTOL, atol=2 * RTOL * float(ref.abs().max()) + 1e-9), (k, rel_err(got, ref))
    model._arena.zero_grads()
    losses = []
    for i in range(3):
        losses.append(float(model.fused_train_step(batches[i])))
    assert close(torch.tensor(losses), g["out"]["step_losses"], RTOL)
    sd = model.state_dict()
    for k, ref in g["w3"].items():
        if not ref.is_floating_point() or stable_part(k, ref, kw).numel() == 0:
            continue
        assert close(stable_part(k, sd[k], kw), stable_part(k, ref, kw), 2e-5), (k, rel_err(sd[k], ref))


def _seq_fm(max_len, dim, n_cat=4):
    from fuxictr_b200.schema import FeatureMap
    specs = [("C%d" % i, {"type": "categorical", "source": "", "padding_idx": 0, "vocab_size": 50 + i})
             for i in range(n_cat)]
    specs += [("item_id", {"type": "categorical", "source": "", "padding_idx": 0, "vocab_size": 200}),
              ("cate_id", {"type": "categorical", "source": "", "padding_idx": 0, "vocab_size": 20}),
              ("click_history", {"type": "sequence", "source": "", "padding_idx": 0, "vocab_size": 200,
                                 "max_len": max_len, "share_embedding": "item_id", "feature_encoder": None}),
              ("cate_history", {"type": "sequence", "source": "", "padding_idx": 0, "vocab_size": 20,
                                "max_len": max_len, "share_embedding": "cate_id", "feature_encoder": None})]
    return FeatureMap.from_specs(specs, embedding_dim=dim)


def _matrix(fm, B, gen):
    """Left-padded histories (TransAct's layout), the same lengths for both sequence fields, empty ones included."""
    cols, lens = [], None
    for name, spec in fm.features.items():
        if spec["type"] == "sequence":
            L_ = spec["max_len"]
            if lens is None:
                lens = torch.randint(0, L_ + 1, (B, 1), generator=gen)
            ids = torch.randint(1, spec["vocab_size"], (B, L_), generator=gen)
            cols.append((ids * (torch.arange(L_).view(1, -1) >= L_ - lens)).double())
        else:
            cols.append(torch.randint(0, spec["vocab_size"], (B, 1), generator=gen).double())
    cols.append((torch.rand(B, 1, generator=gen) < 0.3).double())
    return torch.cat(cols, dim=1)


# model_zoo/TransAct/config/model_config.yaml: TransAct_test and TransAct_default (batch reduced for the oracle)
CONFIGS = {
    "TransAct_test": dict(max_len=5, embedding_dim=4, dcn_hidden_units=[64, 32], mlp_hidden_units=[], num_heads=1,
                          dim_feedforward=512, dcn_cross_layers=3, batch=128),
    "TransAct_default": dict(max_len=50, embedding_dim=64, dcn_hidden_units=[1024, 512, 256], mlp_hidden_units=[],
                             num_heads=1, dim_feedforward=512, dcn_cross_layers=3, batch=512),
}


def _model(fm, cfg, **kw):
    from fuxictr_b200 import zoo
    torch.manual_seed(1)
    args = {k: cfg[k] for k in ("embedding_dim", "dcn_hidden_units", "mlp_hidden_units", "num_heads",
                                "dim_feedforward", "dcn_cross_layers")}
    args.update(kw)
    model = zoo.TransAct(fm, gpu=0, **args)
    with torch.no_grad():
        for m in model.modules():
            if isinstance(m, torch.nn.Embedding):
                m.weight[1:].normal_(0, 0.1)
    return model


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("name", ["TransAct_test", "TransAct_default"])
def test_yaml_configs_train_in_every_mode(name, mode, mode_of):
    """Three fused_train_steps from the same state as the float64 oracle's clip + Adam steps: the losses within the
    mode's bar."""
    mode_of(mode)
    cfg = CONFIGS[name]
    fm = _seq_fm(cfg["max_len"], cfg["embedding_dim"])
    model = _model(fm, cfg)
    kw = {k: cfg[k] for k in ("embedding_dim", "dcn_hidden_units", "mlp_hidden_units", "num_heads",
                              "dcn_cross_layers")}
    tr = O.OracleTrainer({k: v.detach().cpu().double() for k, v in model.state_dict().items()},
                         lambda s, X: torch.sigmoid(TO.transact_logit(fm.features, s, X, kw)), fm.features, fm.labels)
    model.use_fused_optimizer()
    gen = torch.Generator().manual_seed(9)
    losses, ref = [], []
    for _ in range(3):
        mat = _matrix(fm, cfg["batch"], gen)
        losses.append(float(model.fused_train_step(fm.batch_dict(mat.cuda()))))
        ref.append(float(tr.train_step(fm.batch_dict(mat)).detach()))
    # TF32 at TransAct_default: 1.3e-3 measured on the first loss (an 896-wide DCN input through three cross layers,
    # each GEMM rounding its operands)
    bar = {"fp32": 1e-5, "tf32x3": 1e-5, "tf32": 2e-3, "bf16": 5e-3}[mode]
    for a, b in zip(losses, ref):
        assert abs(a - b) <= bar * abs(b), (losses, ref)


def test_eval_mode_is_bit_equal_to_dropout_zero():
    """A model with transformer and net dropout in eval mode against the same weights built with dropout 0 in training
    mode, bit for bit; training mode with dropout differs.  The FFN is 32 wide here: at TransAct_test's 512 the FFN's
    second GEMM (K = 512, 1500 rows) splits K over CTAs and sums the parts with float atomics, so two forwards of the
    same model already differ in the last bits (4.8e-7 measured on the DCN input)."""
    cfg = dict(CONFIGS["TransAct_test"], dim_feedforward=32)
    fm = _seq_fm(cfg["max_len"], cfg["embedding_dim"])
    a = _model(fm, cfg, transformer_dropout=0.2, net_dropout=0.1)
    b = _model(fm, cfg)
    with torch.no_grad():
        for pa, pb in zip(a.parameters(), b.parameters()):
            pb.copy_(pa)
    mat = _matrix(fm, 300, torch.Generator().manual_seed(2)).cuda()
    with torch.no_grad():
        a.train()
        yd = a(fm.batch_dict(mat))["y_pred"]
        a.eval()
        ya = a(fm.batch_dict(mat))["y_pred"]
        b.train()
        y0 = b(fm.batch_dict(mat))["y_pred"]
    assert torch.equal(ya, y0)
    assert not torch.equal(yd, ya)


@pytest.mark.parametrize("drop", [0.0, 0.1])
def test_graph_captured_step_matches_eager(drop, mode_of):
    from fuxictr_b200.pipeline import TrainPipeline
    from fuxictr_b200 import functional as F2
    mode_of("tf32x3")
    cfg = dict(CONFIGS["TransAct_test"], embedding_dim=8, dcn_hidden_units=[32, 16], dim_feedforward=32)
    fm = _seq_fm(9, 8)
    mat = _matrix(fm, 512, torch.Generator().manual_seed(4)).cuda()
    kw = dict(transformer_dropout=drop, net_dropout=drop, transformer_layers=2, num_heads=2, first_k_cols=2)
    eager, graphed = _model(fm, cfg, **kw), _model(fm, cfg, **kw)
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
    # the LayerNorm's float atomics and the split-K weight-gradient sums make two runs differ in the last bits, and
    # Adam's first steps carry that into elements with small gradients
    for a, b in zip(got, ref[3:]):
        assert abs(a - b) <= 1e-5 * abs(b), (got, ref)
    kw = {"embedding_dim": cfg["embedding_dim"], "sequence_item_field": [("click_history", "cate_history")]}
    sd, want = graphed.state_dict(), eager.state_dict()
    for k, v in want.items():
        if v.is_floating_point():
            assert close(stable_part(k, sd[k], kw), stable_part(k, v, kw), 1e-4), (k, rel_err(sd[k], v))


def test_evaluate_and_predict():
    cfg = CONFIGS["TransAct_test"]
    fm = _seq_fm(cfg["max_len"], cfg["embedding_dim"])
    model = _model(fm, cfg)
    mat = _matrix(fm, 256, torch.Generator().manual_seed(3)).cuda()
    batches = [fm.batch_dict(mat[i * 64:(i + 1) * 64]) for i in range(4)]
    model.eval()
    pred = model.predict(batches)
    with torch.no_grad():
        ref = torch.cat([model(b)["y_pred"] for b in batches]).flatten().double().cpu().numpy()
    assert pred.shape == (256,) and abs(pred - ref).max() <= 1e-6
    res = model.evaluate(batches)
    assert set(res) >= {"logloss", "AUC"}


# ------------------------------------------------------------------ row-sharded tables, two virtual ranks
def test_two_sharded_ranks_train_like_the_unsharded_model():
    """test_gpu_sharded_models.py's lock-step harness on its DIN-like map: two virtual ranks, each with half of every
    table's rows and its own mask from its local ids, three fused_train_steps against the unsharded model."""
    import test_gpu_sharded_models as S
    from fuxictr_b200 import zoo, sharded as SH
    world = 2
    fm = S._din_fm()

    def make():
        torch.manual_seed(3)
        m = zoo.TransAct(fm, gpu=0, embedding_dim=S.D, num_heads=2, dcn_hidden_units=[16, 8], dim_feedforward=16,
                         dcn_cross_layers=2, first_k_cols=2, target_item_field=[("item_id", "cate_id")],
                         sequence_item_field=[("click_history", "cate_history")])
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
    kw = {"embedding_dim": S.D, "sequence_item_field": [("click_history", "cate_history")]}
    sd_ref = ref.state_dict()
    for r, m in enumerate(models):
        for k, v in m.state_dict().items():
            if not v.is_floating_point():
                continue
            want = sd_ref[k]
            if "embedding_layers" in k:
                want = SH.shard_rows(want, r, world)
            assert close(stable_part(k, v, kw), stable_part(k, want, kw), 1e-4), (r, k, rel_err(v, want))

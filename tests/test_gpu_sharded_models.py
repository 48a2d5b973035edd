"""Row-sharded tables for DCNv2, xDeepFM and DIN, with unpooled sequence fields in the push and pull.

`world` virtual ranks on ONE GPU (fuxictr_b200.sharded.VirtualPeerGroup): the push / pull kernels cannot tell a
local pointer from a peer pointer.  Front level: the landed rows and the table gradients of DIN-like fields
(two share_embedding histories) against the unsharded FeatureEmbeddingDict.  Model level: three
fused_train_steps of every rank in lock step (the phases of the sharded front between its barriers, the rest of
each rank's step its own fused_train_step) against the unsharded model."""
import sys

import pytest
import torch

from conftest import close, ROOT

sys.path.insert(0, ROOT)
pytestmark = pytest.mark.gpu

D, B_L, L = 8, 16, 6
_SEQ = [
    ("user", {"type": "categorical", "source": "", "padding_idx": 0, "vocab_size": 30}),
    ("item_id", {"type": "categorical", "source": "", "padding_idx": 0, "vocab_size": 50}),
    ("cate_id", {"type": "categorical", "source": "", "padding_idx": 0, "vocab_size": 12}),
    ("click_history", {"type": "sequence", "source": "", "padding_idx": 0, "vocab_size": 50, "max_len": L,
                       "share_embedding": "item_id"}),
    ("cate_history", {"type": "sequence", "source": "", "padding_idx": 0, "vocab_size": 12, "max_len": L,
                      "share_embedding": "cate_id"}),
]
_CAT = [("C%d" % i, {"type": "categorical", "source": "", "padding_idx": 0, "vocab_size": 60 + 17 * i})
        for i in range(7)]


def _build():
    import __graft_entry__
    __graft_entry__.build()


def _din_batch(gen, B, pad_frac=None):
    """Categorical ids (0 now and then) and two post-padded histories of random length, with all-padding and
    full rows included; cate_history follows click_history's length.  pad_frac: histories about that padded."""
    cols = [torch.randint(0, s["vocab_size"], (B, 1), generator=gen) for _, s in _SEQ[:3]]
    if pad_frac is None:
        lens = torch.randint(0, L + 1, (B,), generator=gen)
        lens[0], lens[1] = 0, L
    else:
        lens = torch.full((B,), int(round(L * (1 - pad_frac))))
    pos = torch.arange(L).view(1, L)
    keep = pos < lens.view(B, 1)
    for _, s in _SEQ[3:]:
        h = torch.randint(1, s["vocab_size"], (B, L), generator=gen)
        cols.append(torch.where(keep, h, torch.zeros_like(h)))
    label = (torch.rand(B, 1, generator=gen) < 0.4).long()
    return torch.cat(cols + [label], 1).double().cuda()


def _din_fm():
    from fuxictr_b200.schema import FeatureMap
    return FeatureMap.from_specs(_SEQ, embedding_dim=D)


def _front_ranks(fed, fm, world, registry):
    """`world` ShardedFronts over shards of fed's tables (a shared table: one shard Parameter per rank)."""
    from fuxictr_b200 import sharded as SH
    names = list(fm.features.keys())
    fronts, shards = [], []
    for r in range(world):
        own = {}
        tabs = []
        for f in names:
            emb = fed.embedding_layers[f]
            if id(emb) not in own:
                own[id(emb)] = torch.nn.Parameter(SH.shard_rows(emb.weight.detach(), r, world))
            tabs.append(own[id(emb)])
        cols = [fm.get_column_index(f) for f in names]
        cols = [c[0] if isinstance(c, list) else c for c in cols]
        seq = [fm.features[f].get("max_len", 1) if fm.features[f]["type"] == "sequence" else 1 for f in names]
        fr = SH.ShardedFront(SH.VirtualPeerGroup(r, world, registry), names, tabs, None,
                             [fed.embedding_layers[f].num_embeddings for f in names], cols,
                             [fed.embedding_layers[f].padding_idx for f in names], D, B_L, fm.input_length + 1,
                             torch.float64, want_fm=False, seq_lens=seq)
        fr.pull_scale = 1.0
        fronts.append(fr)
        shards.append(tabs)
    return fronts, shards


def _reference_rows(fed, fm, mat):
    from collections import OrderedDict
    X = OrderedDict((k, v) for k, v in fm.batch_dict(mat).items() if k != "label")
    out = fed(X)
    parts = [out[f].reshape(mat.shape[0], -1, D) for f in fm.features.keys()]
    return torch.cat(parts, 1)          # (B, S, D)


def _push_all(fronts, mats, after_ids=None):
    for fr, m in zip(fronts, mats):
        fr.phase_ids(m)
    if after_ids is not None:
        after_ids()
    for fr in fronts:
        fr.phase_push()
    torch.cuda.synchronize()
    return [fr.emb.view(fr.B, fr.S, fr.dim).clone() for fr in fronts]


@pytest.mark.parametrize("world", [1, 2, 4, 8])
def test_front_rows_and_gradients_match_the_unsharded_dict(world):
    from fuxictr_b200 import sharded as SH
    from fuxictr_b200.layers import FeatureEmbeddingDict
    _build()
    fm = _din_fm()
    torch.manual_seed(1)
    fed = FeatureEmbeddingDict(fm, D).cuda()
    with torch.no_grad():
        for emb in fed.embedding_layers.values():
            emb.weight[1:].normal_(0, 0.3)
    gen = torch.Generator().manual_seed(3)
    mat = _din_batch(gen, B_L * world)
    mats = [mat[r * B_L:(r + 1) * B_L].contiguous() for r in range(world)]
    for nonzero_pad in (False, True):
        if nonzero_pad:          # a loaded checkpoint may hold a non-zero padding row: copied bit for bit
            with torch.no_grad():
                fed.embedding_layers["item_id"].weight[0].normal_(0, 1.0)
                fed.embedding_layers["user"].weight[0].fill_(0.25)
        fronts, shards = _front_ranks(fed, fm, world, {})
        landed = _push_all(fronts, mats)
        ref = _reference_rows(fed, fm, mat)
        for r in range(world):
            assert torch.equal(landed[r], ref[r * B_L:(r + 1) * B_L]), (nonzero_pad, r)
            assert int(fronts[r].status) == 0
    # gradients: every rank's gradient rows -> the owners' shards; the reference is autograd of the gather
    S = fronts[0].S
    G = torch.randn(B_L * world, S * D, generator=gen).cuda()
    ref.backward(G.view(-1, S, D))
    for r, fr in enumerate(fronts):
        fr.gemb.copy_(G[r * B_L:(r + 1) * B_L])
    grads = []
    for fr in fronts:
        distinct = [torch.zeros_like(t) for t in fr._emb_distinct]
        fr.phase_pull([distinct[i] for i in fr._emb_where], None)
        grads.append(distinct)
    torch.cuda.synchronize()
    for i, (name, emb) in enumerate([(n, fed.embedding_layers[n]) for n in ("user", "item_id", "cate_id")]):
        full = SH.unshard_rows([g[i] for g in grads], emb.num_embeddings)
        assert close(full, emb.weight.grad, 1e-5), name     # a shared table: the sum over both fields, once
        assert float(full[0].abs().max()) == 0.0, name       # the padding row gets no gradient


def test_front_autograd_counts_a_shared_table_once():
    """One virtual rank through sharded_front's own autograd: a table read by two fields is one input, and its
    gradient is the sum over both fields (not twice, not a second buffer)."""
    from fuxictr_b200 import sharded as SH
    from fuxictr_b200.layers import FeatureEmbeddingDict
    _build()
    fm = _din_fm()
    torch.manual_seed(2)
    fed = FeatureEmbeddingDict(fm, D).cuda()
    with torch.no_grad():
        for emb in fed.embedding_layers.values():
            emb.weight[1:].normal_(0, 0.3)
    fronts, shards = _front_ranks(fed, fm, 1, {})
    fr = fronts[0]
    assert len(fr.distinct_tables()) == 3 and len(fr.emb_tables) == 5
    mat = _din_batch(torch.Generator().manual_seed(4), B_L)
    emb, _ = SH.sharded_front(fr, mat)
    ref = _reference_rows(fed, fm, mat)
    assert torch.equal(emb, ref)
    G = torch.randn(ref.shape, device="cuda")
    emb.backward(G)
    ref.backward(G)
    for t, name in zip(fr.distinct_tables(), ("user", "item_id", "cate_id")):
        assert close(t.grad, fed.embedding_layers[name].weight.grad, 1e-5), name


def test_out_of_range_id_sets_status_and_lands_a_zero_row():
    _build()
    from fuxictr_b200.layers import FeatureEmbeddingDict
    fm = _din_fm()
    torch.manual_seed(5)
    fed = FeatureEmbeddingDict(fm, D).cuda()
    with torch.no_grad():
        for emb in fed.embedding_layers.values():
            emb.weight[1:].normal_(0, 0.3)
    world = 2
    mat = _din_batch(torch.Generator().manual_seed(6), B_L * world)
    good = mat.clone()
    mat[B_L + 3, fm.get_column_index("click_history")[2]] = 50          # rank 1, sample 3, history position 2
    good[B_L + 3, fm.get_column_index("click_history")[2]] = 0
    fronts, _ = _front_ranks(fed, fm, world, {})
    landed = _push_all(fronts, [mat[r * B_L:(r + 1) * B_L].contiguous() for r in range(world)])
    assert int(fronts[0].status) == 0 and int(fronts[1].status) == 4     # 1 + field index of click_history
    ref = _reference_rows(fed, fm, good)
    slot = fronts[1].slot_start[3] + 2
    assert float(landed[1][3, slot].abs().max()) == 0.0
    mask = torch.ones_like(landed[1], dtype=torch.bool)
    mask[3, slot] = False
    assert torch.equal(landed[1][mask], ref[B_L:][mask])
    assert torch.equal(landed[0], ref[:B_L])


def test_each_rank_fills_its_own_padding_slots():
    """World 4, histories half padding: after the ids launch every rank's published padding rows are replaced by
    a rank-specific marker.  The padding slots a rank receives carry ITS marker: it filled them itself, and no
    other rank (rank 0 owns row 0) served them."""
    _build()
    from fuxictr_b200.layers import FeatureEmbeddingDict
    fm = _din_fm()
    torch.manual_seed(7)
    fed = FeatureEmbeddingDict(fm, D).cuda()
    world = 4
    mat = _din_batch(torch.Generator().manual_seed(8), B_L * world, pad_frac=0.5)
    mats = [mat[r * B_L:(r + 1) * B_L].contiguous() for r in range(world)]
    fronts, _ = _front_ranks(fed, fm, world, {})

    def mark():
        torch.cuda.synchronize()
        for r, fr in enumerate(fronts):
            fr.pad_rows.fill_(100.0 + r)
    landed = _push_all(fronts, mats, after_ids=mark)
    n_pad = 0
    for r, fr in enumerate(fronts):
        for f, s0, n in zip(fr.names, fr.slot_start, fr.seq_lens):
            col = fm.get_column_index(f)
            ids = mats[r][:, col[0]:col[0] + n] if isinstance(col, list) else mats[r][:, col:col + 1]
            pad = ids.long() == 0
            rows = landed[r][:, s0:s0 + n]
            n_pad += int(pad.sum())
            assert bool((rows[pad] == 100.0 + r).all()), (r, f)
            assert not bool((rows[~pad] >= 100.0).any()), (r, f)
    assert n_pad >= world * B_L * L      # half of both histories, at least


# ------------------------------------------------------------------ model level
def _model(name, fm, structure=None, act="Dice"):
    from fuxictr_b200 import zoo
    torch.manual_seed(123)
    if name == "DCNv2":
        m = zoo.DCNv2(fm, gpu=0, embedding_dim=D, model_structure=structure, num_cross_layers=2,
                      parallel_dnn_hidden_units=[16, 8])
    elif name == "xDeepFM":
        m = zoo.xDeepFM(fm, gpu=0, embedding_dim=D, dnn_hidden_units=[16], cin_hidden_units=[8, 8])
    else:
        m = zoo.DIN(fm, gpu=0, embedding_dim=D, dnn_hidden_units=[16, 8], attention_hidden_units=[8],
                    attention_hidden_activations=act)
    with torch.no_grad():
        for mod in m.modules():
            if isinstance(mod, torch.nn.Embedding):
                mod.weight[1:].normal_(0, 0.3)
    return m


def _ranks(make, world, fm, lazy=False):
    from fuxictr_b200 import sharded as SH
    registry, models = {}, []
    for r in range(world):
        m = make()
        m.enable_sharding(SH.VirtualPeerGroup(r, world, registry), B_L, fm.input_length + 1, torch.float64,
                          want_fm=False)
        m.use_fused_optimizer(lazy_tables=lazy)
        models.append(m)
    return models


def _lockstep_train_step(models, mats, fm):
    """fused_train_step of every virtual rank in lock step (see tests/test_gpu_lazy_sharded.py); returns the
    per-rank losses."""
    from fuxictr_b200 import sharded as SH, functional as F2
    fronts = [m._sharded_front for m in models]
    for m in models:
        m._fused_optimizer.zero_grad()
    for fr, mat in zip(fronts, mats):
        fr.phase_ids(mat)
    for fr in fronts:
        fr.phase_push()
    outs = [fr.phase_reduce() for fr in fronts]
    losses, leaves = [], []
    real_front = SH.sharded_front
    try:
        for m, fr, mat, (emb, logit, _) in zip(models, fronts, mats, outs):
            e = emb.view(fr.B, fr.S, fr.dim).detach().requires_grad_(True)
            lg = logit.detach().requires_grad_(True)
            leaves.append((e, lg))
            SH.sharded_front = lambda front, batch_matrix, _e=e, _lg=lg: (_e, _lg)
            m._fused_optimizer.step = lambda: None
            m._fused_optimizer.zero_grad = lambda: None
            losses.append(float(m.fused_train_step(fm.batch_dict(mat)).detach()))
    finally:
        SH.sharded_front = real_front
        for m in models:
            del m._fused_optimizer.step
            del m._fused_optimizer.zero_grad
    for m, fr, (emb, _, sums), (e, lg) in zip(models, fronts, outs, leaves):
        gx = e.grad.reshape(fr.B, -1)
        gl = None
        if fr.lr_tables:
            gl = lg.grad.reshape(-1) if lg.grad is not None else torch.zeros(fr.B, device="cuda")
        gbias = F2._grad_buffer(fr.bias, zero=False) if fr.bias is not None else None
        fr.phase_gprep(gx, emb, sums, gl, gbias)
    for fr in fronts:
        eg = [F2._grad_buffer(t, zero=True) for t in fr._emb_distinct]
        lg_ = [F2._grad_buffer(t, zero=True) for t in fr._lr_distinct]
        fr.phase_pull([eg[i] for i in fr._emb_where], [lg_[i] for i in fr._lr_where] if fr.lr_tables else None)
    SH.lockstep_steps([m._fused_optimizer for m in models])
    return losses


def _reference_steps(ref, batches, world, data_parallel):
    """The unsharded model with torch's Adam + clip_grad_norm_: one step per global batch, or (data_parallel)
    the local batches' losses scaled by 1/world with their gradients summed, then one step."""
    losses = []
    for mat in batches:
        ref.optimizer.zero_grad()
        if data_parallel:
            total = 0.0
            for r in range(world):
                part = ref.fm_.batch_dict(mat[r * B_L:(r + 1) * B_L].contiguous())
                loss = ref.compute_loss(ref.forward(part), ref.get_labels(part)) / world
                loss.backward()
                total += float(loss)
            losses.append(total)
        else:
            batch = ref.fm_.batch_dict(mat)
            loss = ref.compute_loss(ref.forward(batch), ref.get_labels(batch))
            loss.backward()
            losses.append(float(loss))
        torch.nn.utils.clip_grad_norm_(ref.parameters(), ref._max_gradient_norm)
        ref.optimizer.step()
    return losses


def _check_states(models, ref, world, skip=()):
    from fuxictr_b200 import sharded as SH
    sd_ref = ref.state_dict()
    for r, m in enumerate(models):
        for k, v in m.state_dict().items():
            if any(s in k for s in skip):
                continue
            want = sd_ref[k]
            if "embedding_layers" in k:
                want = SH.shard_rows(want, r, world)
            assert close(v, want, 1e-5), (r, k)


_MODELS = [
    ("DCNv2", "parallel", None, False),
    ("DCNv2", "crossnet_only", None, False),
    ("xDeepFM", None, None, False),
    ("DIN", None, "Dice", True),          # Dice: batch statistics per rank -> the data-parallel reference
    ("DIN", None, "ReLU", False),
]


@pytest.mark.parametrize("world", [1, 2, 4])
@pytest.mark.parametrize("name,structure,act,dp", _MODELS)
def test_sharded_models_train_like_the_unsharded_model(name, structure, act, dp, world):
    _build()
    from fuxictr_b200.schema import FeatureMap
    if name == "DIN":
        fm = _din_fm()
    else:
        fm = FeatureMap.from_specs(_CAT, embedding_dim=D)

    def make():
        return _model(name, fm, structure, act)
    ref = make()
    ref.fm_ = fm
    models = _ranks(make, world, fm)
    gen = torch.Generator().manual_seed(21)
    batches = []
    for _ in range(3):
        if name == "DIN":
            batches.append(_din_batch(gen, B_L * world))
        else:
            ids = torch.cat([torch.randint(0, s["vocab_size"], (B_L * world, 1), generator=gen) for _, s in _CAT], 1)
            batches.append(torch.cat([ids.double(), (torch.rand(B_L * world, 1, generator=gen) < 0.4).double()],
                                     1).cuda())
    losses = []
    for mat in batches:
        mats = [mat[r * B_L:(r + 1) * B_L].contiguous() for r in range(world)]
        if world == 1:       # one virtual rank: the model's own fused_train_step, sharded front autograd included
            losses.append(float(models[0].fused_train_step(fm.batch_dict(mats[0])).detach()))
        else:
            losses.append(sum(_lockstep_train_step(models, mats, fm)) / world)
    ref_losses = _reference_steps(ref, batches, world, dp)
    for a, b in zip(losses, ref_losses):
        assert abs(a - b) <= 1e-5 * abs(b), (losses, ref_losses)
    # Dice's running statistics follow each rank's own batches (not a state the ranks share)
    _check_states(models, ref, world, skip=("running_", "num_batches") if dp else ())


def test_din_with_relu_attention_at_eight_ranks():
    _build()
    fm = _din_fm()

    def make():
        return _model("DIN", fm, None, "ReLU")
    world = 8
    ref = make()
    ref.fm_ = fm
    models = _ranks(make, world, fm)
    gen = torch.Generator().manual_seed(22)
    batches = [_din_batch(gen, B_L * world) for _ in range(3)]
    losses = [sum(_lockstep_train_step(models, [m[r * B_L:(r + 1) * B_L].contiguous() for r in range(world)], fm))
              / world for m in batches]
    ref_losses = _reference_steps(ref, batches, world, False)
    for a, b in zip(losses, ref_losses):
        assert abs(a - b) <= 1e-5 * abs(b), (losses, ref_losses)
    _check_states(models, ref, world)


@pytest.mark.parametrize("world", [1, 2])
def test_sharded_lazy_xdeepfm_tracks_sharded_dense_xdeepfm(world):
    """xDeepFM reads its tables (and LR tables) through the push's replay when they are lazy."""
    _build()
    from fuxictr_b200.schema import FeatureMap
    fm = FeatureMap.from_specs(_CAT, embedding_dim=D)

    def make():
        return _model("xDeepFM", fm)
    dense = _ranks(make, world, fm, lazy=False)
    lazy = _ranks(make, world, fm, lazy=True)
    gen = torch.Generator().manual_seed(23)
    for step in range(4):
        ids = torch.cat([torch.randint(0, s["vocab_size"], (B_L * world, 1), generator=gen) for _, s in _CAT], 1)
        mat = torch.cat([ids.double(), (torch.rand(B_L * world, 1, generator=gen) < 0.4).double()], 1).cuda()
        mats = [mat[r * B_L:(r + 1) * B_L].contiguous() for r in range(world)]
        if world == 1:
            l0 = [float(dense[0].fused_train_step(fm.batch_dict(mats[0])))]
            l1 = [float(lazy[0].fused_train_step(fm.batch_dict(mats[0])))]
        else:
            l0 = _lockstep_train_step(dense, mats, fm)
            l1 = _lockstep_train_step(lazy, mats, fm)
        for a, b in zip(l0, l1):
            assert abs(a - b) <= 1e-6 * abs(a), step
    for d, l in zip(dense, lazy):
        sd0, sd1 = d.state_dict(), l.state_dict()
        for k in sd0:
            assert close(sd0[k], sd1[k], 1e-6, atol=1e-9), k

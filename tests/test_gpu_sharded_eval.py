"""Evaluation and prediction of row-sharded models: `world` virtual ranks on ONE GPU
(fuxictr_b200.sharded.VirtualPeerGroup; the kernels cannot tell a local pointer from a peer pointer), driven by
sharded.lockstep_evaluate / lockstep_predict, which run every rank's evaluation round phase by phase in the
order the barriers impose on real ranks.

The validation split has k * B_L * world + 3 rows and every rank reads its shard through
MatrixDataLoader(shard=(rank, world), drop_last=False): the last round is ragged, and at world 8 five ranks have
0 rows in it (they serve their peers and skip their dense forward).  Each model first takes two lockstep
training steps.  The unsharded twin carries the sharded weights (tables unsharded, dense part of rank 0)."""
import sys

import numpy as np
import pytest
import torch

from conftest import close, ROOT

sys.path.insert(0, ROOT)
from oracle import fuxictr_oracle as O  # noqa: E402

pytestmark = pytest.mark.gpu

D, B_L, L, K = 8, 16, 6, 2
_CAT = [("C%d" % i, {"type": "categorical", "source": "", "padding_idx": 0, "vocab_size": 60 + 17 * i})
        for i in range(7)]
_SEQ = [
    ("user", {"type": "categorical", "source": "", "padding_idx": 0, "vocab_size": 30}),
    ("item_id", {"type": "categorical", "source": "", "padding_idx": 0, "vocab_size": 50}),
    ("cate_id", {"type": "categorical", "source": "", "padding_idx": 0, "vocab_size": 12}),
    ("click_history", {"type": "sequence", "source": "", "padding_idx": 0, "vocab_size": 50, "max_len": L,
                       "share_embedding": "item_id"}),
    ("cate_history", {"type": "sequence", "source": "", "padding_idx": 0, "vocab_size": 12, "max_len": L,
                      "share_embedding": "cate_id"}),
]
_MODELS = [("DeepFM", None), ("DLRM", None), ("DCNv2", "parallel"), ("DCNv2", "crossnet_only"), ("xDeepFM", None),
           ("DIN", None)]


@pytest.fixture(scope="module", autouse=True)
def _built():
    import __graft_entry__
    __graft_entry__.build()
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"


@pytest.fixture
def precision(request):
    from fuxictr_b200 import functional as F2
    old = F2.get_matmul_precision()
    yield F2.set_matmul_precision
    F2.set_matmul_precision(old)


def _fm(name):
    from fuxictr_b200.schema import FeatureMap
    return FeatureMap.from_specs(_SEQ if name == "DIN" else _CAT, embedding_dim=D)


def _make(name, fm, structure=None):
    from fuxictr_b200 import zoo
    torch.manual_seed(123)
    if name == "DeepFM":
        m = zoo.DeepFM(fm, gpu=0, embedding_dim=D, hidden_units=[32, 16])
    elif name == "DLRM":
        m = zoo.DLRM(fm, gpu=0, embedding_dim=D, top_mlp_units=[32, 16], bottom_mlp_units=[16], interaction_op="dot")
    elif name == "DCNv2":
        m = zoo.DCNv2(fm, gpu=0, embedding_dim=D, model_structure=structure, num_cross_layers=2,
                      parallel_dnn_hidden_units=[16, 8])
    elif name == "xDeepFM":
        m = zoo.xDeepFM(fm, gpu=0, embedding_dim=D, dnn_hidden_units=[16], cin_hidden_units=[8, 8])
    else:
        m = zoo.DIN(fm, gpu=0, embedding_dim=D, dnn_hidden_units=[16, 8], attention_hidden_units=[8],
                    attention_hidden_activations="ReLU")
    with torch.no_grad():
        for mod in m.modules():
            if isinstance(mod, torch.nn.Embedding):
                mod.weight[1:].normal_(0, 0.3)
    return m


def _ranks(name, fm, world, structure=None, lazy=False):
    from fuxictr_b200 import sharded as SH
    registry, models = {}, []
    for r in range(world):
        m = _make(name, fm, structure)
        m.enable_sharding(SH.VirtualPeerGroup(r, world, registry), B_L, fm.input_length + 1, torch.float64,
                          want_fm=(name == "DeepFM"))
        m.use_fused_optimizer(lazy_tables=lazy)
        models.append(m)
    return models


def _rows(name, gen, n):
    """n rows of the batch matrix (float64, CPU): ids with some padding, DIN histories of random length, labels."""
    specs = _SEQ if name == "DIN" else _CAT
    cols = []
    lens = torch.randint(0, L + 1, (n,), generator=gen)
    keep = torch.arange(L).view(1, L) < lens.view(n, 1)
    for _, s in specs:
        if s["type"] == "sequence":
            h = torch.randint(1, s["vocab_size"], (n, L), generator=gen)
            cols.append(torch.where(keep, h, torch.zeros_like(h)))
        else:
            cols.append(torch.randint(0, s["vocab_size"], (n, 1), generator=gen))
    cols.append((torch.rand(n, 1, generator=gen) < 0.4).long())
    return torch.cat(cols, 1).double()


def _lockstep_train_step(models, mats, fm):
    """fused_train_step of every virtual rank in lock step (as tests/test_gpu_sharded_models.py): the sharded
    front's phases for all ranks between its barriers, the rest of each rank's step its own fused_train_step."""
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
        needs_logit = bool(fr.lr_tables) or fr.want_fm
        gl = (lg.grad.reshape(-1) if lg.grad is not None else torch.zeros(fr.B, device="cuda")) if needs_logit else None
        gbias = F2._grad_buffer(fr.bias, zero=False) if fr.bias is not None else None
        fr.phase_gprep(gx, emb, sums, gl, gbias)
    for fr in fronts:
        eg = [F2._grad_buffer(t, zero=True) for t in fr._emb_distinct]
        lg_ = [F2._grad_buffer(t, zero=True) for t in fr._lr_distinct]
        fr.phase_pull([eg[i] for i in fr._emb_where], [lg_[i] for i in fr._lr_where] if fr.lr_tables else None)
    SH.lockstep_steps([m._fused_optimizer for m in models])
    return losses


def _train(models, name, fm, gen, steps):
    world = len(models)
    out = []
    for _ in range(steps):
        mat = _rows(name, gen, B_L * world).cuda()
        out.append(_lockstep_train_step(models, [mat[r * B_L:(r + 1) * B_L].contiguous() for r in range(world)], fm))
    return out


def _unsharded_twin(name, fm, models, structure=None):
    """The unsharded model with the sharded ranks' weights: every table unsharded, the dense part of rank 0."""
    from fuxictr_b200 import sharded as SH
    ref = _make(name, fm, structure)
    sds = [m.state_dict() for m in models]
    want = {}
    for k, v in ref.state_dict().items():
        want[k] = SH.unshard_rows([sd[k] for sd in sds], v.shape[0]) if "embedding_layers" in k else sds[0][k]
    ref.load_state_dict(want)
    return ref


def _split(name, world, seed=7):
    n = K * B_L * world + 3
    return _rows(name, torch.Generator().manual_seed(seed), n).numpy()


def _loaders(fm, data, world):
    from fuxictr_b200.dataloader import MatrixDataLoader
    return [MatrixDataLoader(fm, data, batch_size=B_L, shard=(r, world), drop_last=False, pin=False)
            for r in range(world)]


def _expected_landed(ref, front, mat):
    """The unsharded gather of the same rows: (rows, S, D), slot order of the front."""
    fed = ref.embedding_layer
    from fuxictr_b200.layers import FeatureEmbeddingDict
    if not isinstance(fed, FeatureEmbeddingDict):
        fed = fed.embedding_layer
    parts = []
    for f, col, n in zip(front.names, front.columns, front.seq_lens):
        ids = mat[:, col:col + n].long().cuda()
        parts.append(fed.embedding_layers[f].weight.detach()[ids])
    return torch.cat(parts, 1)


@pytest.mark.parametrize("world", [2, 8])
@pytest.mark.parametrize("name,structure", _MODELS)
def test_sharded_evaluate_and_predict_match_the_unsharded_model(name, structure, world, precision):
    from fuxictr_b200 import sharded as SH
    fm = _fm(name)
    models = _ranks(name, fm, world, structure)
    _train(models, name, fm, torch.Generator().manual_seed(21), 2)
    ref = _unsharded_twin(name, fm, models, structure)
    data = _split(name, world)
    # the tail: ranks 0..2 get one row each, the others none
    sizes = [list(ld._spans())[-1] for ld in _loaders(fm, data, world)]
    assert [hi - lo for lo, hi in sizes] == ([1, 1, 1] + [0] * (world - 3) if world > 3 else [2, 1])

    # 1. landed rows: bit-identical to the unsharded gather of the same rows
    landed = [[] for _ in range(world)]
    for r, m in enumerate(models):
        fr = m._sharded_front
        real = fr.eval_phase_reduce

        def record(_fr=fr, _real=real, _r=r):
            out = _real()
            landed[_r].append(None if out is None else out[0].clone())
            return out
        fr.eval_phase_reduce = record
    try:
        preds = SH.lockstep_predict(models, _loaders(fm, data, world))
    finally:
        for m in models:
            del m._sharded_front.eval_phase_reduce
    for r, ld in enumerate(_loaders(fm, data, world)):
        for i, mat in enumerate(ld.matrices()):
            if mat.shape[0] == 0:
                assert landed[r][i] is None
                continue
            assert torch.equal(landed[r][i], _expected_landed(ref, models[r]._sharded_front, mat)), (r, i)
        assert int(models[r]._sharded_front.status) == 0

    for mode in ("tf32x3", "fp32"):
        precision(mode)
        # 2. each rank's predict() = the unsharded model on the same rows
        preds = SH.lockstep_predict(models, _loaders(fm, data, world))
        for r, ld in enumerate(_loaders(fm, data, world)):
            want = ref.predict([bt for bt in ld if bt["label"].shape[0] > 0])    # (the unsharded GEMMs take no 0-row batch)
            assert preds[r].dtype == np.float64 and preds[r].shape == want.shape, (mode, r)
            assert np.abs(preds[r] - want).max() <= 1e-5 * np.abs(want).max(), (mode, r)
        # 3. evaluate(): the same on every rank, bit for bit; the oracle's metrics over the rank-ordered union
        seen = []
        real_union = SH._union_metrics

        def union(ps, ys, metrics):
            seen.append(([x.cpu().numpy() for x in ps], [x.cpu().numpy() for x in ys]))
            return real_union(ps, ys, metrics)
        SH._union_metrics = union
        try:
            res = SH.lockstep_evaluate(models, _loaders(fm, data, world), ["logloss", "AUC"])
        finally:
            SH._union_metrics = real_union
        assert all(x == res[0] for x in res) and list(res[0]) == ["logloss", "AUC"]
        ps, ys = seen[0]
        for r, ld in enumerate(_loaders(fm, data, world)):      # in rank order: rank r's rows, in its order
            labels = np.concatenate([m[:, -1].numpy() for m in ld.matrices()]).astype(np.float32)
            assert np.array_equal(ys[r], labels), (mode, r)
            assert np.abs(ps[r] - preds[r]).max() <= 1e-6, (mode, r)
        y, p = np.concatenate(ys), np.concatenate(ps)
        assert y.size == data.shape[0]
        assert res[0]["AUC"] == O.auc(y, p), mode
        ll = O.logloss(y, p)
        assert abs(res[0]["logloss"] - ll) <= 1e-12 * ll, mode
        from fuxictr_b200.dataloader import MatrixDataLoader
        whole = ref.evaluate(MatrixDataLoader(fm, data, batch_size=B_L, pin=False), ["logloss", "AUC"])
        for k in whole:
            assert abs(res[0][k] - whole[k]) <= 1e-5 * abs(whole[k]), (mode, k)


@pytest.mark.parametrize("name", ["DeepFM", "DLRM", "xDeepFM"])
def test_sharded_lazy_models_evaluate_like_their_dense_twins(name):
    from fuxictr_b200 import sharded as SH
    world = 2
    fm = _fm(name)
    dense = _ranks(name, fm, world)
    lazy = _ranks(name, fm, world, lazy=True)
    _train(dense, name, fm, torch.Generator().manual_seed(31), 3)
    _train(lazy, name, fm, torch.Generator().manual_seed(31), 3)
    data = _split(name, world)
    r0 = SH.lockstep_evaluate(dense, _loaders(fm, data, world), ["logloss", "AUC"])[0]
    r1 = SH.lockstep_evaluate(lazy, _loaders(fm, data, world), ["logloss", "AUC"])[0]
    for k in r0:
        assert abs(r0[k] - r1[k]) <= 1e-5 * abs(r0[k]), k
    p0 = SH.lockstep_predict(dense, _loaders(fm, data, world))
    p1 = SH.lockstep_predict(lazy, _loaders(fm, data, world))
    for a, b in zip(p0, p1):
        assert np.abs(a - b).max() <= 1e-5


@pytest.mark.parametrize("name,structure", [("DeepFM", None), ("DLRM", None), ("DCNv2", "parallel"),
                                            ("xDeepFM", None), ("DIN", None)])
@pytest.mark.parametrize("lazy", [False, True])
def test_training_after_an_evaluation_is_unchanged(name, structure, lazy):
    """Three steps after an evaluate() = three steps without it (1e-6: the float-atomic order of the gradient
    scatter already separates two identical runs in the last bits); the owned list and lazy state the
    training push leaves are its own."""
    from fuxictr_b200 import sharded as SH
    if lazy and name not in ("DeepFM", "DLRM", "xDeepFM"):
        pytest.skip("lazy tables are for DeepFM, DLRM and xDeepFM")
    world = 2
    fm = _fm(name)
    a = _ranks(name, fm, world, structure, lazy)
    b = _ranks(name, fm, world, structure, lazy)
    _train(a, name, fm, torch.Generator().manual_seed(41), 2)
    _train(b, name, fm, torch.Generator().manual_seed(41), 2)
    SH.lockstep_evaluate(a, _loaders(fm, _split(name, world), world), ["logloss", "AUC"])
    for m in a + b:
        m.train()
    la = _train(a, name, fm, torch.Generator().manual_seed(42), 3)
    lb = _train(b, name, fm, torch.Generator().manual_seed(42), 3)
    for x, y in zip(la, lb):
        for u, v in zip(x, y):
            assert abs(u - v) <= 1e-6 * abs(v), (la, lb)
    for ma, mb in zip(a, b):
        sa, sb = ma.state_dict(), mb.state_dict()
        for k in sa:
            assert close(sa[k], sb[k], 1e-6, atol=1e-9), k


def test_one_virtual_rank_evaluates_through_the_model():
    """World 1 needs no lock step: RankModel.evaluate / predict of the sharded model run the round themselves."""
    name = "DLRM"
    fm = _fm(name)
    models = _ranks(name, fm, 1)
    _train(models, name, fm, torch.Generator().manual_seed(51), 2)
    ref = _unsharded_twin(name, fm, models)
    data = _split(name, 1)
    ld = _loaders(fm, data, 1)[0]
    got, want = models[0].evaluate(ld, ["logloss", "AUC"]), ref.evaluate(ld, ["logloss", "AUC"])
    for k in want:
        assert abs(got[k] - want[k]) <= 1e-5 * abs(want[k]), k
    p, q = models[0].predict(ld), ref.predict(ld)
    assert np.abs(p - q).max() <= 1e-5

"""TransAct without a GPU: the float64 restatement against the reference's goldens, construction against the
reference's digests (names, children, registration order, initial draws), the refusals, the C-ABI range checks of the
new entry points, their header and ctypes declarations, and the new kernels' register use."""
import ctypes
import hashlib
import json
import os
import subprocess
import sys

import pytest
import torch

from conftest import Golden, GOLDEN, ROOT, close, rel_err

sys.path.insert(0, ROOT)
from oracle import fuxictr_oracle as O  # noqa: E402
import transact_oracle as TO  # noqa: E402
from fuxictr_b200 import _lib, functional as F2, layers, zoo  # noqa: E402
from fuxictr_b200.schema import FeatureMap  # noqa: E402

MODULE_CASES = ["h1_k1_pool", "h2_l2_k3_pool_tuple", "h4_k2_nopool", "h1_l2_k1_pool_ties"]
MODEL_CASES = ["tuple_k1_pool", "two_pairs_k2_nopool", "h4_k3_bn"]
ENTRY_POINTS = ["b2_transact_tokens_fwd", "b2_transact_tokens_bwd", "b2_transact_attn_fwd", "b2_transact_attn_bwd",
                "b2_transact_out_fwd", "b2_transact_out_bwd"]


# ------------------------------------------------------------------ oracle vs the reference's goldens
@pytest.mark.parametrize("c", MODULE_CASES)
def test_oracle_module_matches_reference_golden(c):
    g = Golden("next_TransActTransformer_" + c)
    _, L, D, ns, nt, H, n, ffn, k, pool = g.meta["case"]
    st = {kk: v.clone().double().requires_grad_(True) for kk, v in g["w"].items()}
    seq = g["in"]["seq"].clone().double().requires_grad_(True)
    tgt = g["in"]["tgt"].clone().double().requires_grad_(True)
    out = TO.transformer(seq, tgt, g["in"]["ids"].clone(), st, "", H, n, k, pool)
    assert close(out, g["out"]["y"], 2e-6, atol=1e-7), rel_err(out, g["out"]["y"])
    (out * g["in"]["gout"].double()).sum().backward()
    for got, ref in ((seq.grad, g["gin"]["seq"]), (tgt.grad, g["gin"]["tgt"])):
        assert close(got, ref, 2e-6, atol=2e-6 * float(ref.abs().max())), rel_err(got, ref)
    want = g["g"]
    scale = max(float(v.abs().max()) for v in want.values())
    for kk, ref in want.items():
        assert close(st[kk].grad, ref, 2e-6, atol=2e-6 * scale), (kk, rel_err(st[kk].grad, ref))


def test_module_goldens_cover_empty_full_ragged_and_ties():
    """Every module golden holds an empty history, a full one, left- and right-padded ragged ones, and a repeated item
    whose tokens tie in the max-pool (the reference routes their gradient to the first slot)."""
    for c in MODULE_CASES:
        g = Golden("next_TransActTransformer_" + c)
        ids = g["in"]["ids"]
        lens = (ids != 0).sum(dim=1)
        L = ids.shape[1]
        assert int(lens[0]) == 0 and int(lens[1]) == L, c
        assert bool((ids[3:, 0] == 0).any()) and bool((ids[3:, -1] == 0).any()), c
        assert torch.equal(g["in"]["seq"][2, 0], g["in"]["seq"][2, 1]) and int(ids[2, 0]) == int(ids[2, 1]) != 0, c


def oracle_pred_fn(g):
    kw, specs = g.meta["kwargs"], g.specs()
    return lambda s, X: torch.sigmoid(TO.transact_logit(specs, s, X, kw))


@pytest.mark.parametrize("name", MODEL_CASES)
def test_oracle_models_match_reference_trajectory(name):
    """test_oracle_golden.py's recipe: forward, loss and every gradient on batch 0, then three clip + Adam steps."""
    g = Golden("model_TransAct_" + name)
    fm = FeatureMap.from_specs(g.meta["specs"], labels=g.meta["labels"])
    B = g.meta["batch"]
    mat = g["in"]["matrix"]
    batches = [fm.batch_dict(mat[i * B:(i + 1) * B]) for i in range(3)]
    tr = O.OracleTrainer(dict(g["w"]), oracle_pred_fn(g), g.specs(), g.meta["labels"])
    y_pred, y = tr.forward(batches[0])
    assert rel_err(y_pred, g["out"]["y_pred"]) <= 1e-6
    loss = O.bce_mean(y_pred, y)
    assert rel_err(loss, g["out"]["loss"]) <= 1e-6
    loss.backward()
    for k, ref in g["g"].items():
        if stable_part(k, ref, g.meta["kwargs"]).numel() == 0:         # a bias before BatchNorm: exact gradient 0
            assert float(tr.state[k].grad.abs().max()) <= 1e-7 and float(ref.abs().max()) <= 1e-7, k
            continue
        assert rel_err(tr.state[k].grad, ref) <= 5e-6, k
    losses = []
    for i in range(3):
        losses.append(float(tr.train_step(batches[i]).detach()))
    assert rel_err(torch.tensor(losses), g["out"]["step_losses"]) <= 2e-6
    for k, ref in g["w3"].items():
        if not ref.is_floating_point() or stable_part(k, ref, g.meta["kwargs"]).numel() == 0:
            continue
        assert rel_err(stable_part(k, tr.state[k], g.meta["kwargs"]), stable_part(k, ref, g.meta["kwargs"])) <= 1e-5, k


def stable_part(k, t, kw):
    """t without the parts whose exact gradient is zero: the key part of in_proj_bias and the key rows' target columns
    of in_proj_weight, which add a term to every score of a query that does not depend on the key (the target part of
    a token is the same in every slot) and the softmax cancels; and a DNN bias before a BatchNorm, which the batch mean
    cancels (with that BatchNorm's running mean, which it shifts).  Adam turns the rounding noise of any implementation into +-lr steps there."""
    if kw.get("batch_norm") and k.startswith("parallel_dnn.mlp."):
        idx = int(k.split(".")[2])
        if (k.endswith(".bias") and idx % 3 == 0) or k.endswith("running_mean"):    # the bias, and the mean it moves
            return t[:0]
    if "self_attn.in_proj" not in k:
        return t
    md = t.shape[0] // 3
    if k.endswith("in_proj_bias"):
        return torch.cat([t[:md], t[2 * md:]])
    seqs = kw.get("sequence_item_field", [("click_history", "cate_history")])
    seqs = seqs if isinstance(seqs, list) else [seqs]
    pair = int(k.split(".")[1])
    sw = kw["embedding_dim"] * len(TO._flat(seqs[pair]))
    return torch.cat([t[:md].flatten(), t[md:2 * md, :sw].flatten(), t[2 * md:].flatten()])


def test_model_goldens_cover_empty_full_and_ties():
    for name in MODEL_CASES:
        g = Golden("model_TransAct_" + name)
        fm = FeatureMap.from_specs(g.meta["specs"], labels=g.meta["labels"])
        col = fm.get_column_index("click_history")
        ids = g["in"]["matrix"][:, col[0]:col[-1] + 1]
        lens = (ids != 0).sum(dim=1)
        assert int(lens.min()) == 0 and int(lens.max()) == 7, name
        assert int(ids[2, 0]) == int(ids[2, 1]) != 0, name


# ------------------------------------------------------------------ construction
def _digests(module):
    return [[k, str(v.dtype), list(v.shape), hashlib.sha256(v.detach().contiguous().numpy().tobytes()).hexdigest()]
            for k, v in module.state_dict().items()]


def _init_cases():
    with open(os.path.join(GOLDEN, "transact_init.json")) as fd:
        return json.load(fd)


def test_modules_match_reference_construction():
    """Every layer of the encoder starts as a copy of one layer (one in_proj_weight draw), as in the reference."""
    cases = _init_cases()["modules"]
    assert len(cases) == 4
    for name, case in cases.items():
        md, ffn, H, n, k, pool = case["args"]
        torch.manual_seed(case["seed"])
        m = layers.TransActTransformer(md, dim_feedforward=ffn, num_heads=H, transformer_layers=n, first_k_cols=k,
                                       concat_max_pool=pool)
        assert _digests(m) == case["state_dict"], name
        lyrs = m.transformer_encoder.layers
        for lyr in lyrs[1:]:
            assert torch.equal(lyr.self_attn.in_proj_weight, lyrs[0].self_attn.in_proj_weight)


@pytest.mark.parametrize("name", MODEL_CASES)
def test_zoo_state_dict_matches_reference_construction(name):
    """The whole model after construction: embedding, transformer encoders, CrossNetV2, parallel DNN, mlp, then
    reset_parameters (xavier-normal for the exact nn.Linears: linear1, linear2, out_linear, the cross and DNN layers;
    torch's init kept for in_proj and out_proj, a NonDynamicallyQuantizableLinear)."""
    case = _init_cases()["models"][name]
    torch.manual_seed(case["seed"])
    fm = FeatureMap.from_specs(case["specs"], labels=case["labels"], embedding_dim=case["kwargs"]["embedding_dim"])
    model = zoo.TransAct(fm, gpu=-1, **case["kwargs"])
    assert _digests(model) == case["state_dict"]


# ------------------------------------------------------------------ refusals
def _seq_fm(max_len=7, dim=4):
    specs = [("item_id", {"type": "categorical", "source": "", "padding_idx": 0, "vocab_size": 20}),
             ("click_history", {"type": "sequence", "source": "", "padding_idx": 0, "vocab_size": 20,
                                "max_len": max_len, "share_embedding": "item_id", "feature_encoder": None})]
    return FeatureMap.from_specs(specs, embedding_dim=dim)


def _transact(fm, **kw):
    args = dict(gpu=-1, embedding_dim=4, num_heads=2, dcn_hidden_units=[8], dim_feedforward=8,
                target_item_field="item_id", sequence_item_field="click_history")
    args.update(kw)
    return zoo.TransAct(fm, **args)


def test_refusals():
    with pytest.raises(AssertionError):
        _transact(_seq_fm(), num_heads=3)                         # model_dim 8, the reference's assert
    with pytest.raises(NotImplementedError, match="max_len"):
        _transact(_seq_fm(max_len=257))
    with pytest.raises(NotImplementedError, match="model_dim"):
        _transact(_seq_fm(dim=260), embedding_dim=260)
    with pytest.raises(NotImplementedError, match="head width"):
        _transact(_seq_fm(dim=160), embedding_dim=160, num_heads=1)
    with pytest.raises(NotImplementedError, match="num_heads"):
        _transact(_seq_fm(dim=32), embedding_dim=32, num_heads=32)
    with pytest.raises(NotImplementedError, match="time_window"):
        _transact(_seq_fm(), use_time_window_mask=True)
    with pytest.raises(NotImplementedError, match="first_k_cols"):
        _transact(_seq_fm(), first_k_cols=0)
    with pytest.raises(NotImplementedError, match="first_k_cols"):
        _transact(_seq_fm(max_len=7), first_k_cols=8)
    with pytest.raises(NotImplementedError, match="time_window"):
        layers.TransActTransformer(8, use_time_window_mask=True)
    m = _transact(_seq_fm(max_len=7), first_k_cols=7, unknown_keyword=1)     # k = L, unknown keywords ignored
    with pytest.raises(NotImplementedError, match="lazy"):
        m.use_fused_optimizer(lazy_tables=True)
    with pytest.raises(ValueError, match="FM"):
        m.enable_sharding(None, 8, 10, want_fm=True)
    with pytest.raises(NotImplementedError):
        m.transformer_encoders[0](None, None)
    assert F2.transact_bound(256, 512, 2, 8) is None and F2.transact_bound(100, 256, 1) is None
    assert F2.transact_bound(1, 2, 1) is None
    assert F2.transact_bound(257, 8, 1) and F2.transact_bound(0, 8, 1) and F2.transact_bound(6, 513, 1)
    assert F2.transact_bound(6, 8, 17) and F2.transact_bound(6, 514, 2) and F2.transact_bound(6, 8, 1, parts=9)
    assert F2.transact_bound(6, 9, 2) and "head width" in F2.transact_bound(6, 258, 1)


# ------------------------------------------------------------------ C-ABI
def test_header_and_ctypes_declare_the_entry_points():
    from test_abi import header_prototypes
    protos = header_prototypes()
    for name in ENTRY_POINTS:
        assert name in protos and name in _lib.SIGNATURES, name
        assert len(_lib.SIGNATURES[name][1]) == protos[name], name
    with open(os.path.join(ROOT, "include", "fuxictr_b200.h")) as fd:
        text = fd.read()
    for const in ("MAX_LEN", "MAX_DIM", "MAX_HEAD_DIM", "MAX_HEADS", "MAX_PARTS"):
        assert "#define B2_TRANSACT_%s %d" % (const, getattr(_lib, "B2_TRANSACT_" + const)) in text, const


def test_kernel_range_is_checked_before_any_cuda_call():
    import __graft_entry__
    __graft_entry__.build()
    L = _lib.load()
    p = ctypes.c_void_p(4096)
    z = ctypes.c_void_p(0)

    def afwd(B=8, Lt=50, md=128, H=1, v=p, aux=z, dt=0, ld=0, scale=0.09):
        return L.b2_transact_attn_fwd(p, v, B, Lt, md, H, scale, z, 0, 0, 0.0, p, aux, dt, ld, p, p, None)

    def abwd(B=8, Lt=50, md=128, H=1, aux=z, dt=0, ld=0, delta=p):
        return L.b2_transact_attn_bwd(p, p, p, p, p, p, B, Lt, md, H, 0.09, z, 0, 0, 0.0, delta, p, aux, dt, ld, None)
    assert afwd(Lt=257) == -1 and b"max_len" in L.b2_last_error()
    assert afwd(Lt=0) == -1 and b"max_len" in L.b2_last_error()
    assert afwd(md=513, H=9) == -1 and b"model_dim" in L.b2_last_error()
    assert afwd(H=17, md=34) == -1 and b"heads" in L.b2_last_error()
    assert afwd(H=3) == -1 and b"divide" in L.b2_last_error()
    assert afwd(md=258, H=1) == -1 and b"head width" in L.b2_last_error()
    assert afwd(B=-1) == -1 and b"negative" in L.b2_last_error()
    assert afwd(B=(1 << 31) // 50 + 1) == -1 and b"2^31" in L.b2_last_error()
    assert afwd(v=z) == -1 and b"NULL" in L.b2_last_error()
    assert afwd(scale=0.0) == -1 and b"scale" in L.b2_last_error()
    assert afwd(aux=p, dt=_lib.B2_BF16, ld=127) == -1 and b"ld_aux" in L.b2_last_error()
    assert abwd(aux=p, dt=_lib.B2_F32, ld=383) == -1 and b"ld_aux" in L.b2_last_error()     # dQKV's row is 3 md wide
    assert abwd(delta=z) == -1 and b"NULL" in L.b2_last_error()
    assert abwd(md=512, H=1) == -1 and b"head width" in L.b2_last_error()
    assert afwd(B=0) == 0 and abwd(B=0) == 0 and afwd(B=0, md=256, Lt=256) == 0
    arr = (ctypes.c_void_p * 8)(*([4096] * 8))
    lds = (ctypes.c_int64 * 8)(*([4096] * 8))

    def tfwd(ns=1, nt=1, ids=p, dt=_lib.B2_F64, ld_ids=50, B=8, Lt=50, D=64, tok=p, valid=p):
        return L.b2_transact_tokens_fwd(arr, lds, ns, arr, lds, nt, ids, dt, ld_ids, B, Lt, D, tok, z, 0, 0, valid,
                                        None)
    assert tfwd(ns=5, nt=4) == -1 and b"fields per token" in L.b2_last_error()
    assert tfwd(nt=0) == -1 and b"fields per token" in L.b2_last_error()
    assert tfwd(ids=z) == -1 and b"NULL" in L.b2_last_error()
    assert tfwd(valid=z) == -1 and b"NULL" in L.b2_last_error()
    assert tfwd(dt=_lib.B2_BF16) == -1 and b"ids dtype" in L.b2_last_error()
    assert tfwd(ld_ids=49) == -1 and b"ld_ids" in L.b2_last_error()
    assert tfwd(D=300) == -1 and b"model_dim" in L.b2_last_error()
    assert tfwd(B=0) == 0
    assert L.b2_transact_tokens_bwd(p, 8, 50, 64, 1, 1, arr, z, None) == -1 and b"NULL" in L.b2_last_error()
    assert L.b2_transact_tokens_bwd(p, 8, 50, 64, 8, 1, arr, arr, None) == -1
    assert L.b2_transact_tokens_bwd(p, 0, 50, 64, 1, 1, arr, arr, None) == 0

    def ofwd(k=1, maxv=p, arg=p, aux=z, B=8):
        return L.b2_transact_out_fwd(p, p, B, 50, 128, k, p, maxv, arg, aux, 0, 128, None)
    assert ofwd(k=0) == -1 and b"first_k_cols" in L.b2_last_error()
    assert ofwd(k=51) == -1 and b"first_k_cols" in L.b2_last_error()
    assert ofwd(arg=z) == -1 and b"both or neither" in L.b2_last_error()
    assert ofwd(maxv=z, arg=z, aux=p) == -1 and b"max_aux" in L.b2_last_error()
    assert ofwd(B=0, k=50) == 0
    assert L.b2_transact_out_bwd(p, p, z, p, 8, 50, 128, 1, p, None) == -1 and b"argmax" in L.b2_last_error()
    assert L.b2_transact_out_bwd(p, z, z, p, 8, 50, 128, 51, p, None) == -1 and b"first_k_cols" in L.b2_last_error()
    assert L.b2_transact_out_bwd(p, z, z, p, 0, 50, 128, 1, p, None) == 0


# ------------------------------------------------------------------ register use
def test_new_kernels_do_not_spill(tmp_path):
    nvcc = "/usr/local/cuda/bin/nvcc"
    from fuxictr_b200 import build
    nvcc = os.environ.get("NVCC") or (nvcc if os.path.exists(nvcc) else "nvcc")
    r = subprocess.run([nvcc] + build.NVCC_FLAGS + ["-Xptxas", "-v", "-I", build.INCLUDE, "-c",
                        os.path.join(build.CSRC, "transact.cu"), "-o", str(tmp_path / "transact.o")],
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    log = r.stdout + r.stderr
    kernels = [line for line in log.splitlines() if "Compiling entry function" in line]
    assert len(kernels) == 16, log           # tokens 2, out 2, and fwd, dQ, dKV at 1, 2, 4, 8 columns per lane
    assert all("ta_" in k for k in kernels)
    spills = [line for line in log.splitlines() if "spill" in line]
    assert len(spills) == 16 and all("0 bytes spill stores, 0 bytes spill loads" in s for s in spills), log

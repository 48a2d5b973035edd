"""BST without a GPU: the float64 restatement against the reference's goldens, construction against the reference's
digests (names, children, registration order, initial draws), the refusals, the C-ABI range checks (BST's entry points
and the LeakyReLU activation code in every entry point that takes an activation), and the new kernels' register
use."""
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
import bst_oracle as BO  # noqa: E402
from fuxictr_b200 import _lib, functional as F2, layers, zoo  # noqa: E402
from fuxictr_b200.schema import FeatureMap  # noqa: E402

BLOCK_CASES = ["ln_h4", "noln_h3_causal", "nores_h1", "ln_h2_causal"]
MODEL_CASES = ["tuple_mean", "sum_nopos_causal", "target_two_pairs", "concat_noln"]


# ------------------------------------------------------------------ oracle vs the reference's goldens
@pytest.mark.parametrize("c", BLOCK_CASES)
def test_oracle_block_matches_reference_golden(c):
    g = Golden("next_TransformerBlock_" + c)
    _, md, H, ln, res, causal = g.meta["case"]
    st = {k: v.clone().double().requires_grad_(True) for k, v in g["w"].items()}
    x = g["in"]["x"].clone().double().requires_grad_(True)
    out = BO.transformer_block(x, g["in"]["valid"].bool(), st, "", H, ln, res, causal)
    assert close(out, g["out"]["y"], 2e-6), rel_err(out, g["out"]["y"])
    (out * g["in"]["gout"].double()).sum().backward()
    assert close(x.grad, g["gin"]["x"], 2e-6), rel_err(x.grad, g["gin"]["x"])
    want = g["g"]
    scale = max(float(v.abs().max()) for v in want.values())
    for k, ref in want.items():
        assert close(st[k].grad, ref, 2e-6, atol=2e-6 * scale), (k, rel_err(st[k].grad, ref))


def oracle_pred_fn(g):
    kw, specs = g.meta["kwargs"], g.specs()
    return lambda s, X: torch.sigmoid(BO.bst_logit(specs, s, X, kw))


@pytest.mark.parametrize("name", MODEL_CASES)
def test_oracle_models_match_reference_trajectory(name):
    """test_oracle_golden.py's recipe: forward, loss and every gradient on batch 0, then three clip + Adam steps."""
    g = Golden("model_BST_" + name)
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
        assert rel_err(tr.state[k].grad, ref) <= 5e-6, k
    for k in g["g"]:
        if k.endswith("attention.in_proj_bias"):
            assert float(key_bias(k, tr.state[k].grad).abs().max()) < 1e-8, k
    losses = []
    for i in range(3):
        losses.append(float(tr.train_step(batches[i]).detach()))
        if i == 0:
            for k, ref in g["w1"].items():
                assert rel_err(without_key_bias(k, tr.state[k]), without_key_bias(k, ref)) <= 5e-6, k
    assert rel_err(torch.tensor(losses), g["out"]["step_losses"]) <= 2e-6
    for k, ref in g["w3"].items():
        assert rel_err(without_key_bias(k, tr.state[k]), without_key_bias(k, ref)) <= 1e-5, k


def key_bias(k, t):
    """The key part of in_proj_bias: it adds q . b_k to every score of a query, which the softmax cancels, so its
    exact gradient is zero and Adam turns the rounding noise of any implementation into +-lr steps."""
    md = t.shape[0] // 3
    return t[md:2 * md]


def without_key_bias(k, t):
    if not k.endswith("attention.in_proj_bias"):
        return t
    md = t.shape[0] // 3
    return torch.cat([t[:md], t[2 * md:]])


def test_goldens_cover_empty_and_full_histories():
    for name in MODEL_CASES:
        g = Golden("model_BST_" + name)
        fm = FeatureMap.from_specs(g.meta["specs"], labels=g.meta["labels"])
        col = fm.get_column_index("click_history")
        lens = (g["in"]["matrix"][:, col[0]:col[-1] + 1] != 0).sum(dim=1)
        assert int(lens.min()) == 0 and int(lens.max()) == 7, name


# ------------------------------------------------------------------ construction
def _digests(module):
    return [[k, str(v.dtype), list(v.shape), hashlib.sha256(v.detach().contiguous().numpy().tobytes()).hexdigest()]
            for k, v in module.state_dict().items()]


def _init_cases():
    with open(os.path.join(GOLDEN, "bst_init.json")) as fd:
        return json.load(fd)


def test_blocks_match_reference_construction():
    cases = _init_cases()
    assert len(cases["blocks"]) == 4 and len(cases["transformers"]) == 2
    for name, case in cases["blocks"].items():
        md, H, pa, pn, ln, res = case["args"]
        torch.manual_seed(case["seed"])
        m = layers.TransformerBlock(model_dim=md, ffn_dim=md, num_heads=H, attn_dropout=pa, net_dropout=pn,
                                    layer_norm=ln, use_residual=res)
        assert _digests(m) == case["state_dict"], name
    for name, case in cases["transformers"].items():
        L, md, H, n, pd, pos = case["args"]
        torch.manual_seed(case["seed"])
        m = layers.BehaviorTransformer(seq_len=L, model_dim=md, num_heads=H, stacked_transformer_layers=n,
                                       position_dim=pd, use_position_emb=pos)
        assert _digests(m) == case["state_dict"], name


@pytest.mark.parametrize("name", MODEL_CASES)
def test_zoo_state_dict_matches_reference_construction(name):
    """The whole model after construction: embedding, transformer stacks, DNN, then reset_parameters (xavier-normal
    for the FFN Linears, torch's MHA init kept for out_proj, the sinusoidal position table kept)."""
    case = _init_cases()["models"][name]
    torch.manual_seed(case["seed"])
    fm = FeatureMap.from_specs(case["specs"], labels=case["labels"], embedding_dim=case["kwargs"]["embedding_dim"])
    model = zoo.BST(fm, gpu=-1, **case["kwargs"])
    assert _digests(model) == case["state_dict"]


# ------------------------------------------------------------------ refusals
def _seq_fm(max_len=7, dim=4):
    specs = [("item_id", {"type": "categorical", "source": "", "padding_idx": 0, "vocab_size": 20}),
             ("click_history", {"type": "sequence", "source": "", "padding_idx": 0, "vocab_size": 20,
                                "max_len": max_len, "share_embedding": "item_id", "feature_encoder": None})]
    return FeatureMap.from_specs(specs, embedding_dim=dim)


def _bst(fm, **kw):
    args = dict(gpu=-1, embedding_dim=4, num_heads=2, dnn_hidden_units=[8], bst_target_field="item_id",
                bst_sequence_field="click_history")
    args.update(kw)
    return zoo.BST(fm, **args)


def test_refusals():
    with pytest.raises(AssertionError):
        _bst(_seq_fm(), num_heads=3)                              # model_dim 8, the reference's assert
    with pytest.raises(NotImplementedError, match="max_len"):
        _bst(_seq_fm(max_len=256))
    with pytest.raises(NotImplementedError, match="model_dim"):
        _bst(_seq_fm(dim=300), embedding_dim=300)
    with pytest.raises(NotImplementedError, match="head width"):
        _bst(_seq_fm(dim=80), embedding_dim=80, num_heads=2)
    with pytest.raises(NotImplementedError, match="num_heads"):
        _bst(_seq_fm(dim=32), embedding_dim=32, num_heads=32)
    with pytest.raises(ValueError, match="seq_pooling_type"):
        _bst(_seq_fm(), seq_pooling_type="max")
    m = _bst(_seq_fm(), unknown_keyword=1)                     # unknown keywords are ignored
    with pytest.raises(NotImplementedError, match="lazy"):
        m.use_fused_optimizer(lazy_tables=True)
    with pytest.raises(ValueError, match="FM"):
        m.enable_sharding(None, 8, 10, want_fm=True)
    assert F2.bst_bound(256, 512, 8) is None and F2.bst_bound(257, 8, 1) and F2.bst_bound(6, 513, 1)
    assert F2.bst_bound(6, 8, 17) and F2.bst_bound(6, 130, 2) and F2.bst_bound(6, 8, 1, parts=9)


# ------------------------------------------------------------------ C-ABI range checks
def test_kernel_range_is_checked_before_any_cuda_call():
    import __graft_entry__
    __graft_entry__.build()
    L = _lib.load()
    p = ctypes.c_void_p(4096)
    z = ctypes.c_void_p(0)

    def afwd(B=8, Lt=51, md=32, H=4, v=p, aux=z, dt=0, ld=0, scale=0.35):
        return L.b2_bst_attn_fwd(p, v, B, Lt, md, H, 0, scale, z, 0, 0, 0.0, p, aux, dt, ld, p, p, None)

    def abwd(B=8, Lt=51, md=32, H=4, aux=z, dt=0, ld=0):
        return L.b2_bst_attn_bwd(p, p, p, p, p, p, B, Lt, md, H, 1, 0.35, z, 0, 0, 0.0, p, aux, dt, ld, None)
    assert afwd(Lt=257) == -1 and b"L = max_len + 1" in L.b2_last_error()
    assert afwd(Lt=1) == -1 and b"L = max_len + 1" in L.b2_last_error()
    assert afwd(md=513, H=9) == -1 and b"model_dim" in L.b2_last_error()
    assert afwd(H=17, md=34) == -1 and b"heads" in L.b2_last_error()
    assert afwd(H=3) == -1 and b"divide" in L.b2_last_error()
    assert afwd(md=130, H=2) == -1 and b"head width" in L.b2_last_error()
    assert afwd(B=-1) == -1 and b"negative" in L.b2_last_error()
    assert afwd(B=(1 << 31) // 51 + 1) == -1 and b"2^31" in L.b2_last_error()
    assert afwd(v=z) == -1 and b"NULL" in L.b2_last_error()
    assert afwd(scale=0.0) == -1 and b"scale" in L.b2_last_error()
    assert afwd(aux=p, dt=_lib.B2_BF16, ld=31) == -1 and b"ld_aux" in L.b2_last_error()
    assert abwd(aux=p, dt=_lib.B2_F32, ld=95) == -1 and b"ld_aux" in L.b2_last_error()     # dQKV's row is 3 md wide
    assert afwd(B=0) == 0 and abwd(B=0) == 0
    arr = (ctypes.c_void_p * 8)(*([4096] * 8))
    lds = (ctypes.c_int64 * 8)(*([4096] * 8))
    assert L.b2_bst_tokens_fwd(arr, lds, arr, lds, 9, z, 8, 6, 4, p, z, 0, 0, None) == -1
    assert b"fields per token" in L.b2_last_error()
    assert L.b2_bst_tokens_fwd(arr, lds, arr, lds, 1, z, 8, 6, 4, z, z, 0, 0, None) == -1       # NULL tokens
    assert L.b2_bst_tokens_fwd(arr, lds, arr, lds, 1, z, 0, 6, 4, p, z, 0, 0, None) == 0
    assert L.b2_bst_tokens_bwd(p, z, 8, 6, 4, 1, 1, arr, arr, z, None) == -1 and b"dpos" in L.b2_last_error()
    assert L.b2_bst_addnorm_fwd(p, z, 8, 513, z, z, 1e-5, z, 0, 0, 0.0, p, z, 0, 0, z, z, None) == -1
    assert L.b2_bst_addnorm_fwd(p, z, 8, 8, p, z, 1e-5, z, 0, 0, 0.0, p, z, 0, 0, p, p, None) == -1   # gamma, no beta
    assert L.b2_bst_addnorm_bwd(p, z, p, z, 8, 8, p, p, p, z, 0, 0, 0.0, p, z, 0, 0, z, z, z, None) == -1
    assert L.b2_bst_pool_fwd(p, p, 8, 6, 8, 3, p, 8, None) == -1 and b"pooling mode" in L.b2_last_error()
    assert L.b2_bst_pool_fwd(p, p, 8, 6, 8, 0, p, 7, None) == -1 and b"ld_out" in L.b2_last_error()
    assert L.b2_bst_pool_bwd(p, 8, z, 8, 6, 8, 0, p, None) == -1 and b"NULL" in L.b2_last_error()


def test_leaky_relu_code_is_accepted_where_activations_are():
    """B2_ACT_LEAKY_RELU passes the activation check of the SIMT GEMM, the tensor-core GEMM's act and act_bwd,
    b2_prep_operand and the head kernels: each call below stops at a later check (or, empty, returns 0), never at the
    activation's; the unused code 5 is refused."""
    import __graft_entry__
    __graft_entry__.build()
    L = _lib.load()
    p = ctypes.c_void_p(4096)
    z = ctypes.c_void_p(0)
    assert _lib.B2_ACT_LEAKY_RELU == 4
    for act, ok in ((_lib.B2_ACT_LEAKY_RELU, True), (5, False)):
        assert (L.b2_gemm_f32(p, 4, 1, p, 1, 4, p, 4, 0, 4, 4, z, act, z, z, 0, None) == 0) == ok
        assert (L.b2_prep_operand(p, p, act, 0, 4, z, z, z, z, z, z, 0, 0, 0.0, None) == 0) == ok
        assert (L.b2_head_fwd(p, p, z, 0, 4, act, p, None) == 0) == ok
        assert (L.b2_head_bwd_ex(p, p, p, p, 0, 4, act, p, p, z, act, z, z, 1, z, 0, 0, 0.0, None) == 0) == ok
        desc = _lib.b2_gemm_desc()
        desc.a = desc.b = desc.c = 4096
        desc.M = desc.N = desc.K = desc.lda = desc.ldb = desc.ldc = 16
        desc.act = desc.act_bwd = act           # the act_bwd check needs ybwd: the last check before any launch
        assert L.b2_gemm_tc_ex(ctypes.byref(desc), None) == -1
        assert (b"act_bwd needs ybwd" in L.b2_last_error()) == ok, L.b2_last_error()


# ------------------------------------------------------------------ register use
def test_new_kernels_do_not_spill(tmp_path):
    nvcc = "/usr/local/cuda/bin/nvcc"
    from fuxictr_b200 import build
    nvcc = os.environ.get("NVCC") or (nvcc if os.path.exists(nvcc) else "nvcc")
    r = subprocess.run([nvcc] + build.NVCC_FLAGS + ["-Xptxas", "-v", "-I", build.INCLUDE, "-c",
                        os.path.join(build.CSRC, "bst.cu"), "-o", str(tmp_path / "bst.o")],
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    log = r.stdout + r.stderr
    kernels = [line for line in log.splitlines() if "Compiling entry function" in line]
    assert len(kernels) == 19, log
    assert all("bst_" in k for k in kernels)
    spills = [line for line in log.splitlines() if "spill" in line]
    assert len(spills) == 19 and all("0 bytes spill stores, 0 bytes spill loads" in s for s in spills), log

"""DIEN without a GPU: the float64 restatement against the reference's goldens, construction against the reference's
digests (names, children, registration order, initial draws), the refusals, the C-ABI range checks and the new
kernels' register use."""
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
import dien_oracle as DO  # noqa: E402
from fuxictr_b200 import _lib, functional as F2, zoo  # noqa: E402
from fuxictr_b200.schema import FeatureMap  # noqa: E402

CASES = ["augru_bilinear", "agru_dot", "augru_din_sumpool", "gru_dice_bn"]


# ------------------------------------------------------------------ oracle vs the reference's goldens
@pytest.mark.parametrize("c", CASES)
def test_oracle_stack_matches_reference_golden(c):
    g = Golden("next_DIEN_" + c)
    st = {k: v.clone().double().requires_grad_(True) for k, v in g["w"].items()}
    seq = g["in"]["seq"].clone().double().requires_grad_(True)
    tgt = g["in"]["target"].clone().double().requires_grad_(True)
    out = DO.interest_stack(0, seq, tgt, g["in"]["mask"].bool(), st, g.meta["kwargs"])
    assert close(out, g["out"]["h_out"], 2e-6), rel_err(out, g["out"]["h_out"])
    (out * g["in"]["gout"].double()).sum().backward()
    assert close(seq.grad, g["gin"]["seq"], 2e-6), rel_err(seq.grad, g["gin"]["seq"])
    tgrad = torch.zeros_like(tgt) if tgt.grad is None else tgt.grad        # gru_type="GRU" reads no target
    assert close(tgrad, g["gin"]["target"], 2e-6), rel_err(tgrad, g["gin"]["target"])
    for k, ref in g["g"].items():
        assert close(st[k].grad, ref, 2e-6), (k, rel_err(st[k].grad, ref))


@pytest.mark.parametrize("name", CASES)
def test_oracle_models_match_reference_trajectory(name):
    """test_oracle_golden.py's recipe: forward, loss and every gradient on batch 0, then three clip + Adam steps."""
    g = Golden("model_DIEN_" + name)
    fm = FeatureMap.from_specs(g.meta["specs"], labels=g.meta["labels"])
    B = g.meta["batch"]
    mat = g["in"]["matrix"]
    batches = [fm.batch_dict(mat[i * B:(i + 1) * B]) for i in range(3)]
    kw, specs = g.meta["kwargs"], g.specs()
    tr = O.OracleTrainer(dict(g["w"]), lambda s, X: torch.sigmoid(DO.dien_logit(specs, s, X, kw)), specs,
                         g.meta["labels"])
    y_pred, y = tr.forward(batches[0])
    assert rel_err(y_pred, g["out"]["y_pred"]) <= 1e-6
    loss = O.bce_mean(y_pred, y)
    assert rel_err(loss, g["out"]["loss"]) <= 1e-6
    loss.backward()
    inert = inert_params(g)
    for k, ref in g["g"].items():
        if k in inert:
            assert float(tr.state[k].grad.abs().max()) < 1e-6, k
        else:
            assert rel_err(tr.state[k].grad, ref) <= 5e-6, k
    losses = []
    for i in range(3):
        losses.append(float(tr.train_step(batches[i]).detach()))
        if i == 0:
            for k, ref in g["w1"].items():
                assert k in inert or k.endswith("num_batches_tracked") or close(tr.state[k], ref, 5e-6, atol=1e-7), k
    assert rel_err(torch.tensor(losses), g["out"]["step_losses"]) <= 2e-6
    for k, ref in g["w3"].items():     # a BatchNorm's running mean follows the inert bias ahead of it
        assert k in inert or "running_" in k or k.endswith("num_batches_tracked") or close(tr.state[k], ref, 1e-5, atol=1e-7), k


def inert_params(g):
    """Parameters the output does not depend on: a DNN bias ahead of a BatchNorm, the attention MLP's last bias under
    the softmax.  Their exact gradient is zero, and Adam turns any implementation's rounding noise into +-lr steps.
    (Dice's running mean after a BatchNorm is rounding noise too: the states are compared with an absolute floor.)"""
    return set(k for k, v in g["g"].items() if float(v.abs().max()) < 1e-6)


def test_goldens_cover_the_history_kinds():
    """Each batch has an empty row, a full row, a row of length 1 and a row with a zero id inside its history."""
    for name in CASES:
        g = Golden("model_DIEN_" + name)
        fm = FeatureMap.from_specs(g.meta["specs"], labels=g.meta["labels"])
        col = fm.get_column_index("click_history")
        ids = g["in"]["matrix"][:, col[0]:col[-1] + 1]
        B, L = g.meta["batch"], ids.shape[1]
        for i in range(3):
            rows = ids[i * B:(i + 1) * B] != 0
            lens = rows.sum(dim=1)
            assert int(lens.min()) == 0 and int(lens.max()) == L and bool((lens == 1).any()), name
            last = torch.where(rows, torch.arange(L), torch.full((L,), -1)).max(dim=1).values
            assert bool((last + 1 > lens).any()), name       # a zero before the last id
    for name in CASES:
        mask = Golden("next_DIEN_" + name)["in"]["mask"].bool()
        lens = mask.sum(dim=1)
        assert int(lens.min()) == 0 and int(lens.max()) == mask.shape[1] and bool((lens == 1).any())


# ------------------------------------------------------------------ construction
def _digests(module):
    return [[k, str(v.dtype), list(v.shape), hashlib.sha256(v.detach().contiguous().numpy().tobytes()).hexdigest()]
            for k, v in module.state_dict().items()]


@pytest.mark.parametrize("name", CASES)
def test_zoo_state_dict_matches_reference_construction(name):
    """Embedding, the GRUs (torch's nn.GRU init kept), the attention (W_kernel the identity, attn_mlp xavier-normal),
    the DNN, then reset_parameters: the reference's keys, order and draws."""
    with open(os.path.join(GOLDEN, "dien_init.json")) as fd:
        case = json.load(fd)["models"][name]
    torch.manual_seed(case["seed"])
    fm = FeatureMap.from_specs(case["specs"], labels=case["labels"], embedding_dim=case["kwargs"]["embedding_dim"])
    model = zoo.DIEN(fm, gpu=-1, **case["kwargs"])
    assert _digests(model) == case["state_dict"]


# ------------------------------------------------------------------ refusals
def _seq_fm(max_len=7, dim=4, neg=False, extra_seq=False):
    specs = [("item_id", {"type": "categorical", "source": "", "padding_idx": 0, "vocab_size": 20}),
             ("click_history", {"type": "sequence", "source": "", "padding_idx": 0, "vocab_size": 20,
                                "max_len": max_len, "share_embedding": "item_id", "feature_encoder": None})]
    if neg or extra_seq:
        specs.append(("neg_click_history" if neg else "other_history",
                      {"type": "sequence", "source": "", "padding_idx": 0, "vocab_size": 20, "max_len": max_len,
                       "share_embedding": "item_id", "feature_encoder": None}))
    return FeatureMap.from_specs(specs, embedding_dim=dim)


def _dien(fm, **kw):
    args = dict(gpu=-1, embedding_dim=4, dnn_hidden_units=[8], dien_target_field="item_id",
                dien_sequence_field="click_history", dien_neg_seq_field=[])
    args.update(kw)
    return zoo.DIEN(fm, **args)


def test_refusals():
    # the reference fails in interest_emb * attn_scores: (B, L, H) times (B, L) does not broadcast
    with pytest.raises(NotImplementedError, match="AIGRU"):
        _dien(_seq_fm(), gru_type="AIGRU")
    # the reference fails in add_loss: loss += alpha * aux_loss adds an (N,) vector in place into a 0-d tensor
    with pytest.raises(NotImplementedError, match="aux_loss_alpha"):
        _dien(_seq_fm(), aux_loss_alpha=0.1)
    with pytest.raises(NotImplementedError, match="DNN input"):
        _dien(_seq_fm(), dien_neg_seq_field=["neg_click_history"])     # not in the map
    with pytest.raises(NotImplementedError, match="DNN input"):
        _dien(_seq_fm(extra_seq=True))                                  # a sequence field outside the pairs
    _dien(_seq_fm(neg=True), dien_neg_seq_field=["neg_click_history"])  # in the map: left out, the width holds
    with pytest.raises(NotImplementedError, match="Dice"):
        _dien(_seq_fm(), attention_type="din_attention", attention_activation="Dice")
    _dien(_seq_fm(), gru_type="GRU", attention_type="din_attention", attention_activation="Dice")  # no attention
    with pytest.raises(NotImplementedError, match="model_dim"):
        _dien(_seq_fm(dim=65), embedding_dim=65)
    with pytest.raises(NotImplementedError, match="max_len"):
        _dien(_seq_fm(max_len=1025))
    with pytest.raises(AssertionError):
        _dien(_seq_fm(), attention_type="general")
    m = _dien(_seq_fm(), unknown_keyword=1)                     # unknown keywords are ignored
    with pytest.raises(NotImplementedError, match="lazy"):
        m.use_fused_optimizer(lazy_tables=True)
    with pytest.raises(ValueError, match="FM"):
        m.enable_sharding(None, 8, 10, want_fm=True)
    assert F2.dien_bound(4, 1) is None and F2.dien_bound(16, 50) is None and F2.dien_bound(32, 50) is None
    assert F2.dien_bound(64, 1024) is None and F2.dien_bound(65, 8) and F2.dien_bound(0, 8) and F2.dien_bound(8, 1025)


# ------------------------------------------------------------------ C-ABI range checks
def test_kernel_range_is_checked_before_any_cuda_call():
    import __graft_entry__
    __graft_entry__.build()
    L = _lib.load()
    p = ctypes.c_void_p(4096)
    z = ctypes.c_void_p(0)

    def fwd(B=8, Lt=50, H=16, cell=1, att=p, x=p, ld=800):
        return L.b2_gru_fwd(x, ld, p, p, p, p, p, att, cell, B, Lt, H, p, z, None)

    def bwd(B=8, Lt=50, H=16, cell=1, da=p):
        return L.b2_gru_bwd(p, 800, p, p, p, p, p, p, cell, B, Lt, H, p, z, z, p, 0, da, p, p, p, p, None)
    assert fwd(H=65) == -1 and b"GRU width" in L.b2_last_error()
    assert fwd(H=0) == -1 and b"GRU width" in L.b2_last_error()
    assert fwd(Lt=1025) == -1 and b"sequence length" in L.b2_last_error()
    assert fwd(B=-1) == -1 and b"negative" in L.b2_last_error()
    assert fwd(B=(1 << 31) // 50 + 1) == -1 and b"2^31" in L.b2_last_error()
    assert fwd(x=z) == -1 and b"NULL" in L.b2_last_error()
    assert fwd(att=z) == -1 and b"attention" in L.b2_last_error()
    assert fwd(cell=3) == -1 and b"cell code" in L.b2_last_error()
    assert fwd(ld=799) == -1 and b"ld_x" in L.b2_last_error()
    assert fwd(cell=0, att=z, B=0) == 0 and fwd(B=0) == 0
    assert bwd(da=z) == -1 and b"da" in L.b2_last_error()
    assert bwd(H=65) == -1 and bwd(B=0) == 0 and bwd(cell=0, da=z, B=0) == 0
    assert L.b2_dien_scores_fwd(p, p, 15, z, p, 8, 50, 16, p, p, None) == -1 and b"ld_t" in L.b2_last_error()
    assert L.b2_dien_scores_fwd(p, p, 16, z, z, 8, 50, 16, p, p, None) == -1 and b"NULL" in L.b2_last_error()
    assert L.b2_dien_scores_bwd(p, p, 16, z, p, p, p, 8, 50, 65, p, 1, p, p, None) == -1
    assert L.b2_dien_sum_pool_fwd(p, p, 16, 8, 50, 16, p, 31, None) == -1 and b"ld_out" in L.b2_last_error()
    assert L.b2_dien_sum_pool_bwd(p, p, 16, p, 32, 8, 50, 16, z, p, 0, None) == -1 and b"NULL" in L.b2_last_error()


# ------------------------------------------------------------------ register use
def test_new_kernels_do_not_spill(tmp_path):
    from fuxictr_b200 import build
    nvcc = "/usr/local/cuda/bin/nvcc"
    nvcc = os.environ.get("NVCC") or (nvcc if os.path.exists(nvcc) else "nvcc")
    r = subprocess.run([nvcc] + build.NVCC_FLAGS + ["-Xptxas", "-v", "-I", build.INCLUDE, "-c",
                        os.path.join(build.CSRC, "dien.cu"), "-o", str(tmp_path / "dien.o")],
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    log = r.stdout + r.stderr
    kernels = [line for line in log.splitlines() if "Compiling entry function" in line]
    assert len(kernels) == 6 and all("dien_" in k for k in kernels), log
    spills = [line for line in log.splitlines() if "spill" in line]
    assert len(spills) == 6 and all("0 bytes spill stores, 0 bytes spill loads" in s for s in spills), log

"""FinalMLP without a GPU: the float64 oracle against the reference's goldens (InteractionAggregation,
FeatureSelection and four model configurations), the mirrors' and zoo models' construction against the reference's,
the refusals, the C-ABI's range checks, the launch sequences per matmul mode, and the new kernels' register use."""
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
import finalmlp_oracle as FO  # noqa: E402
from fuxictr_b200 import _lib, functional as F2, layers, zoo  # noqa: E402
from fuxictr_b200.schema import FeatureMap  # noqa: E402

AGG_TAGS = ["h1", "h2", "h3", "h2w"]
MODEL_CASES = ["FinalMLP", "FinalMLP_ctx", "FinalMLP_nofs", "DualMLP"]


# ------------------------------------------------------------------ oracle vs the reference's goldens
def _agg_config(g, tag):
    return next(c for c in g.meta["configs"] if c[0] == tag)


@pytest.mark.parametrize("tag", AGG_TAGS)
def test_oracle_aggregation_matches_reference_golden(tag):
    g = Golden("next_InteractionAggregation")
    heads = _agg_config(g, tag)[3]
    st = {k: v.clone().double().requires_grad_(True) for k, v in g["w_" + tag].items()}
    x = g["in"]["x_" + tag].clone().double().requires_grad_(True)
    y = g["in"]["y_" + tag].clone().double().requires_grad_(True)
    out = FO.interaction_aggregation(st, "", x, y, heads)
    assert close(out, g["out"][tag], 2e-6), rel_err(out, g["out"][tag])
    (out * g["in"]["gout_" + tag].double()).sum().backward()
    assert close(x.grad, g["gin"]["x_" + tag], 2e-6) and close(y.grad, g["gin"]["y_" + tag], 2e-6)
    want = g["g_" + tag]
    assert set(want) == set(st)
    for k, ref in want.items():
        assert close(st[k].grad, ref, 2e-6), (k, rel_err(st[k].grad, ref))


@pytest.mark.parametrize("tag", ["noctx", "ctx"])
def test_oracle_feature_selection_matches_reference_golden(tag):
    g = Golden("next_FeatureSelection")
    specs = g.specs()
    fm = FeatureMap.from_specs(g.meta["specs"], labels=g.meta["labels"])
    X, _ = O.split_inputs(specs, g.meta["labels"], fm.batch_dict(g["in"]["matrix"]))
    st = {k: v.clone().double().requires_grad_(True) for k, v in g["w_" + tag].items()}
    emb = g["in"]["emb_" + tag].clone().double().requires_grad_(True)
    f1, f2 = FO.feature_selection(specs, st, "", X, emb, g.meta["contexts"][tag], len(g.meta["fs_hidden_units"]))
    assert close(f1, g["out"]["f1_" + tag], 2e-6) and close(f2, g["out"]["f2_" + tag], 2e-6)
    ((f1 * g["in"]["gout1_" + tag].double()).sum() + (f2 * g["in"]["gout2_" + tag].double()).sum()).backward()
    assert close(emb.grad, g["gin"]["emb_" + tag], 2e-6), rel_err(emb.grad, g["gin"]["emb_" + tag])
    want = g["g_" + tag]
    assert set(want) == set(st)
    for k, ref in want.items():
        assert close(st[k].grad, ref, 2e-6), (k, rel_err(st[k].grad, ref))


def oracle_pred_fn(g):
    kw, specs = g.meta["kwargs"], g.specs()
    fn = FO.finalmlp_logit if g.meta["model"] == "FinalMLP" else FO.dualmlp_logit
    return lambda s, X: torch.sigmoid(fn(specs, s, X, kw))


@pytest.mark.parametrize("case", MODEL_CASES)
def test_oracle_models_match_reference_trajectory(case):
    """test_oracle_golden.py's recipe: forward, loss and every gradient on batch 0, then three clip + Adam steps."""
    g = Golden("model_" + case)
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
    assert set(g["g"]) <= set(tr.state)
    for k, ref in g["g"].items():
        assert rel_err(tr.state[k].grad, ref) <= 2e-6, k
    losses = []
    for i in range(3):
        losses.append(float(tr.train_step(batches[i])))
        if i == 0:
            for k, ref in g["w1"].items():
                assert rel_err(tr.state[k], ref) <= 2e-6, k
    assert rel_err(torch.tensor(losses), g["out"]["step_losses"]) <= 2e-6
    for k, ref in g["w3"].items():
        assert rel_err(tr.state[k], ref) <= 5e-6, k


# ------------------------------------------------------------------ construction
def _digests(module):
    return [[k, str(v.dtype), list(v.shape), hashlib.sha256(v.detach().contiguous().numpy().tobytes()).hexdigest()]
            for k, v in module.state_dict().items()]


def _init_cases():
    with open(os.path.join(GOLDEN, "finalmlp_init.json")) as fd:
        return json.load(fd)


def test_mirrors_state_dict_match_reference_construction():
    """Keys, registration order, shapes and initial values (same RNG draws) of the reference's
    InteractionAggregation (w_xy's xavier draw included) and FeatureSelection, with and without context."""
    init = _init_cases()
    assert len(init["aggregation"]) == 4 and len(init["feature_selection"]) == 2
    for name, case in init["aggregation"].items():
        torch.manual_seed(case["seed"])
        assert _digests(layers.InteractionAggregation(*case["args"])) == case["state_dict"], name
    for name, case in init["feature_selection"].items():
        fm = FeatureMap.from_specs(case["specs"], labels=case["labels"])
        torch.manual_seed(case["seed"])
        assert _digests(layers.FeatureSelection(fm, *case["args"])) == case["state_dict"], name


@pytest.mark.parametrize("case", MODEL_CASES)
def test_zoo_state_dict_matches_reference_construction(case):
    """The whole model after construction, ending in reset_parameters (which re-draws the Linears, not w_xy)."""
    c = _init_cases()["models"][case]
    torch.manual_seed(c["seed"])
    fm = FeatureMap.from_specs(c["specs"], labels=c["labels"], embedding_dim=c["kwargs"]["embedding_dim"])
    model = getattr(zoo, c["model"])(fm, gpu=-1, **c["kwargs"])
    assert _digests(model) == c["state_dict"]


def _tiny_fm(n=3):
    return FeatureMap.from_specs([("C%d" % i, {"type": "categorical", "source": "", "padding_idx": 0,
                                               "vocab_size": 9}) for i in range(n)], embedding_dim=4)


def test_unknown_keywords_are_ignored_and_use_fs_false_builds_no_gates():
    fm = _tiny_fm()
    m = zoo.FinalMLP(fm, gpu=-1, embedding_dim=4, mlp1_hidden_units=[8], mlp2_hidden_units=[8], use_fs=False,
                     batch_size=128, epochs=1, shuffle=True)
    assert not hasattr(m, "fs_module") and list(dict(m.named_children())) == ["output_activation", "embedding_layer",
                                                                                "mlp1", "mlp2", "fusion_module"]
    zoo.DualMLP(fm, gpu=-1, embedding_dim=4, num_heads=3, fs_hidden_units=[4])


@pytest.mark.parametrize("units", [dict(mlp1_hidden_units=[]), dict(mlp2_hidden_units=[])])
def test_empty_tower_is_refused_at_construction(units):
    with pytest.raises(ValueError, match="mlp1_hidden_units and mlp2_hidden_units"):
        zoo.FinalMLP(_tiny_fm(), gpu=-1, embedding_dim=4, **units)


def test_aggregation_refuses_other_output_dims_and_keeps_the_divisibility_assertion():
    with pytest.raises(NotImplementedError, match="output_dim 1"):
        layers.InteractionAggregation(8, 8, output_dim=2)
    with pytest.raises(AssertionError, match="divisible by num_heads"):
        layers.InteractionAggregation(8, 6, num_heads=4)


@pytest.mark.parametrize("name", ["FinalMLP", "DualMLP"])
def test_sharded_front_routing_and_lazy_tables_refusal(name):
    cls = getattr(zoo, name)
    assert cls._routes_sharded_front is True
    assert not getattr(cls, "_replays_lazy_tables", False)
    model = cls(_tiny_fm(), gpu=-1, embedding_dim=4, mlp1_hidden_units=[8], mlp2_hidden_units=[8])
    with pytest.raises(NotImplementedError, match="lazy"):
        model.use_fused_optimizer(lazy_tables=True)


def test_sharding_with_context_features_is_refused_before_any_table_is_touched():
    model = zoo.FinalMLP(_tiny_fm(), gpu=-1, embedding_dim=4, mlp1_hidden_units=[8], mlp2_hidden_units=[8],
                         fs1_context=["C0"])
    before = {k: v.clone() for k, v in model.state_dict().items()}
    with pytest.raises(NotImplementedError, match="fs1_context"):
        model.enable_sharding(group=None, batch_local=4, matrix_width=4)
    assert getattr(model, "_sharded_front", None) is None
    after = model.state_dict()
    assert all(torch.equal(before[k], after[k]) and before[k].shape == after[k].shape for k in before)


# ------------------------------------------------------------------ C-ABI range checks (no CUDA call is reached)
def test_kernel_range_is_checked_before_any_cuda_call():
    import __graft_entry__
    __graft_entry__.build()
    L = _lib.load()
    p = ctypes.c_void_p(4096)
    bf16 = _lib.B2_BF16

    def err():
        return L.b2_last_error()
    assert L.b2_fs_gate_fwd(p, p, p, 0, 0, 8, 0, p, p, None, None, 0, 0, None) == -1 and b"d = 0" in err()
    assert L.b2_fs_gate_fwd(None, p, p, 0, 0, 8, 16, p, p, None, None, 0, 0, None) == -1 and b"NULL" in err()
    assert L.b2_fs_gate_fwd(p, p, p, 0, 1, 8, 16, p, p, p, None, bf16, 16, None) == -1 and b"both" in err()
    assert L.b2_fs_gate_fwd(p, p, p, 0, 0, -1, 16, p, p, None, None, 0, 0, None) == -1 and b"negative" in err()
    assert L.b2_fs_gate_fwd(p, p, p, 0, 0, 1 << 26, 64, p, p, None, None, 0, 0, None) == -1 and b"2^31" in err()
    assert L.b2_fs_gate_fwd(p, p, p, 0, 0, 8, 16, p, p, p, p, bf16, 8, None) == -1 and b"ld_aux" in err()
    assert L.b2_fs_gate_fwd(p, p, p, 0, 0, 8, 16, p, p, p, p, 7, 16, None) == -1 and b"aux_dtype" in err()
    assert L.b2_fs_gate_bwd(p, p, p, 0, 0, p, p, 8, 16, p, p, None, None) == -1 and b"NULL" in err()
    assert L.b2_fs_gate_bwd(p, p, p, 1, 1, p, p, 8, -2, p, p, p, None) == -1 and b"d = -2" in err()
    assert L.b2_agg_pack(p, p, p, 10, 6, 4, p, p, None) == -1 and b"num_heads" in err()
    assert L.b2_agg_pack(p, p, p, 8, 8, 0, p, p, None) == -1 and b"num_heads" in err()
    assert L.b2_agg_pack(p, p, p, 0, 8, 1, p, p, None) == -1 and b"widths" in err()
    assert L.b2_agg_pack(p, p, None, 8, 8, 1, p, p, None) == -1 and b"NULL" in err()
    assert L.b2_agg_fwd(p, p, p, p, -1, 8, p, None) == -1 and b"negative" in err()
    assert L.b2_agg_fwd(p, p, None, p, 8, 8, p, None) == -1 and b"NULL" in err()
    assert L.b2_agg_fwd(p, p, p, p, 1 << 28, 8, p, None) == -1 and b"2^31" in err()
    assert L.b2_agg_bwd(p, p, p, 8, 8, p, p, p, _lib.B2_F32, 8, p, p, p, None) == -1 \
        and b"ld_aux" in err()                                             # ys's row is B2_AGG_COLS(8) = 12 wide
    assert L.b2_agg_bwd(p, p, p, 8, 8, p, p, None, 0, 0, p, None, p, None) == -1 and b"NULL" in err()
    assert L.b2_agg_unpack(p, 9, 6, 2, p, p, None) == -1 and b"num_heads" in err()
    assert L.b2_agg_unpack(p, 8, 6, 2, None, p, None) == -1 and b"NULL" in err()
    assert L.b2_fs_gate_fwd(p, p, p, 0, 0, 0, 16, p, p, None, None, 0, 0, None) == 0     # empty batch: no launch
    assert L.b2_fs_gate_bwd(p, p, p, 0, 0, p, p, 0, 7, p, p, p, None) == 0
    assert L.b2_agg_fwd(p, p, p, p, 0, 8, p, None) == 0
    assert L.b2_agg_bwd(p, p, p, 0, 7, p, p, None, 0, 0, p, p, p, None) == 0


# ------------------------------------------------------------------ launch sequence (no GPU: _lib.call recorded)
@pytest.fixture
def recorder(monkeypatch):
    calls = []

    def fake_call(name, *a):
        info = None
        if name == "b2_gemm_tc_ex":
            d = ctypes.cast(a[0], ctypes.POINTER(_lib.b2_gemm_desc)).contents
            info = dict(M=d.M, N=d.N, K=d.K, a_mn=d.a_mn_major, b_mn=d.b_mn_major, bias=bool(d.bias),
                        add=bool(d.add), bf16=d.elem_dtype == _lib.B2_BF16, inline=bool(d.flags & _lib.B2_GEMM_X3_INLINE))
        elif name == "b2_gemm_f32":
            info = dict(M=a[8], N=a[9], K=a[10], bias=bool(a[11].value))
        elif name == "b2_fs_gate_fwd":
            info = dict(rows=(a[3], a[4]), aux=bool(a[9].value) and bool(a[10].value), dtype=a[11], ld=a[12])
        elif name == "b2_agg_bwd":
            info = dict(aux=bool(a[7].value), dtype=a[8], ld=a[9])
        calls.append((name, info))
        return 0

    monkeypatch.setattr(_lib, "call", fake_call)
    monkeypatch.setattr(F2, "_stream", lambda: None)
    monkeypatch.setattr(F2, "_require_cuda", lambda *t: None)
    yield calls
    F2.set_matmul_precision("fp32")
    F2.set_x3_inline(True)


AUX = ("b2_to_bf16", "b2_split_tf32")


@pytest.mark.parametrize("mode", ["tf32x3", "tf32", "bf16"])
def test_gates_without_context_run_their_mlps_on_one_row(recorder, mode):
    """FinalMLP_default's gates (fs [1024, 512], d 624) at B 2048: every gate-MLP GEMM has M = 1, and the gating
    products are one launch forward and one backward.  In bf16 the gate kernel writes both towers' operand copies."""
    F2.set_matmul_precision(mode)
    torch.manual_seed(5)
    fm = FeatureMap.from_specs([("C%d" % i, {"type": "categorical", "source": "", "padding_idx": 0, "vocab_size": 9})
                                for i in range(39)], embedding_dim=16)
    fs = layers.FeatureSelection(fm, 624, 16, [1024, 512])
    emb = torch.randn(2048, 624, requires_grad=True)
    f1, f2 = fs({}, emb)
    fwd = list(recorder)
    assert [n for n, _ in fwd].count("b2_fs_gate_fwd") == 1 and fwd[-1][0] == "b2_fs_gate_fwd"
    info = fwd[-1][1]
    assert info["rows"] == (0, 0) and info["aux"] == (mode == "bf16")
    if mode == "bf16":
        assert info["dtype"] == _lib.B2_BF16 and info["ld"] == 624
    del recorder[:]
    (f1.sum() + 2 * f2.sum()).backward()
    bwd = list(recorder)
    assert bwd[0][0] == "b2_fs_gate_bwd" and [n for n, _ in bwd].count("b2_fs_gate_bwd") == 1
    gemms = [i for n, i in fwd + bwd if n == "b2_gemm_tc_ex"]
    assert len(gemms) == 2 * 9                  # per gate: 3 layers forward, 3 dgrads (down to fs<s>_ctx_bias), 3 wgrads
    # the forward and dgrad GEMMs have the one row as M; a wgrad contracts over it (K = 1)
    assert all(g["M"] == 1 or (g["a_mn"] and g["b_mn"] and g["K"] == 1) for g in gemms), gemms
    assert not [n for n, _ in fwd + bwd if n == "b2_gemm_f32"]
    assert fs.fs1_ctx_bias.grad is not None and fs.fs2_ctx_bias.grad.shape == (1, 16)


def test_gates_with_context_run_per_row(recorder):
    F2.set_matmul_precision("tf32x3")
    fm = _tiny_fm(4)
    fs = layers.FeatureSelection(fm, 16, 4, [16], ["C0"], ["C1", "C2"])
    X = {"C%d" % i: torch.randint(0, 9, (64,)).double() for i in range(4)}
    fs(X, torch.randn(64, 16))
    gate = [i for n, i in recorder if n == "b2_fs_gate_fwd"]
    assert len(gate) == 1 and gate[0]["rows"] == (1, 1)
    assert all(i["M"] == 64 for n, i in recorder if n == "b2_gemm_tc_ex")


FWD = ["b2_agg_pack", "b2_gemm_tc_ex", "b2_agg_fwd"]
BWD = ["b2_agg_bwd", "b2_gemm_tc_ex", "b2_gemm_tc_ex", "b2_agg_unpack"]


def run_agg(mode, B, dx, dy, heads):
    F2.set_matmul_precision(mode)
    torch.manual_seed(3)
    agg = layers.InteractionAggregation(dx, dy, num_heads=heads)
    x, y = torch.randn(B, dx, requires_grad=True), torch.randn(B, dy, requires_grad=True)
    out = agg(x, y)
    assert out.shape == (B, 1) and type(out.grad_fn).__name__ == "_InteractionAggregationBackward"
    out.backward(torch.randn_like(out))
    for p in agg.parameters():
        assert p.grad is not None and p.grad.shape == p.shape
    assert x.grad is not None and y.grad is not None


@pytest.mark.parametrize("heads", [1, 2, 4])
@pytest.mark.parametrize("mode", ["tf32x3", "tf32", "bf16"])
def test_aggregation_is_three_launches_forward_and_four_backward(recorder, mode, heads):
    """FinalMLP_default's fusion (dx 512, dy 256) at B 4096: pack, Q = x W_aug^T + [w_y, 0], the row kernel;
    backward the row kernel, dx = ys W_aug, dW_aug = ys^T x and the unpack, whatever the head count.  bf16 adds only
    the bf16 copies of x and W_aug (b2_agg_bwd writes ys's)."""
    B, dx, dy = 4096, 512, 256
    n = dy + 4
    run_agg(mode, B, dx, dy, heads)
    assert [n_ for n_, _ in recorder if n_ not in AUX] == FWD + BWD
    assert [n_ for n_, _ in recorder].count("b2_to_bf16") == (2 if mode == "bf16" else 0)
    assert not [n_ for n_, _ in recorder if n_ == "b2_split_tf32"]
    q, gx, gw = [i for n_, i in recorder if n_ == "b2_gemm_tc_ex"]
    assert all(g["bf16"] == (mode == "bf16") and g["inline"] == (mode == "tf32x3") for g in (q, gx, gw))
    assert (q["M"], q["N"], q["K"], q["a_mn"], q["b_mn"], q["bias"]) == (B, n, dx, 0, 0, True)
    assert (gx["M"], gx["N"], gx["K"], gx["a_mn"], gx["b_mn"], gx["bias"]) == (B, dx, n, 0, 1, False)
    assert (gw["M"], gw["N"], gw["K"], gw["a_mn"], gw["b_mn"]) == (n, dx, B, 1, 1)
    bwd = [i for n_, i in recorder if n_ == "b2_agg_bwd"][0]
    assert bwd["aux"] == (mode == "bf16")
    if mode == "bf16":
        assert bwd["dtype"] == _lib.B2_BF16 and bwd["ld"] == 264           # n padded to 16 bytes


@pytest.mark.parametrize("mode,inline", [("tf32x3", True), ("tf32x3", False), ("tf32", True), ("bf16", True)])
def test_rebuilt_weight_operand_is_never_taken_from_the_weight_cache(recorder, monkeypatch, mode, inline):
    """W_aug is packed anew every step: its operand copy comes from make_aux in that step (a b2_to_bf16 or
    b2_split_tf32 launch after the pack), never from weight_aux's per-weight cache."""
    def no_cache(w):
        raise AssertionError("weight_aux consulted for a weight rebuilt every step")
    monkeypatch.setattr(F2, "weight_aux", no_cache)
    F2.set_x3_inline(inline)
    run_agg(mode, 256, 64, 32, 2)
    names = [n for n, _ in recorder]
    copy = {"bf16": "b2_to_bf16"}.get(mode, "b2_split_tf32" if not inline else None)
    assert names.count(copy) == 2 if copy else not [n for n in names if n in AUX]


@pytest.mark.parametrize("mode,dx,dy,heads", [("fp32", 512, 256, 2), ("tf32x3", 26, 14, 2), ("bf16", 20, 8, 1),
                                              ("tf32", 30, 18, 3)])
def test_simt_gemm_where_the_tensor_cores_cannot_go(recorder, mode, dx, dy, heads):
    """fp32 mode, dx % 4 != 0, or W_aug under 16 rows (dy 8): the SIMT GEMM, with the same row kernels."""
    B = 37
    run_agg(mode, B, dx, dy, heads)
    assert [n_ for n_, _ in recorder] == [n_.replace("gemm_tc_ex", "gemm_f32") for n_ in FWD + BWD]
    q, gx, gw = [i for n_, i in recorder if n_ == "b2_gemm_f32"]
    n = (dy + 4) // 4 * 4
    assert (q["M"], q["N"], q["K"], q["bias"]) == (B, n, dx, True)
    assert (gx["M"], gx["N"], gx["K"]) == (B, dx, n) and (gw["M"], gw["N"], gw["K"]) == (n, dx, B)
    assert not [i for n_, i in recorder if n_ == "b2_agg_bwd"][0]["aux"]


# ------------------------------------------------------------------ register use
def test_new_kernels_do_not_spill(tmp_path):
    nvcc = "/usr/local/cuda/bin/nvcc"
    from fuxictr_b200 import build
    nvcc = os.environ.get("NVCC") or (nvcc if os.path.exists(nvcc) else "nvcc")
    r = subprocess.run([nvcc] + build.NVCC_FLAGS + ["-Xptxas", "-v", "-I", build.INCLUDE, "-c",
                        os.path.join(build.CSRC, "finalmlp.cu"), "-o", str(tmp_path / "finalmlp.o")],
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    log = r.stdout + r.stderr
    kernels = [line for line in log.splitlines() if "Compiling entry function" in line]
    assert len(kernels) == 10, log
    assert all("fs_gate_" in k or "agg_" in k for k in kernels)
    spills = [line for line in log.splitlines() if "spill" in line]
    assert len(spills) == 10 and all("0 bytes spill stores, 0 bytes spill loads" in s for s in spills), log

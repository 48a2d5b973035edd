"""MaskNet without a GPU: the float64 oracle against the reference's goldens (block and the three model trajectories),
the mirror's and zoo.MaskNet's construction against the reference's, the refusals (lazy tables, activations, widths,
an empty SerialMaskNet), the C-ABI's range checks, the launch sequence of a block per matmul mode, and the new kernels'
register use."""
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
import masknet_oracle as MO  # noqa: E402
from fuxictr_b200 import _lib, functional as F2, layers, zoo  # noqa: E402
from fuxictr_b200.schema import FeatureMap  # noqa: E402


# ------------------------------------------------------------------ oracle vs the reference's goldens
@pytest.mark.parametrize("n", [20, 13])
def test_oracle_block_matches_reference_golden(n):
    g = Golden("next_MaskBlock")
    act = g.meta["widths"][str(n)]
    st = {k: v.clone().double().requires_grad_(True) for k, v in g["w_n%d" % n].items()}
    emb = g["in"]["emb_n%d" % n].clone().double().requires_grad_(True)
    hid = g["in"]["hid_n%d" % n].clone().double().requires_grad_(True)
    out = MO.mask_block(st, "", emb, hid, act, True)
    assert close(out, g["out"]["y_n%d" % n], 2e-6), rel_err(out, g["out"]["y_n%d" % n])
    (out * g["in"]["gout_n%d" % n].double()).sum().backward()
    assert close(emb.grad, g["gin"]["emb_n%d" % n], 2e-6), rel_err(emb.grad, g["gin"]["emb_n%d" % n])
    assert close(hid.grad, g["gin"]["hid_n%d" % n], 2e-6), rel_err(hid.grad, g["gin"]["hid_n%d" % n])
    want = g["g_n%d" % n]
    assert set(want) == set(st)
    for k, ref in want.items():
        scale = float(ref.abs().max())
        assert close(st[k].grad, ref, 2e-6, atol=2e-6 * scale), (k, rel_err(st[k].grad, ref))


@pytest.mark.parametrize("case", ["serial", "parallel", "noln"])
def test_oracle_models_match_reference_trajectory(case):
    g = Golden("model_MaskNet_" + case)
    fm = FeatureMap.from_specs(g.meta["specs"], labels=g.meta["labels"])
    B = g.meta["batch"]
    mat = g["in"]["matrix"]
    batches = [fm.batch_dict(mat[i * B:(i + 1) * B]) for i in range(3)]
    specs, kw = g.specs(), g.meta["kwargs"]
    tr = O.OracleTrainer(dict(g["w"]), lambda s, X: torch.sigmoid(MO.masknet_logit(specs, s, X, kw)), specs,
                         g.meta["labels"])
    y_pred, y = tr.forward(batches[0])
    assert rel_err(y_pred, g["out"]["y_pred"]) <= 1e-6
    loss = O.bce_mean(y_pred, y)
    loss.backward()
    for k, ref in g["g"].items():
        assert rel_err(tr.state[k].grad, ref) <= 5e-6, k
    losses = [float(tr.train_step(batches[i])) for i in range(3)]
    assert rel_err(torch.tensor(losses), g["out"]["step_losses"]) <= 2e-6
    for k, ref in g["w3"].items():
        assert rel_err(tr.state[k], ref) <= 5e-6, k


# ------------------------------------------------------------------ construction
def _digests(module):
    return [[k, str(v.dtype), list(v.shape), hashlib.sha256(v.detach().contiguous().numpy().tobytes()).hexdigest()]
            for k, v in module.state_dict().items()]


def _init_cases():
    with open(os.path.join(GOLDEN, "masknet_init.json")) as fd:
        return json.load(fd)


def test_mirror_state_dict_matches_reference_construction():
    for name, case in _init_cases()["blocks"].items():
        torch.manual_seed(case["seed"])
        assert _digests(layers.MaskBlock(*case["args"])) == case["state_dict"], name


@pytest.mark.parametrize("name", ["serial", "parallel_dropout", "parallel_head"])
def test_zoo_state_dict_matches_reference_construction(name):
    """Registration order embedding_layer, mask_net, emb_norm; LayerNorms keep 1 / 0; float reduction_ratio."""
    case = _init_cases()["models"][name]
    torch.manual_seed(case["seed"])
    fm = FeatureMap.from_specs(case["specs"], labels=case["labels"], embedding_dim=case["kwargs"]["embedding_dim"])
    model = zoo.MaskNet(fm, gpu=-1, some_unknown_keyword=3, **case["kwargs"])
    assert _digests(model) == case["state_dict"]


def test_embedding_layernorm_parameters_lie_at_one_stride():
    fm = FeatureMap.from_specs([("C%d" % i, {"type": "categorical", "source": "", "padding_idx": 0, "vocab_size": 9})
                                for i in range(5)], embedding_dim=6)
    model = zoo.MaskNet(fm, gpu=-1, embedding_dim=6, dnn_hidden_units=[8])
    ws, bs = [m.weight for m in model.emb_norm], [m.bias for m in model.emb_norm]
    gamma, beta, pstride = F2.field_param_layout(ws, bs)
    assert pstride == 16 and beta.data_ptr() - gamma.data_ptr() == 8 * 4
    assert F2.field_param_layout([torch.ones(6) for _ in range(3)], [torch.zeros(6) for _ in range(3)]) is None


# ------------------------------------------------------------------ refusals
def _fm(nf=3, dim=4):
    return FeatureMap.from_specs([("C%d" % i, {"type": "categorical", "source": "", "padding_idx": 0,
                                               "vocab_size": 9}) for i in range(nf)], embedding_dim=dim)


def test_empty_serial_dnn_is_refused_and_parallel_head_is_built():
    with pytest.raises(ValueError, match="dnn_hidden_units"):
        zoo.MaskNet(_fm(), gpu=-1, embedding_dim=4, dnn_hidden_units=[])
    model = zoo.MaskNet(_fm(), gpu=-1, embedding_dim=4, dnn_hidden_units=[], model_type="ParallelMaskNet",
                        parallel_num_blocks=2, parallel_block_dim=8)
    assert [type(m).__name__ for m in model.mask_net.dnn.mlp] == ["Linear", "Sigmoid"]
    with pytest.raises(ValueError, match="model_type"):
        zoo.MaskNet(_fm(), gpu=-1, embedding_dim=4, model_type="Serial")


@pytest.mark.parametrize("act", ["tanh", "PReLU", "LeakyReLU"])
def test_unsupported_activation_is_refused_at_construction(act):
    with pytest.raises((NotImplementedError, AssertionError)) as e:
        zoo.MaskNet(_fm(), gpu=-1, embedding_dim=4, dnn_hidden_units=[8], dnn_hidden_activations=act)
    if e.type is NotImplementedError:
        assert "MaskBlock" in str(e.value)
    with pytest.raises(NotImplementedError, match="Tanh"):
        layers.MaskBlock(8, 8, 8, "tanh")


def test_widths_are_checked_before_any_cuda_call():
    lim = _lib.B2_MASKNET_MAX_WIDTH
    layers.MaskBlock(4, 4, lim)
    with pytest.raises(ValueError, match="output_dim"):
        layers.MaskBlock(4, 4, lim + 1)
    with pytest.raises(ValueError, match="output_dim"):
        layers.MaskBlock(4, 4, 0)
    with pytest.raises(ValueError, match="embedding_dim"):
        zoo.MaskNet(_fm(dim=lim + 1), gpu=-1, embedding_dim=lim + 1, dnn_hidden_units=[8])
    zoo.MaskNet(_fm(dim=6), gpu=-1, embedding_dim=6, dnn_hidden_units=[lim], emb_layernorm=False)


def test_sharded_front_routing_and_lazy_tables_refusal():
    assert zoo.MaskNet._routes_sharded_front is True
    assert not getattr(zoo.MaskNet, "_replays_lazy_tables", False)
    model = zoo.MaskNet(_fm(), gpu=-1, embedding_dim=4, dnn_hidden_units=[8])
    with pytest.raises(NotImplementedError, match="lazy"):
        model.use_fused_optimizer(lazy_tables=True)


# ------------------------------------------------------------------ C-ABI range checks (no CUDA call is reached)
def test_kernel_range_is_checked_before_any_cuda_call():
    import __graft_entry__
    __graft_entry__.build()
    L = _lib.load()
    p = ctypes.c_void_p(4096)
    lim = _lib.B2_MASKNET_MAX_WIDTH
    err = lambda: L.b2_last_error()  # noqa: E731
    assert L.b2_field_ln_fwd(p, 8, 3, lim + 1, p, p, 2 * lim + 8, 1e-5, p, p, p, None) == -1 and b"width" in err()
    assert L.b2_field_ln_fwd(p, 8, 3, 0, p, p, 8, 1e-5, p, p, p, None) == -1 and b"width" in err()
    assert L.b2_field_ln_fwd(p, 8, 3, 8, p, p, 4, 1e-5, p, p, p, None) == -1 and b"stride" in err()
    assert L.b2_field_ln_fwd(None, 8, 3, 8, p, p, 16, 1e-5, p, p, p, None) == -1 and b"NULL" in err()
    assert L.b2_field_ln_fwd(p, -1, 3, 8, p, p, 16, 1e-5, p, p, p, None) == -1 and b"negative" in err()
    assert L.b2_field_ln_fwd(p, 1 << 28, 3, 8, p, p, 16, 1e-5, p, p, p, None) == -1 and b"2^31" in err()
    assert L.b2_field_ln_bwd(p, p, p, p, 8, 3, 8, p, 16, p, 0, None, p, None) == -1 and b"NULL" in err()
    assert L.b2_mask_row_fwd(p, 8, lim + 1, p, p, 1e-5, 1, None, 0, 0, 0.0, p, lim + 1, None, 0, 0, p, p,
                             None) == -1 and b"width" in err()
    assert L.b2_mask_row_fwd(p, 8, 16, p, p, 1e-5, 5, None, 0, 0, 0.0, p, 16, None, 0, 0, p, p, None) == -1 \
        and b"act" in err()
    assert L.b2_mask_row_fwd(p, 8, 16, p, None, 1e-5, 1, None, 0, 0, 0.0, p, 16, None, 0, 0, p, p, None) == -1 \
        and b"both or neither" in err()
    assert L.b2_mask_row_fwd(p, 8, 16, p, p, 1e-5, 1, None, 0, 0, 0.0, p, 8, None, 0, 0, p, p, None) == -1 \
        and b"ld_out" in err()
    assert L.b2_mask_row_fwd(p, 8, 16, p, p, 1e-5, 1, None, 0, 0, 0.0, p, 16, p, 7, 16, p, p, None) == -1 \
        and b"aux_dtype" in err()
    assert L.b2_mask_row_bwd(p, p, p, p, p, 1, None, 0, 0, 0.0, p, 8, 8, 16, p, None, 0, 0, p, p, None) == -1 \
        and b"ld_g" in err()
    assert L.b2_mask_row_bwd(p, p, p, p, p, 1, None, 0, 0, 0.0, p, 16, 8, 16, p, None, 0, 0, None, p, None) == -1
    assert L.b2_mask_mul(p, None, 8, p, 0, None) == -1 and L.b2_mask_mul(p, p, -1, p, 0, None) == -1
    assert L.b2_mask_row_fwd(p, 0, 16, p, p, 1e-5, 1, None, 0, 0, 0.0, p, 16, None, 0, 0, p, p, None) == 0
    assert L.b2_field_ln_bwd(p, p, p, p, 0, 3, 8, p, 16, p, 0, p, p, None) == 0
    assert L.b2_mask_mul(p, p, 0, p, 0, None) == 0


# ------------------------------------------------------------------ launch sequence (no GPU: _lib.call recorded)
@pytest.fixture
def recorder(monkeypatch):
    calls = []

    def fake_call(name, *a):
        info = None
        if name == "b2_gemm_tc_ex":
            d = ctypes.cast(a[0], ctypes.POINTER(_lib.b2_gemm_desc)).contents
            info = dict(M=d.M, N=d.N, K=d.K, a_mn=d.a_mn_major, b_mn=d.b_mn_major, bias=bool(d.bias), mul=bool(d.mul),
                        c_pre=bool(d.c_pre), colsum=bool(d.colsum), ybwd=bool(d.ybwd), acc=d.beta_accumulate,
                        small=bool(d.c_small), act=d.act)
        elif name == "b2_gemm_f32":
            info = dict(M=a[8], N=a[9], K=a[10], acc=a[15])
        calls.append((name, info))
        return 0

    monkeypatch.setattr(_lib, "call", fake_call)
    monkeypatch.setattr(F2, "_stream", lambda: None)
    monkeypatch.setattr(F2, "_require_cuda", lambda *t: None)
    yield calls
    F2.set_matmul_precision("fp32")
    F2.set_x3_inline(True)


FWD = ["b2_gemm_tc_ex", "b2_gemm_tc_ex", "b2_gemm_tc_ex", "b2_mask_row_fwd"]
BWD = ["b2_mask_row_bwd", "b2_gemm_tc_ex", "b2_gemm_tc_ex", "b2_mask_mul", "b2_gemm_tc_ex", "b2_gemm_tc_ex",
       "b2_gemm_tc_ex", "b2_gemm_tc_ex"]


def run_block(mode, B, d, hd, n, inline=True, ln=True):
    F2.set_x3_inline(inline)
    F2.set_matmul_precision(mode)
    torch.manual_seed(3)
    blk = layers.MaskBlock(d, hd, n, "relu", 1, 0, ln)
    emb = torch.randn(B, d, requires_grad=True)
    hid = torch.randn(B, hd, requires_grad=True)
    out = blk(emb, hid)
    assert type(out.grad_fn).__name__ == "_MaskBlocksBackward"
    out.backward(torch.randn_like(out))
    for p in blk.parameters():
        assert p.grad is not None and p.grad.shape == p.shape
    return emb, hid


@pytest.mark.parametrize("mode", ["tf32x3", "tf32", "bf16"])
def test_block_is_four_launches_forward_and_eight_backward(recorder, mode):
    """Forward: the mask MLP's two GEMMs (bias + ReLU; bias + mul = v_in keeping V_mask), the hidden GEMM, the row
    kernel.  Backward: the row kernel, dV_mask = v_in * (dz W3) keeping du (+ b2's sum), dW3, dv_in = du * V_mask,
    dh (ReLU' of h, b1's sum), dW2, V_emb's gradient (first writer: no accumulate), dW1.  bf16 adds only the bf16 copies
    of V_emb and the three weights: every other operand copy comes from an epilogue or the row kernel."""
    B, d, hd, n = 4096, 624, 624, 64
    emb, hid = run_block(mode, B, d, hd, n)
    assert emb.grad is not None and hid.grad is not None
    names = [c for c, _ in recorder if c not in ("b2_to_bf16", "b2_split_tf32")]
    assert names == FWD + BWD
    g = [i for c, i in recorder if c == "b2_gemm_tc_ex"]
    g1, g2, g3 = g[:3]
    assert (g1["M"], g1["N"], g1["K"], g1["bias"], g1["act"]) == (B, hd, d, True, _lib.B2_ACT_RELU)
    assert (g2["N"], g2["K"], g2["bias"], g2["mul"], g2["c_pre"]) == (hd, hd, True, True, True)
    assert (g3["N"], g3["K"], g3["bias"], g3["mul"]) == (n, hd, False, False)
    d3, w3, d2, w2, d1, w1 = g[3:]
    assert (d3["N"], d3["K"], d3["b_mn"], d3["mul"], d3["c_pre"], d3["colsum"]) == (hd, n, 1, True, True, True)
    assert (w3["M"], w3["N"], w3["K"], w3["a_mn"], w3["b_mn"]) == (n, hd, B, 1, 1)
    assert (d2["N"], d2["ybwd"], d2["colsum"]) == (hd, True, True)
    assert (d1["N"], d1["K"], d1["acc"]) == (d, hd, 0)
    assert (w1["M"], w1["N"], w1["K"]) == (hd, d, B)
    assert [c for c, _ in recorder].count("b2_to_bf16") == (1 + 3 if mode == "bf16" else 0)


def test_blocks_share_one_embedding_gradient_buffer(recorder):
    """SerialMaskNet, 3 blocks: the last block's backward runs first and writes V_emb's buffer, the two before it
    and the embedding LayerNorm's backward add into it."""
    F2.set_matmul_precision("tf32")
    torch.manual_seed(5)
    fm = _fm(nf=8, dim=12)
    model = zoo.MaskNet(fm, gpu=-1, embedding_dim=12, dnn_hidden_units=[32, 32, 16])
    emb = torch.randn(40, 96, requires_grad=True)
    x, sink = F2.shared_grad(emb)
    ws, bs = [m.weight for m in model.emb_norm], [m.bias for m in model.emb_norm]
    v = model.mask_net.blocks_out(x, F2.field_layernorm(x, sink, ws, bs), sink)
    v.sum().backward()
    assert emb.grad is not None and emb.grad.shape == emb.shape
    dgrad1 = [i for c, i in recorder if c == "b2_gemm_tc_ex" and i["N"] == 96 and i["b_mn"] and not i["a_mn"]
              and not i["mul"] and not i["ybwd"]]
    assert [i["acc"] for i in dgrad1] == [0, 1, 1]
    names = [c for c, _ in recorder]
    assert names.count("b2_field_ln_fwd") == 1 and names.count("b2_field_ln_bwd") == 1
    assert names.index("b2_field_ln_bwd") > max(i for i, c in enumerate(names) if c == "b2_mask_row_bwd")


def test_x3_aux_layout_adds_only_the_input_splits(recorder):
    run_block("tf32x3", 512, 624, 624, 64, inline=False)
    names = [c for c, _ in recorder]
    assert names.count("b2_split_tf32") == 1 + 3          # V_emb and the three weights; the rest come with theirs
    g = [i for c, i in recorder if c == "b2_gemm_tc_ex"]
    assert len(g) == 9


@pytest.mark.parametrize("mode,shape", [("fp32", (624, 624, 64)), ("tf32x3", (13, 13, 7)), ("tf32", (30, 30, 7)),
                                        ("bf16", (12, 12, 12))])
def test_simt_gemm_where_the_tensor_cores_cannot_go(recorder, mode, shape):
    """fp32 mode or shapes the tensor cores cannot take: the SIMT GEMM; the mul epilogue becomes a b2_mask_mul
    forward and a b2_prep_operand backward (which also sums b2's gradient)."""
    d, hd, n = shape
    run_block(mode, 37, d, hd, n)
    names = [c for c, _ in recorder if c not in ("b2_to_bf16", "b2_split_tf32")]
    assert "b2_gemm_tc_ex" not in names
    assert names[:5] == ["b2_gemm_f32", "b2_gemm_f32", "b2_mask_mul", "b2_gemm_f32", "b2_mask_row_fwd"]
    assert names[5:] == ["b2_mask_row_bwd", "b2_gemm_f32", "b2_prep_operand", "b2_gemm_f32", "b2_mask_mul",
                         "b2_gemm_f32", "b2_prep_operand", "b2_gemm_f32", "b2_gemm_f32", "b2_gemm_f32"]


# ------------------------------------------------------------------ register use
def test_new_kernels_do_not_spill(tmp_path):
    nvcc = "/usr/local/cuda/bin/nvcc"
    from fuxictr_b200 import build
    nvcc = os.environ.get("NVCC") or (nvcc if os.path.exists(nvcc) else "nvcc")
    r = subprocess.run([nvcc] + build.NVCC_FLAGS + ["-Xptxas", "-v", "-I", build.INCLUDE, "-c",
                        os.path.join(build.CSRC, "masknet.cu"), "-o", str(tmp_path / "masknet.o")],
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    log = r.stdout + r.stderr
    kernels = [line for line in log.splitlines() if "Compiling entry function" in line]
    assert len(kernels) == 10, log
    assert all("mn_" in k for k in kernels)
    spills = [line for line in log.splitlines() if "spill" in line]
    assert len(spills) == 10 and all("0 bytes spill stores, 0 bytes spill loads" in s for s in spills), log

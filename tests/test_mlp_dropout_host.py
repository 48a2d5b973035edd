"""Dropout in the fused MLP chain, host side: the mask function restated in numpy (Philox4x32-10 and keep()), the
launches a dropout chain issues (with `_lib.call` recorded, as in test_launch_sequence_dryrun.py), which stacks
MLP_Block sends to the chain, and the GEMM plans of descriptors that carry a mask."""
import ctypes
import itertools

import numpy as np
import pytest
import torch

from fuxictr_b200 import _lib, functional as F2, layers
from fuxictr_b200._lib import B2_ACT_NONE, B2_ACT_RELU

M0, M1, W0, W1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57), 0x9E3779B9, 0xBB67AE85
MASK32 = np.uint64(0xFFFFFFFF)


def philox4x32_10(ctr, key):
    """Philox4x32-10 over arrays: ctr = 4 uint32 arrays (broadcastable), key = 2 uint32 scalars; returns 4 arrays."""
    c = [np.asarray(v, dtype=np.uint64) & MASK32 for v in ctr]
    k0, k1 = int(key[0]) & 0xFFFFFFFF, int(key[1]) & 0xFFFFFFFF
    for _ in range(10):
        p0, p1 = M0 * c[0], M1 * c[2]
        hi0, lo0, hi1, lo1 = p0 >> np.uint64(32), p0 & MASK32, p1 >> np.uint64(32), p1 & MASK32
        c = [hi1 ^ c[1] ^ np.uint64(k0), lo1, hi0 ^ c[3] ^ np.uint64(k1), lo0]
        k0, k1 = (k0 + W0) & 0xFFFFFFFF, (k1 + W1) & 0xFFFFFFFF
    return [v.astype(np.uint32) for v in c]


def keep_mask(seed, offset, M, N, p):
    """keep(seed, offset, m, n) of include/fuxictr_b200.h for every element of an (M, N) output (bool array)."""
    thresh, _ = F2.dropout_consts(p)
    seed, offset = int(seed) & (2 ** 64 - 1), int(offset) & (2 ** 64 - 1)
    i = np.arange(M * N, dtype=np.uint64)
    g = i >> np.uint64(2)
    r = philox4x32_10([g & MASK32, g >> np.uint64(32), np.uint64(offset & 0xFFFFFFFF), np.uint64(offset >> 32)],
                      [seed & 0xFFFFFFFF, seed >> 32])
    word = np.choose((i & np.uint64(3)).astype(np.int64), r)
    return (word < np.uint32(thresh)).reshape(M, N)


def test_philox_known_answers():
    """Random123's known-answer vectors for philox4x32-10; the first is also cuRAND's PHILOX4_32_10 host generator
    at seed 0 (its first four outputs), whose next four are counter {0, 0, 1, 0}."""
    def one(ctr, key):
        return [int(v) for v in philox4x32_10([np.uint64(c) for c in ctr], key)]
    assert one([0, 0, 0, 0], [0, 0]) == [0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8]
    assert one([0, 0, 1, 0], [0, 0]) == [0x844515e1, 0xf08d6eaa, 0x0f19c053, 0x83f875f0]
    assert one([0xffffffff] * 4, [0xffffffff, 0xffffffff]) == [0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd]
    assert one([0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344], [0xa4093822, 0x299f31d0]) == \
        [0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1]


def test_keep_function_layout():
    """One Philox call per group of 4 consecutive elements of the row-major (M, N) matrix (across row ends), the
    64-bit group index in counter words 0-1, the offset in words 2-3, the seed as the key."""
    seed, off, M, N, p = 0x0123456789ABCDEF, (7 << 32) + 3, 5, 7, 0.3
    mask = keep_mask(seed, off, M, N, p).reshape(-1)
    thresh, scale = F2.dropout_consts(p)
    for i in range(M * N):
        r = philox4x32_10([np.uint64(i // 4), np.uint64(0), np.uint64(3), np.uint64(7)],
                          [0x89ABCDEF, 0x01234567])
        assert mask[i] == (int(r[i % 4]) < thresh), i
    # different offsets (forwards, or layers of one forward) and seeds give unrelated masks
    a = keep_mask(seed, off, 64, 64, 0.5)
    assert 0.4 < (a == keep_mask(seed, off + 1, 64, 64, 0.5)).mean() < 0.6
    assert 0.4 < (a == keep_mask(seed + 1, off, 64, 64, 0.5)).mean() < 0.6
    assert scale == np.float32(1.0 / 0.7) and thresh == round(0.7 * 2 ** 32)


def test_dropout_constants():
    for p in (1e-9, 0.1, 0.2, 0.5, 0.999):
        thresh, scale = F2.dropout_consts(p)
        assert 0 < thresh <= 2 ** 32 - 1 and abs(thresh / 2 ** 32 - (1 - p)) <= 2 ** -32
        assert scale == float(np.float32(1 / (1 - p)))
    for p in (0.0, 1.0, -0.1, 1.5):
        with pytest.raises(ValueError):
            F2.dropout_consts(p)


# ------------------------------------------------------------------ launch sequence (nothing is computed)
@pytest.fixture
def recorder(monkeypatch):
    calls = []

    def fake_call(name, *a):
        info = None
        if name == "b2_gemm_tc_ex":
            d = ctypes.cast(a[0], ctypes.POINTER(_lib.b2_gemm_desc)).contents
            info = dict(M=d.M, N=d.N, K=d.K, a_mn=d.a_mn_major, b_mn=d.b_mn_major, act=d.act, ybwd=bool(d.ybwd),
                        act_bwd=d.act_bwd, colsum=bool(d.colsum), c_small=bool(d.c_small),
                        drop=bool(d.drop_rng), layer=d.drop_layer, thresh=d.drop_thresh, scale=d.drop_scale)
        elif name == "b2_head_bwd_ex":
            info = dict(prev_act=a[10], drop=bool(a[14].value), layer=a[15], thresh=a[16], scale=a[17])
        elif name == "b2_dropout_rng_take":
            info = dict(n_layers=a[2])
        calls.append((name, info))
        return 0

    monkeypatch.setattr(_lib, "call", fake_call)
    monkeypatch.setattr(F2, "_stream", lambda: None)
    monkeypatch.setattr(F2, "_require_cuda", lambda *t: None)
    yield calls
    F2.set_matmul_precision("fp32")


def c2_block(rate=0.2, **kw):
    torch.manual_seed(0)
    return layers.MLP_Block(624, hidden_units=[300, 300, 300], output_dim=1, dropout_rates=rate, **kw)


def run_block(mlp, mode="tf32x3"):
    F2.set_matmul_precision(mode)
    chain = mlp.chain_layers()
    assert chain is not None
    x = torch.randn(4096, 624, requires_grad=True)
    y = F2.mlp_chain(x, chain)
    assert type(y.grad_fn).__name__.startswith("_MLPChain")
    y.backward(torch.randn_like(y))


def test_c2_dropout_step_is_one_rng_take_then_the_eleven_launches(recorder):
    run_block(c2_block(0.2).train())
    names = [n for n, _ in recorder]
    assert names == ["b2_dropout_rng_take"] + ["b2_gemm_tc_ex"] * 3 + ["b2_head_fwd", "b2_head_bwd_ex"] + \
        ["b2_gemm_tc_ex"] * 6
    assert recorder[0][1] == dict(n_layers=3)
    thresh, scale = F2.dropout_consts(0.2)
    fwd = [i for n, i in recorder[1:4]]
    for layer, d in enumerate(fwd):        # each hidden layer's forward epilogue applies its own mask after ReLU
        assert d["drop"] and d["layer"] == layer and d["thresh"] == thresh and d["scale"] == np.float32(scale)
        assert d["act"] == B2_ACT_RELU and not d["ybwd"]
    head = recorder[5][1]                  # the head backward folds the last hidden layer's ReLU and mask
    assert head["drop"] and head["layer"] == 2 and head["prev_act"] == B2_ACT_RELU and head["thresh"] == thresh
    bwd = [i for _, i in recorder[6:]]     # (dgrad, wgrad) of layers 2, 1, 0
    assert [(d["M"], d["N"], d["K"], d["a_mn"], d["b_mn"]) for d in bwd] == [
        (4096, 300, 300, 0, 1), (300, 300, 4096, 1, 1),
        (4096, 300, 300, 0, 1), (300, 300, 4096, 1, 1),
        (4096, 624, 300, 0, 1), (300, 624, 4096, 1, 1)]
    for k, d in enumerate(bwd):
        if k in (0, 2):    # the dgrads of layers 2 and 1 fold layers 1 and 0: ReLU backward, mask, bias gradient
            assert d["drop"] and d["layer"] == (1 if k == 0 else 0) and d["ybwd"] and d["colsum"]
        else:              # the input gradient and the wgrads carry no mask
            assert not d["drop"] and not d["ybwd"]


@pytest.mark.parametrize("mode", ["tf32x3", "tf32", "bf16"])
def test_eval_mode_is_todays_sequence(recorder, mode):
    run_block(c2_block(0.0), mode)
    plain = list(recorder)
    del recorder[:]
    run_block(c2_block(0.2).eval(), mode)
    assert recorder == plain
    assert all(not i["drop"] for n, i in recorder if n == "b2_gemm_tc_ex")


def test_descriptor_without_dropout_is_unchanged(recorder):
    """A chain of 3-tuples and one of 4-tuples with p = 0 issue the same launches with the dropout fields zero."""
    mlp = c2_block(0.0)
    F2.set_matmul_precision("tf32x3")
    x = torch.randn(256, 624, requires_grad=True)
    chain = mlp.chain_layers()
    F2.mlp_chain(x, chain).sum().backward()
    three = list(recorder)
    del recorder[:]
    F2.mlp_chain(x, [c + (0.0,) for c in chain]).sum().backward()
    assert recorder == three
    assert all(i["layer"] == 0 and i["thresh"] == 0 and i["scale"] == 0.0 for n, i in three if n == "b2_gemm_tc_ex")


def test_top_dropout_and_odd_layers_take_the_explicit_pass(recorder):
    """A tower that ends on ReLU + Dropout (DCNv2's parallel DNN) applies the top mask in the explicit pass over dY.
    Layers the tensor-core kernel cannot take (widths 18 and 36 over K = 18) get their masks from b2_dropout_apply;
    the head backward folds the second one's, the explicit pass below the SIMT layer the first one's."""
    F2.set_matmul_precision("tf32x3")
    torch.manual_seed(0)
    tower = layers.MLP_Block(624, hidden_units=[500, 500, 500], dropout_rates=0.1).train()
    x = torch.randn(512, 624, requires_grad=True)
    F2.mlp_chain(x, tower.chain_layers()).sum().backward()
    names = [n for n, _ in recorder]
    assert names[:4] == ["b2_dropout_rng_take"] + ["b2_gemm_tc_ex"] * 3 and names[4] == "b2_prep_operand"
    del recorder[:]
    odd = layers.MLP_Block(40, hidden_units=[18, 36], output_dim=1, dropout_rates=0.5).train()
    x = torch.randn(130, 40, requires_grad=True)
    F2.mlp_chain(x, odd.chain_layers()).sum().backward()
    names = [n for n, _ in recorder]
    assert names.count("b2_dropout_apply") == 2 and names.count("b2_prep_operand") == 1
    assert [i for n, i in recorder if n == "b2_head_bwd_ex"][0]["layer"] == 1


def test_stacks_that_stay_per_layer():
    assert c2_block(0.2, batch_norm=True).train().chain_layers() is None
    dice = layers.MLP_Block(40, hidden_units=[16, 16], hidden_activations=[layers.Dice(16), layers.Dice(16)],
                            output_dim=1, dropout_rates=0.2)
    assert dice.train().chain_layers() is None
    one = c2_block(0.2)
    one.mlp[2] = torch.nn.Dropout(p=1.0)
    assert one.train().chain_layers() is None and one.eval().chain_layers() is None
    zero = c2_block(0.2)
    zero.mlp[2] = torch.nn.Dropout(p=0.0)
    assert zero.chain_layers() is None
    tanh = layers.MLP_Block(40, hidden_units=[16], hidden_activations="Tanh", output_dim=1, dropout_rates=0.2)
    assert tanh.chain_layers() is None


def test_module_tree_and_state_dict_keep_the_dropout_modules():
    mlp = c2_block(0.2)
    assert [type(m).__name__ for m in mlp.mlp] == ["Linear", "ReLU", "Dropout"] * 3 + ["Linear"]
    assert list(mlp.state_dict()) == ["mlp.%d.%s" % (i, n) for i in (0, 3, 6, 9) for n in ("weight", "bias")]
    chain = mlp.train().chain_layers()
    assert [len(c) for c in chain] == [4, 4, 4, 3] and [c[3] for c in chain[:3]] == [0.2] * 3


# ------------------------------------------------------------------ GEMM plans of descriptors with a mask
def _plan(M, N, K, a_mn, b_mn, mode, dgrad):
    d = _lib.b2_gemm_desc()
    d.a, d.b, d.c = 0x10000000, 0x20000000, 0x30000000
    esz = 2 if mode == "bf16" else 4
    pad = 16 // esz
    d.lda = ((M if a_mn else K) + pad - 1) // pad * pad
    d.ldb = ((N if b_mn else K) + pad - 1) // pad * pad
    d.ldc = N
    d.M, d.N, d.K = M, N, K
    d.a_mn_major, d.b_mn_major = int(a_mn), int(b_mn)
    d.elem_dtype = _lib.B2_BF16 if mode == "bf16" else _lib.B2_F32
    if mode == "tf32x3":
        d.flags = _lib.B2_GEMM_X3_INLINE
    if dgrad:                  # dZ_{i-1} = act'(ybwd) * keep * scale * (dZ_i W_i), its bias gradient and operand
        d.ybwd, d.act_bwd, d.colsum, d.c_small = 0x60000000, B2_ACT_RELU, 0x70000000, 0x80000000
    else:                      # y = act(x W^T + b) * keep * scale
        d.bias, d.act = 0x60000000, B2_ACT_RELU
    d.drop_rng, d.drop_layer = 0x90000000, 2
    d.drop_thresh, d.drop_scale = F2.dropout_consts(0.2)
    plan = _lib.b2_gemm_plan()
    _lib.call("b2_gemm_tc_plan", ctypes.byref(d), ctypes.byref(plan))
    return plan


def test_gemm_plans_with_dropout_fit_the_sm():
    shapes = [(4096, 300, 624), (4096, 624, 300), (300, 624, 4096), (8192, 624, 624), (624, 624, 8192), (2048, 500, 432),
              (65536, 64, 415), (64, 415, 65536), (128, 32, 32), (76, 44, 36), (1, 16, 8), (130, 18, 40), (4096, 1024, 1024),
              (100000, 400, 624), (777, 64, 128), (33, 257, 1000), (8192, 256, 256), (8192, 512, 2048)]
    checked = 0
    for (M, N, K), a_mn, b_mn, mode, dgrad in itertools.product(shapes, (False, True), (False, True),
                                                                 ("tf32", "tf32x3", "bf16"), (False, True)):
        esz = 2 if mode == "bf16" else 4
        if (a_mn and M % (16 // esz)) or (b_mn and N % (16 // esz)):
            continue
        p = _plan(M, N, K, a_mn, b_mn, mode, dgrad)
        tag = (M, N, K, a_mn, b_mn, mode, dgrad)
        assert 1024 <= p.smem_bytes <= 227 * 1024 and 2 <= p.stages <= 4, tag
        assert p.splits == 1, tag            # a masked epilogue is never split over K
        assert p.tiles_m * 128 >= M and p.tiles_n * p.bn >= N and p.grid == p.tiles_m * p.tiles_n, tag
        assert p.bn <= (64 if mode == "tf32x3" else 128) and p.threads == 384, tag
        checked += 1
    assert checked > 200


def test_dropout_arguments_are_validated_before_cuda():
    d = _lib.b2_gemm_desc()
    d.a, d.b, d.c = 0x10000000, 0x20000000, 0x30000000
    d.lda = d.ldb = 64
    d.ldc, d.M, d.N, d.K = 64, 128, 64, 64
    d.drop_rng, d.drop_scale = 0x90000000, 0.0
    with pytest.raises(_lib.B2Error, match="dropout"):
        _lib.call("b2_gemm_tc_plan", ctypes.byref(d), ctypes.byref(_lib.b2_gemm_plan()))
    null, ptr = ctypes.c_void_p(0), ctypes.c_void_p(4096)
    with pytest.raises(_lib.B2Error, match="dropout"):
        _lib.call("b2_dropout_apply", ptr, ptr, 4, 4, 4, ptr, -1, 5, 1.25, null)
    with pytest.raises(_lib.B2Error, match="n_layers"):
        _lib.call("b2_dropout_rng_take", ptr, ptr, 0, null)
    with pytest.raises(_lib.B2Error, match="PREP_MUL"):
        _lib.call("b2_prep_operand", ptr, ptr, _lib.B2_PREP_MUL, 4, 4, ptr, null, null, null, null, ptr, 0, 5, 1.25,
                  null)

"""MIRRN without a GPU: the float64 restatement against the reference's goldens, the filter's circulant table against
torch.fft, construction against the reference's digests (state_dict keys, registration order, frozen parameters,
initial draws), the refusals, the tie rule in position order, the C-ABI range checks, the header and bindings, and
the new kernels' register use."""
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
import mirrn_oracle as MO  # noqa: E402
from fuxictr_b200 import functional as F2, zoo  # noqa: E402
from fuxictr_b200.schema import FeatureMap  # noqa: E402

CASES = ["k5_L8_reuse_b16", "k4_L20_percall_b64", "k2_L20_reuse_b48_one_field", "k1_L8_percall_b7",
         "k12_L6_reuse_b33"]
MODEL_CASES = ["k5_L8_reuse_b16", "k2_L20_reuse_b48_one_field", "k12_L6_reuse_b33"]


def block_from_golden(g):
    """(outputs, leaf x, weight leaves) of the oracle's block on a next_MIRRN_* golden, in float64."""
    kw = g.meta["kwargs"]
    x = g["in"]["x"].clone().double().requires_grad_(True)
    w = {k: v.clone().double().requires_grad_(True) for k, v in g["w"].items()}
    Ws, Wl, P, cws, gammas, betas = MO.block_params(w)
    out = MO.mirrn_block(x, g["in"]["mask"], g["in"]["R"].double(), kw["short_seq_len"], kw["topk"],
                         kw["num_heads"], kw["use_scale"], Ws, Wl, P, cws, gammas, betas)
    return out, x, w


@pytest.mark.parametrize("c", CASES)
def test_oracle_block_matches_reference_golden(c):
    g = Golden("next_MIRRN_%s" % c)
    (target, short, long, pos, interests), x, w = block_from_golden(g)
    assert torch.equal(pos.int(), g["out"]["pos"])
    for got, key in ((short, "short"), (long, "long"), (interests, "interests")):
        assert close(got, g["out"][key], 2e-6), (key, rel_err(got, g["out"][key]))
    gi = g["in"]
    ((target * gi["g_target"].double()).sum() + (short * gi["g_short"].double()).sum()
     + (long * gi["g_long"].double()).sum()).backward()
    assert close(x.grad, g["gin"]["x"], 2e-6), rel_err(x.grad, g["gin"]["x"])
    for k, ref in g["g"].items():
        assert close(w[k].grad, ref, 2e-6, atol=1e-9), (k, rel_err(w[k].grad, ref))


@pytest.mark.parametrize("c", CASES)
def test_golden_complex_weight_gradients_are_diagonal(c):
    """The reference's einsum reads only complex_weight[n, j, j, :]: every other entry gets exactly zero gradient."""
    g = Golden("next_MIRRN_%s" % c)
    for q in range(3):
        gw = g["g"]["MHFT_block.%d.complex_weight" % q].clone()
        assert float(gw.abs().max()) > 0
        for n in range(gw.shape[0]):
            gw[n].diagonal(dim1=0, dim2=1).zero_()
        assert float(gw.abs().max()) == 0.0
    rows = (g["g"]["pos.weight"].abs().sum(1) > 0).nonzero().flatten()
    assert int(rows.min()) >= 1 and int(rows.max()) <= g.meta["L"]     # row 0 never receives gradient


def test_filter_table_matches_torch_fft():
    """a u + b (H u) against irfft(rfft(u) (a + i b), n=k, ortho) for k = 1..256; H = 0 for k <= 2."""
    gen = torch.Generator().manual_seed(3)
    for k in range(1, 257):
        h = F2.mirrn_filter_table(k)
        if k <= 2:
            assert float(h.abs().max()) == 0.0
        u = torch.randn(2, k, 3, generator=gen, dtype=torch.float64)
        a, b = 0.7, -1.3
        ref = torch.fft.irfft(torch.fft.rfft(u, dim=1, norm="ortho") * complex(a, b), n=k, dim=1, norm="ortho")
        idx = (torch.arange(k).view(-1, 1) - torch.arange(k).view(1, -1)) % k
        got = a * u + b * torch.einsum("ts,bsc->btc", h[idx], u)
        assert float((got - ref).abs().max()) < 1e-12 * max(1.0, float(ref.abs().max())), k
        assert torch.allclose(h[idx], -h[idx].t(), atol=1e-14)          # antisymmetric


def _digests(model):
    return [[k, str(v.dtype), list(v.shape), hashlib.sha256(v.detach().contiguous().numpy().tobytes()).hexdigest()]
            for k, v in model.state_dict().items()]


@pytest.mark.parametrize("c", CASES)
def test_construction_matches_reference(c):
    with open(os.path.join(GOLDEN, "mirrn_init.json")) as fd:
        case = json.load(fd)["models"][c]
    torch.manual_seed(case["seed"])
    fm = FeatureMap.from_specs(case["specs"], labels=case["labels"], embedding_dim=case["kwargs"]["embedding_dim"])
    model = zoo.MIRRN(fm, gpu=-1, unknown_keyword=1, **case["kwargs"])
    assert _digests(model) == case["state_dict"]
    names = [k for k, _ in model.named_parameters()]
    assert names[0] == "random_rotations"
    order = ["embedding_layer.", "short_attention.", "pos.", "MHFT_block.0.", "MHFT_block.1.", "MHFT_block.2.",
             "long_attention.", "dnn."]
    firsts = [next(i for i, n in enumerate(names) if n.startswith(p)) for p in order]
    assert firsts == sorted(firsts)
    assert [k for k, p in model.named_parameters() if not p.requires_grad] == ["random_rotations"]
    assert tuple(model.random_rotations.shape) == (model.item_info_dim, case["kwargs"]["hash_bits"])
    assert model.MHFT_block[0].out_dropout.p == 0.1 and model.MHFT_block[0].LayerNorm.eps == 1e-12


# ------------------------------------------------------------------ refusals
def _fm(dim=4, items=2):
    specs = [("user_id", {"type": "categorical", "source": "user", "padding_idx": 0, "vocab_size": 10}),
             ("item_id", {"type": "categorical", "source": "item", "padding_idx": 0, "vocab_size": 20}),
             ("cate_id", {"type": "categorical", "source": "item", "padding_idx": 0, "vocab_size": 5}),
             ("brand_id", {"type": "categorical", "source": "item", "padding_idx": 0, "vocab_size": 5})]
    return FeatureMap.from_specs(specs[:1 + items], embedding_dim=dim)


ARGS = dict(gpu=-1, embedding_dim=4, dnn_hidden_units=[8], attention_dim=8, max_len=60)


@pytest.mark.parametrize("kw,exc,text", [
    (dict(attention_dropout=0.1), NotImplementedError, "attention_dropout"),
    (dict(short_seq_len=1), ValueError, "short_seq_len"),
    (dict(accumulation_steps=2), NotImplementedError, "accumulation_steps"),
    (dict(hash_bits=65), NotImplementedError, "hash_bits"),
    (dict(topk=257), NotImplementedError, "topk"),
    (dict(embedding_dim=132), NotImplementedError, "item width"),
])
def test_constructor_refusals(kw, exc, text):
    with pytest.raises(exc, match=text):
        zoo.MIRRN(_fm(kw.get("embedding_dim", 4)), **dict(ARGS, **kw))


def test_item_width_not_divisible_by_4_is_refused():
    """The reference's default embedding_dim=10 with three item fields (d = 30) fails at its first forward."""
    with pytest.raises(ValueError, match="divisible by 4"):
        zoo.MIRRN(_fm(10, items=3), **dict(ARGS, embedding_dim=10))
    assert F2.mirrn_bound(30, 50, 50, 32) is not None


def test_lazy_tables_and_sharding_are_refused():
    model = zoo.MIRRN(_fm(), **ARGS)
    with pytest.raises(NotImplementedError, match="lazy"):
        model.use_fused_optimizer(lazy_tables=True)
    with pytest.raises(NotImplementedError, match="sharded"):
        model.enable_sharding(None, 8, 4)


def test_history_longer_than_max_len_is_refused():
    model = zoo.MIRRN(_fm(), **dict(ARGS, max_len=10))
    with pytest.raises(ValueError, match="max_len"):
        model.interest(torch.zeros(2, 12, 8), torch.ones(2, 11))


def test_dnn_width_and_bounds():
    model = zoo.MIRRN(_fm(), **dict(ARGS, num_heads=2))
    assert model.item_info_dim == 8
    assert model.dnn.mlp[0].in_features == 12 + 2 * 8
    assert F2.mirrn_bound(48, 50, 4, 32, 8192) is None                      # MIRRN_default: D 16, three item fields
    assert F2.mirrn_bound(48, 1000, 50, 32, 4096) is None
    assert F2.mirrn_bound(12, 4096, 256, 64, 4096) is None
    assert F2.mirrn_bound(12, 4097, 50, 32) is not None
    assert F2.mirrn_bound(12, 50, 50, 65) is not None
    assert F2.mirrn_bound(256, 256, 256, 32) is not None                    # the filter's shared memory
    assert F2.mirrn_bound(12, 1024, 50, 32, 2 ** 31 // 1025 + 1) is not None


def test_filter_layer_runs_inside_the_block():
    from fuxictr_b200.layers import FilterLayer2
    layer = FilterLayer2(5, 8, 0.1, 4)
    assert [k for k in layer.state_dict()] == ["complex_weight", "LayerNorm.weight", "LayerNorm.bias"]
    with pytest.raises(NotImplementedError, match="mirrn_interest"):
        layer(torch.zeros(1, 5, 8))
    with pytest.raises(NotImplementedError, match="n_block"):
        FilterLayer2(5, 8, 0.1, 2)


# ------------------------------------------------------------------ the tie rule, in position order
def test_tie_rule_in_position_order():
    dist = torch.tensor([[3, 1, 1, 0, 1, 3, 1],
                         [5, 5, 5, 5, 5, 5, 5],
                         [2, 0, 2, 0, 1, 0, 2]])
    assert MO.select(dist, 4).tolist() == [[1, 2, 3, 4], [0, 1, 2, 3], [1, 3, 4, 5]]
    assert MO.select(dist, 2).tolist() == [[1, 3], [0, 1], [1, 3]]


# ------------------------------------------------------------------ C-ABI
@pytest.fixture(scope="module")
def lib():
    import __graft_entry__
    __graft_entry__.build()
    from fuxictr_b200 import _lib
    return _lib.load()


def _p(v=0x1000):
    return ctypes.c_void_p(v)


def test_abi_range_and_null_checks(lib):
    n = None
    # retrieval: d % 4, L, k, bits, r_stride, NULL
    assert lib.b2_mirrn_retrieve_fwd(_p(), _p(), _p(), 0, 2, 10, 6, 32, 4, _p(), n) != 0
    assert lib.b2_mirrn_retrieve_fwd(_p(), _p(), _p(), 0, 2, 0, 8, 32, 1, _p(), n) != 0
    assert lib.b2_mirrn_retrieve_fwd(_p(), _p(), _p(), 0, 2, 10, 8, 32, 11, _p(), n) != 0
    assert lib.b2_mirrn_retrieve_fwd(_p(), _p(), _p(), 0, 2, 10, 8, 65, 4, _p(), n) != 0
    assert lib.b2_mirrn_retrieve_fwd(_p(), _p(), _p(), 7, 2, 10, 8, 32, 4, _p(), n) != 0
    assert lib.b2_mirrn_retrieve_fwd(_p(), _p(), _p(0), 0, 2, 10, 8, 32, 4, _p(), n) != 0
    assert lib.b2_mirrn_retrieve_fwd(_p(), _p(), _p(), 0, 0, 10, 8, 32, 4, _p(), n) == 0       # B = 0: no launch
    # filter: the position table must reach row L
    w = [_p()] * 3
    assert lib.b2_mirrn_filter_fwd(_p(), _p(), _p(), 10, *w, _p(), 2, 10, 8, 4, _p(), _p(), n) != 0
    assert lib.b2_mirrn_filter_fwd(_p(), _p(), _p(), 11, *w, _p(0), 2, 10, 8, 4, _p(), _p(), n) != 0
    assert lib.b2_mirrn_filter_fwd(_p(), _p(), _p(), 11, *w, _p(), 0, 10, 8, 4, _p(), _p(), n) == 0
    assert lib.b2_mirrn_filter_bwd(_p(), _p(), _p(), _p(), 10, *w, _p(), 2, 10, 8, 4, _p(), *w, _p(), n) != 0
    assert lib.b2_mirrn_filter_bwd(_p(), _p(), _p(), _p(), 11, *w, _p(), 2, 10, 8, 4, _p(), *w, _p(0), n) != 0
    assert lib.b2_mirrn_filter_bwd(_p(), _p(), _p(), _p(), 257, *w, _p(), 2, 256, 256, 256, _p(), *w, _p(), n) != 0
    assert b"shared memory" in lib.b2_last_error()
    assert lib.b2_mirrn_filter_fwd(_p(), _p(), _p(), 257, *w, _p(), 2, 256, 256, 256, _p(), _p(), n) != 0
    assert b"shared memory" in lib.b2_last_error()
    assert lib.b2_mirrn_mean_fwd(_p(0), 2, 8, 4, _p(), n) != 0
    assert lib.b2_mirrn_mean_bwd(_p(), 2, 8, 0, _p(), n) != 0
    assert lib.b2_mirrn_assemble_bwd(_p(), _p(), _p(), _p(), 11, _p(), _p(), 2, 10, 8, 4, _p(), n) != 0
    assert lib.b2_mirrn_assemble_bwd(_p(), _p(), _p(), _p(), 3, _p(0), _p(), 2, 10, 8, 4, _p(), n) != 0
    assert lib.b2_mirrn_assemble_bwd(_p(), _p(), _p(), _p(), 3, _p(), _p(), 0, 10, 8, 4, _p(), n) == 0


def test_header_and_bindings():
    from fuxictr_b200 import _lib
    header = open(os.path.join(ROOT, "include", "fuxictr_b200.h")).read()
    names = ["b2_mirrn_retrieve_fwd", "b2_mirrn_filter_fwd", "b2_mirrn_filter_bwd", "b2_mirrn_mean_fwd",
             "b2_mirrn_mean_bwd", "b2_mirrn_assemble_bwd"]
    for name in names:
        assert ("B2_API int %s(" % name) in header and name in _lib.SIGNATURES
    assert "#define B2_MIRRN_MAX_BITS %d" % _lib.B2_MIRRN_MAX_BITS in header


def test_new_kernels_do_not_spill():
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    src = os.path.join(ROOT, "fuxictr_b200", "csrc", "mirrn.cu")
    out = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v",
                          "-I", os.path.join(ROOT, "include"), "-c", src, "-o", os.devnull],
                         capture_output=True, text=True, check=True).stderr
    lines = [ln for ln in out.splitlines() if "spill" in ln]
    assert len(lines) == 6 and all("0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in ln
                                   for ln in lines), out

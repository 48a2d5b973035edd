"""ETA and SDIM without a GPU: the float64 restatement against the reference's goldens, construction against the
reference's digests (state_dict keys, frozen parameters, initial draws), the refusals, the DNN width formula, the tie
rule and the new kernels' register use."""
import hashlib
import json
import os
import subprocess
import sys

import pytest
import torch

from conftest import Golden, GOLDEN, ROOT, close, rel_err

sys.path.insert(0, ROOT)
import longctr_oracle as LO  # noqa: E402
from fuxictr_b200 import functional as F2, zoo  # noqa: E402
from fuxictr_b200.schema import FeatureMap  # noqa: E402

ETA_CASES = ["reuse_b32", "perbatch_b64_Lbelowk", "reuse_b7_one_field"]
SDIM_CASES = ["l2_h3_b3", "noqkvo_h1_b2", "perbatch_l2_h2_b4"]
ATT = ("W_q", "W_k", "W_v", "W_o")


def _weights(w, prefix):
    keys = ["%s.%s.weight" % (prefix, n) for n in ATT]
    return tuple(w[k] for k in keys) if keys[0] in w else None


def block_from_golden(name, g, double=True):
    """(outputs, leaf x, weight leaves) of the oracle's block on a next_* golden."""
    cast = (lambda t: t.clone().double()) if double else (lambda t: t.clone())
    kw = g.meta["kwargs"]
    x = cast(g["in"]["x"]).requires_grad_(True)
    w = {k: cast(v).requires_grad_(True) for k, v in g["w"].items()}
    mask, R = g["in"]["mask"], cast(g["in"]["R"])
    heads = 1 if (name == "SDIM" and not kw["use_qkvo"]) else kw["num_heads"]
    if name == "ETA":
        out = LO.eta_block(x, mask, R, kw["short_seq_len"], kw["topk"], heads, kw["use_scale"],
                           _weights(w, "short_attention"), _weights(w, "long_attention"))
    else:
        out = LO.sdim_block(x, mask, R, kw["short_seq_len"], kw["l2_norm"], kw["num_heads"], kw["use_scale"],
                            _weights(w, "short_attention"))
    return out, x, w


@pytest.mark.parametrize("name,c", [("ETA", c) for c in ETA_CASES] + [("SDIM", c) for c in SDIM_CASES])
def test_oracle_block_matches_reference_golden(name, c):
    g = Golden("next_%s_%s" % (name, c))
    out, x, w = block_from_golden(name, g)
    target, short, long = out[:3]
    assert close(short, g["out"]["short"], 2e-6), rel_err(short, g["out"]["short"])
    assert close(long, g["out"]["long"], 2e-6), rel_err(long, g["out"]["long"])
    if name == "ETA":
        assert torch.equal(out[3].sort(dim=1).values.int(), g["out"]["pos"])
    gi = g["in"]
    ((target * gi["g_target"].double()).sum() + (short * gi["g_short"].double()).sum()
     + (long * gi["g_long"].double()).sum()).backward()
    assert close(x.grad, g["gin"]["x"], 2e-6), rel_err(x.grad, g["gin"]["x"])
    for k, ref in g["g"].items():
        assert close(w[k].grad, ref, 2e-6), (k, rel_err(w[k].grad, ref))


def _digests(model):
    return [[k, str(v.dtype), list(v.shape), hashlib.sha256(v.detach().contiguous().numpy().tobytes()).hexdigest()]
            for k, v in model.state_dict().items()]


@pytest.mark.parametrize("name,c", [("ETA", c) for c in ETA_CASES] + [("SDIM", c) for c in SDIM_CASES])
def test_construction_matches_reference(name, c):
    with open(os.path.join(GOLDEN, name.lower() + "_init.json")) as fd:
        case = json.load(fd)["models"][c]
    torch.manual_seed(case["seed"])
    fm = FeatureMap.from_specs(case["specs"], labels=case["labels"], embedding_dim=case["kwargs"]["embedding_dim"])
    model = getattr(zoo, name)(fm, gpu=-1, unknown_keyword=1, **case["kwargs"])
    assert _digests(model) == case["state_dict"]
    frozen = [k for k, p in model.named_parameters() if not p.requires_grad]
    assert frozen == (["random_rotations"] if name == "ETA" else ["powers_of_two", "random_rotations"])


# ------------------------------------------------------------------ refusals and the width formula
def _fm(dim=4, two_items=True):
    specs = [("user_id", {"type": "categorical", "source": "user", "padding_idx": 0, "vocab_size": 10}),
             ("item_id", {"type": "categorical", "source": "item", "padding_idx": 0, "vocab_size": 20})]
    if two_items:
        specs.append(("cate_id", {"type": "categorical", "source": "item", "padding_idx": 0, "vocab_size": 5}))
    return FeatureMap.from_specs(specs, embedding_dim=dim)


@pytest.mark.parametrize("name", ["ETA", "SDIM"])
def test_item_info_dim_and_dnn_width(name):
    model = getattr(zoo, name)(_fm(), gpu=-1, embedding_dim=4, dnn_hidden_units=[8], attention_dim=8, num_heads=2)
    assert model.item_info_dim == 8
    assert model.dnn.mlp[0].in_features == 12 + 2 * 8      # sum_emb_out_dim() + 2 item_info_dim


@pytest.mark.parametrize("name", ["ETA", "SDIM"])
@pytest.mark.parametrize("kw,exc,text", [
    (dict(attention_dropout=0.1), NotImplementedError, "attention_dropout"),
    (dict(short_seq_len=1), ValueError, "short_seq_len"),
    (dict(accumulation_steps=2), NotImplementedError, "accumulation_steps"),
])
def test_constructor_refusals(name, kw, exc, text):
    with pytest.raises(exc, match=text):
        getattr(zoo, name)(_fm(), gpu=-1, embedding_dim=4, dnn_hidden_units=[8], attention_dim=8, **kw)


@pytest.mark.parametrize("kw,text", [(dict(hash_bits=65), "hash_bits"), (dict(topk=257), "topk"),
                                     (dict(embedding_dim=200), "item width")])
def test_eta_bound_refusals(kw, text):
    args = dict(gpu=-1, embedding_dim=4, dnn_hidden_units=[8], attention_dim=8)
    args.update(kw)
    with pytest.raises(NotImplementedError, match=text):
        zoo.ETA(_fm(), **args)


@pytest.mark.parametrize("kw,text", [(dict(hash_bits=25), "hash_bits"), (dict(num_hashes=33), "num_hashes")])
def test_sdim_bound_refusals(kw, text):
    with pytest.raises(NotImplementedError, match=text):
        zoo.SDIM(_fm(), gpu=-1, embedding_dim=4, dnn_hidden_units=[8], attention_dim=8, **kw)


def test_bounds_cover_the_default_configs():
    for items in (1, 2, 3, 4):
        assert F2.eta_bound(4 * items, 50, 50, 32, 8192) is None            # ETA_default: D 4
        assert F2.sdim_bound(32 * items, 50, 2, 4, 10000) is None           # SDIM_default: D 32
    assert F2.eta_bound(12, 4096, 256, 64, 4096) is None
    assert F2.eta_bound(12, 4097, 50, 32) is not None
    assert F2.eta_bound(12, 0, 50, 32) is not None
    assert F2.eta_bound(12, 1024, 50, 32, 2 ** 31 // 1025 + 1) is not None
    assert F2.sdim_bound(256, 4096, 32, 24) is not None                     # shared memory


def test_lazy_tables_and_sharding_are_refused():
    model = zoo.ETA(_fm(), gpu=-1, embedding_dim=4, dnn_hidden_units=[8], attention_dim=8)
    with pytest.raises(NotImplementedError, match="lazy"):
        model.use_fused_optimizer(lazy_tables=True)
    with pytest.raises(NotImplementedError, match="sharded"):
        model.enable_sharding(None, 8, 4)


# ------------------------------------------------------------------ the tie rule
def test_tie_rule_on_hand_made_distances():
    dist = torch.tensor([[3, 1, 1, 0, 1, 3, 1],
                         [5, 5, 5, 5, 5, 5, 5],
                         [2, 0, 2, 0, 1, 0, 2]])
    assert LO.select(dist, 4).tolist() == [[3, 1, 2, 4], [0, 1, 2, 3], [1, 3, 5, 4]]
    assert LO.select(dist, 7)[2].tolist() == [1, 3, 5, 4, 0, 2, 6]


def test_new_kernels_do_not_spill():
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    src = os.path.join(ROOT, "fuxictr_b200", "csrc", "lsh.cu")
    out = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v",
                          "-I", os.path.join(ROOT, "include"), "-c", src, "-o", os.devnull],
                         capture_output=True, text=True, check=True).stderr
    lines = [ln for ln in out.splitlines() if "spill" in ln]
    assert len(lines) == 3 and all("0 bytes spill stores, 0 bytes spill loads" in ln for ln in lines), out

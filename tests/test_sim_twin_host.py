"""SIM and TWIN without a GPU: the float64 restatement against the reference's goldens, construction against the
reference's digests (state_dict keys, registration order, initial draws), the refusals, the tie rule, the C-ABI range
checks and the new kernels' register use."""
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
import sim_twin_oracle as SO  # noqa: E402
from fuxictr_b200 import _lib, functional as F2, zoo  # noqa: E402
from fuxictr_b200.schema import FeatureMap  # noqa: E402

CASES = ["h2_k5", "h1_k8_one_field", "h2_k12"]
MHTA = ("W_q", "W_k", "W_v", "W_o")
TOPK = ("W_q", "W_h", "W_v", "W_o")


def block_from_golden(name, g, double=True):
    """(outputs, output names, leaf x, weight leaves) of the oracle's block on a next_* golden."""
    cast = (lambda t: t.clone().double()) if double else (lambda t: t.clone())
    kw = g.meta["kwargs"]
    x = cast(g["in"]["x"]).requires_grad_(True)
    w = {k: cast(v).requires_grad_(True) for k, v in g["w"].items()}
    att = lambda p, n=MHTA: tuple(w["%s.%s.weight" % (p, m)] for m in n)     # noqa: E731
    mask = g["in"]["mask"]
    if name == "SIM":
        out = SO.sim_block(x, mask, kw["short_seq_len"], kw["topk"], kw["num_heads"], w["W_a.weight"],
                           w["W_b.weight"], att("short_attention"), att("long_attention"))
        return out, ("target", "short", "long", "pooled"), x, w
    out = SO.twin_block(x, mask, kw["short_seq_len"], kw["topk"], kw["num_heads"], att("short_attention"),
                        att("long_attention", TOPK))
    return out, ("target", "short", "long"), x, w


@pytest.mark.parametrize("name", ["SIM", "TWIN"])
@pytest.mark.parametrize("c", CASES)
def test_oracle_block_matches_reference_golden(name, c):
    g = Golden("next_%s_%s" % (name, c))
    out, names, x, w = block_from_golden(name, g)
    for o, n in zip(out, names):
        assert close(o, g["out"][n], 2e-6), (n, rel_err(o, g["out"][n]))
    assert torch.equal(out[-1].sort(dim=-1).values.int(), g["out"]["pos"])
    sum((o * g["in"]["g_" + n].double()).sum() for o, n in zip(out, names)).backward()
    assert close(x.grad, g["gin"]["x"], 2e-6), rel_err(x.grad, g["gin"]["x"])
    for k, ref in g["g"].items():
        assert close(w[k].grad, ref, 2e-6), (k, rel_err(w[k].grad, ref))


def test_goldens_cover_the_selection_cases():
    """L below, at and above topk; a SIM row with fewer positive valid scores than k (masked rows fill the selection);
    empty and full histories."""
    Ls = {Golden("next_SIM_" + c).meta["kwargs"]["topk"] for c in CASES}
    assert min(Ls) < 8 and 8 in Ls and max(Ls) > 8
    filled = False
    for c in CASES:
        g = Golden("next_SIM_" + c)
        x, mask, kw = g["in"]["x"].double(), g["in"]["mask"], g.meta["kwargs"]
        w = g["w"]
        qk = torch.einsum("ba,bla->bl", x[:, -1] @ w["W_a.weight"].double().t(),
                          x[:, :-1] @ w["W_b.weight"].double().t()) * mask.double()
        k = min(kw["topk"], 8)
        filled |= bool((((qk > 0).sum(1) < k) & ((mask == 0).sum(1) > 0)).any())
    assert filled
    for name in ("SIM", "TWIN"):
        masks = [Golden("next_%s_%s" % (name, c))["in"]["mask"] for c in CASES]
        assert any(bool((m.sum(1) == 0).any()) for m in masks) and all(bool((m.sum(1) == 8).any()) for m in masks)


def _digests(model):
    return [[k, str(v.dtype), list(v.shape), hashlib.sha256(v.detach().contiguous().numpy().tobytes()).hexdigest()]
            for k, v in model.state_dict().items()]


@pytest.mark.parametrize("name", ["SIM", "TWIN"])
@pytest.mark.parametrize("c", CASES)
def test_construction_matches_reference(name, c):
    with open(os.path.join(GOLDEN, name.lower() + "_init.json")) as fd:
        case = json.load(fd)["models"][c]
    torch.manual_seed(case["seed"])
    fm = FeatureMap.from_specs(case["specs"], labels=case["labels"], embedding_dim=case["kwargs"]["embedding_dim"])
    model = getattr(zoo, name)(fm, gpu=-1, unknown_keyword=1, **case["kwargs"])
    assert _digests(model) == case["state_dict"]


def test_sim_module_order():
    model = zoo.SIM(_fm(), gpu=-1, embedding_dim=4, dnn_hidden_units=[8], attention_dim=8)
    assert [n for n, _ in model.named_children()] == ["output_activation", "embedding_layer", "W_a", "W_b",
                                                      "short_attention", "long_attention", "dnn_aux", "dnn"]


# ------------------------------------------------------------------ refusals
def _fm(dim=4, two_items=True):
    specs = [("user_id", {"type": "categorical", "source": "user", "padding_idx": 0, "vocab_size": 10}),
             ("item_id", {"type": "categorical", "source": "item", "padding_idx": 0, "vocab_size": 20})]
    if two_items:
        specs.append(("cate_id", {"type": "categorical", "source": "item", "padding_idx": 0, "vocab_size": 5}))
    return FeatureMap.from_specs(specs, embedding_dim=dim)


@pytest.mark.parametrize("name", ["SIM", "TWIN"])
@pytest.mark.parametrize("kw,exc,text", [
    (dict(attention_dropout=0.1), NotImplementedError, "attention_dropout"),
    (dict(short_seq_len=1), ValueError, "short_seq_len"),
    (dict(accumulation_steps=2), NotImplementedError, "accumulation_steps"),
    (dict(attention_dim=9, num_heads=2), ValueError, "not divisible"),
    (dict(topk=257), NotImplementedError, "topk"),
    (dict(embedding_dim=200), NotImplementedError, "item width"),
])
def test_constructor_refusals(name, kw, exc, text):
    args = dict(gpu=-1, embedding_dim=4, dnn_hidden_units=[8], attention_dim=8)
    args.update(kw)
    with pytest.raises(exc, match=text):
        getattr(zoo, name)(_fm(), **args)


def test_sim_gsu_type_and_twin_cross_features_are_refused():
    with pytest.raises(NotImplementedError, match="gsu_type"):
        zoo.SIM(_fm(), gpu=-1, embedding_dim=4, dnn_hidden_units=[8], attention_dim=8, gsu_type="hard")
    with pytest.raises(NotImplementedError, match="Kc_cross_features.*L = 1"):
        zoo.TWIN(_fm(), gpu=-1, embedding_dim=4, dnn_hidden_units=[8], attention_dim=8, Kc_cross_features=1)


@pytest.mark.parametrize("name", ["SIM", "TWIN"])
def test_lazy_tables_and_sharding_are_refused(name):
    model = getattr(zoo, name)(_fm(), gpu=-1, embedding_dim=4, dnn_hidden_units=[8], attention_dim=8)
    with pytest.raises(NotImplementedError, match="lazy"):
        model.use_fused_optimizer(lazy_tables=True)
    with pytest.raises(NotImplementedError, match="sharded"):
        model.enable_sharding(None, 8, 4)


def test_bounds():
    for items in (1, 2, 3):
        assert F2.sim_bound(4 * items, 50, 50, 2, 8192) is None             # SIM_default / TWIN_default: D 4
        assert F2.twin_bound(4 * items, 50, 50, 2, 8192) is None
    assert F2.sim_bound(12, 4096, 256, 4, 4096) is None
    assert F2.twin_bound(12, 4096, 256, 4, 4096) is None
    assert "history length" in F2.sim_bound(12, 4097, 50, 2)
    assert "history length" in F2.twin_bound(12, 0, 50, 2)
    assert "2^31" in F2.twin_bound(12, 1024, 50, 2, 2 ** 31 // 1025 + 1)
    assert "num_heads" in F2.twin_bound(64, 50, 50, 17)
    assert "shared memory" in F2.twin_bound(32, 4096, 256, 32)


# ------------------------------------------------------------------ the tie rule
def test_tie_rule_on_hand_made_scores():
    s = torch.tensor([[0.0, -0.0, 0.0, -0.0, 0.2],
                      [-1e9, -1e9, -1e9, -1e9, -1e9],
                      [1.0, -1e9, 1.0, 0.5, -1e9]])
    assert SO.select(s, 3).tolist() == [[4, 0, 1], [0, 1, 2], [0, 2, 3]]
    assert SO.select(s, 5)[2].tolist() == [0, 2, 3, 1, 4]
    assert SO.select(torch.tensor([[-0.0, 0.0, -0.5, -0.0]]), 4).tolist() == [[0, 1, 3, 2]]


# ------------------------------------------------------------------ C-ABI range checks
def test_kernel_range_is_checked_before_any_cuda_call():
    import __graft_entry__
    __graft_entry__.build()
    L = _lib.load()
    p = ctypes.c_void_p(4096)
    z = ctypes.c_void_p(0)

    def sim(B=8, Lt=50, d=12, k=50, x=p):
        return L.b2_sim_retrieve_fwd(x, p, p, B, Lt, d, k, p, p, p, p, p, None)

    def twin(B=8, Lt=50, d=12, H=2, k=50, q=p):
        return L.b2_twin_topk_fwd(q, p, p, B, Lt, d, H, k, p, p, p, None)
    assert sim(d=257) == -1 and b"item width" in L.b2_last_error()
    assert sim(Lt=4097) == -1 and b"history length" in L.b2_last_error()
    assert sim(Lt=0) == -1 and sim(k=0) == -1 and sim(k=51) == -1 and b"k must" in L.b2_last_error()
    assert sim(Lt=300, k=257) == -1
    assert sim(B=-1) == -1 and b"negative" in L.b2_last_error()
    assert sim(B=(1 << 31) // 51 + 1) == -1 and b"2^31" in L.b2_last_error()
    assert sim(x=z) == -1 and b"NULL" in L.b2_last_error()
    assert sim(B=0) == 0
    assert twin(H=33) == -1 and twin(d=256, H=5) == -1 and b"heads" in L.b2_last_error()
    assert twin(q=z) == -1 and b"NULL" in L.b2_last_error()
    assert twin(B=0) == 0
    assert L.b2_sim_gsu_bwd(p, p, z, 8, 50, 12, p, p, None) == -1 and b"NULL" in L.b2_last_error()
    assert L.b2_sim_gsu_bwd(p, p, p, 8, 50, 0, p, p, None) == -1
    assert L.b2_sim_assemble_bwd(p, p, p, p, p, 0, p, p, p, p, p, p, 8, 50, 12, 50, p, None) == -1 \
        and b"short window" in L.b2_last_error()
    assert L.b2_sim_assemble_bwd(p, p, p, z, p, 4, p, p, p, p, p, p, 8, 50, 12, 50, p, None) == -1
    assert L.b2_twin_topk_bwd(p, p, p, p, p, p, p, p, p, p, p, 51, 8, 50, 12, 2, 50, p, p, None) == -1 \
        and b"short window" in L.b2_last_error()
    assert L.b2_twin_topk_bwd(p, p, p, p, p, p, p, z, p, p, p, 4, 8, 50, 12, 2, 50, p, p, None) == -1 \
        and b"NULL" in L.b2_last_error()
    assert L.b2_twin_topk_bwd(p, p, p, p, p, p, p, p, p, p, p, 4, 0, 50, 12, 2, 50, p, p, None) == 0


# ------------------------------------------------------------------ register use
def test_new_kernels_do_not_spill(tmp_path):
    from fuxictr_b200 import build
    nvcc = "/usr/local/cuda/bin/nvcc"
    nvcc = os.environ.get("NVCC") or (nvcc if os.path.exists(nvcc) else "nvcc")
    r = subprocess.run([nvcc] + build.NVCC_FLAGS + ["-Xptxas", "-v", "-I", build.INCLUDE, "-c",
                        os.path.join(build.CSRC, "topk_retrieval.cu"), "-o", str(tmp_path / "topk.o")],
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    log = r.stdout + r.stderr
    kernels = [line for line in log.splitlines() if "Compiling entry function" in line]
    assert len(kernels) == 5 and all("sim_" in k or "twin_" in k for k in kernels), log
    spills = [line for line in log.splitlines() if "spill" in line]
    assert len(spills) == 5 and all("0 bytes spill stores, 0 bytes spill loads" in s for s in spills), log

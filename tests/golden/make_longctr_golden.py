"""Generates the ETA and SDIM fixtures by running the REAL reference (model_zoo/LongCTR/ETA/ETA.py and
model_zoo/LongCTR/SDIM/SDIM.py, imported by path), with make_golden.py's helpers and settings (reference import stubs,
one thread, deterministic algorithms) and its own generators, so no other fixture changes.  Run in the build container
only:

    python tests/golden/make_longctr_golden.py

Writes
  eta_init.json / sdim_init.json   state_dict keys, dtypes, shapes and SHA-256 of each tensor right after construction
                                   under torch.manual_seed(777), for every configuration below;
  next_<ETA|SDIM>_<c>.npz          the interest block on a (B, L + 1, d) item_feat_emb leaf: in/x, in/mask, in/R (the
                                   rotations the block used, (1 or B, d, ...)), in/g_target, in/g_short, in/g_long;
                                   out/short, out/long, out/pos (ETA: the chosen positions, sorted ascending); gin/x;
                                   w and g the two attentions' weights and gradients;
  model_<ETA|SDIM>_<c>.npz         (reuse_hash=True configurations) the LongCTR triples of three batches (in/<feature>,
                                   in/mask, in/label), w the state after construction, out/y_pred and out/loss of
                                   batch 0 and g its gradients, w1 / w3 the state after 1 and 3 train_step()s.
Each batch holds a full history (row 1) and a shortest one (row 0): empty, or for ETA with topk < L exactly topk items;
the rest are pre-padded with random lengths, as the reference's collator pads.  The maker asserts, for every valid row of every recorded step, that no SimHash projection
lies within 1e-4 |x| |R_j| of its hyperplane (so no summation order flips a bit) and that no ETA row has a distance tie
across its k boundary (so the reference's selected set is well defined); it re-draws the embeddings and the ids until
both hold.
"""
import hashlib
import importlib.util
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_golden as G  # noqa: E402  (imports the reference)

torch = G.torch

SPECS = [("user_id", {"type": "categorical", "source": "user", "padding_idx": 0, "vocab_size": 30}),
         ("item_id", {"type": "categorical", "source": "item", "padding_idx": 0, "vocab_size": 80}),
         ("cate_id", {"type": "categorical", "source": "item", "padding_idx": 0, "vocab_size": 12})]
ONE_ITEM_SPECS = SPECS[:2]
COMMON = dict(dnn_hidden_units=[16, 8], dnn_activations="ReLU", attention_dim=8, num_heads=2, use_scale=True,
              net_dropout=0, batch_norm=False)
CASES = {
    "ETA": {
        "reuse_b32": dict(embedding_dim=4, reuse_hash=True, hash_bits=32, topk=5, short_seq_len=4, **COMMON),
        "perbatch_b64_Lbelowk": dict(embedding_dim=4, reuse_hash=False, hash_bits=64, topk=12, short_seq_len=3,
                                     **COMMON),
        "reuse_b7_one_field": dict(embedding_dim=8, reuse_hash=True, hash_bits=7, topk=8, short_seq_len=5,
                                   **dict(COMMON, num_heads=1)),
    },
    "SDIM": {
        "l2_h3_b3": dict(embedding_dim=4, reuse_hash=True, num_hashes=3, hash_bits=3, l2_norm=True, use_qkvo=True,
                         short_seq_len=4, **COMMON),
        "noqkvo_h1_b2": dict(embedding_dim=4, reuse_hash=True, num_hashes=1, hash_bits=2, l2_norm=False,
                             use_qkvo=False, short_seq_len=3, **COMMON),
        "perbatch_l2_h2_b4": dict(embedding_dim=4, reuse_hash=False, num_hashes=2, hash_bits=4, l2_norm=True,
                                  use_qkvo=True, short_seq_len=5, **COMMON),
    },
}
L_HIST = 8


def specs_of(case):
    return ONE_ITEM_SPECS if case.endswith("one_field") else SPECS


def load(name):
    path = os.path.join(G.REF, "model_zoo", "LongCTR", name, name + ".py")
    spec = importlib.util.spec_from_file_location("longctr_" + name, path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def digests(module):
    return [[k, str(v.dtype), list(v.shape), hashlib.sha256(v.detach().contiguous().numpy().tobytes()).hexdigest()]
            for k, v in module.state_dict().items()]


def build(M, model, case, seed):
    kwargs = CASES[model][case]
    torch.manual_seed(seed)
    fm = G.synthetic_fm(specs_of(case), emb_dim=kwargs["embedding_dim"])
    return fm, getattr(M, model)(fm, **G.model_params(**kwargs))


def rotations_for(model, B, d, gen):
    """The rotations a forward uses: the shared parameter, or a fresh per-batch draw."""
    if model.reuse_hash:
        return model.random_rotations.detach()
    shape = (B, d, model.hash_bits) if not hasattr(model, "num_hashes") else (B, d, model.num_hashes, model.hash_bits)
    return torch.randn(shape, generator=gen)


def well_posed(model, x, mask, R):
    """No projection within 1e-4 |x| |R_j| of a hyperplane on any valid row (and the target); no ETA distance tie across
    the k boundary (masked positions, all at distance bits + 1, tie with each other)."""
    x = x.detach().double()
    R = R.double().expand(x.shape[0], *R.shape[1:])
    Rf = R.reshape(R.shape[0], R.shape[1], -1)
    proj = torch.einsum("bld,bdh->blh", x, Rf)
    margin = 1e-4 * x.norm(dim=-1, keepdim=True) * Rf.norm(dim=1, keepdim=True)
    valid = torch.cat([mask != 0, torch.ones(mask.shape[0], 1, dtype=torch.bool)], dim=1)
    nonzero = x.norm(dim=-1) > 0
    close = (proj.abs() <= margin) & (valid & nonzero).unsqueeze(-1)
    if bool(close.any()):
        return False
    if hasattr(model, "topk"):
        bits = model.hash_bits
        code = proj > 0
        dist = (code[:, :-1] ^ code[:, -1:]).sum(-1)
        dist = torch.where(mask != 0, dist, torch.full_like(dist, bits + 1))
        k = min(model.topk, mask.shape[1])
        if k < mask.shape[1]:
            s = dist.sort(dim=1).values
            tie = s[:, k - 1] == s[:, k]
            if bool(tie.any()):
                return False
    return True


def triple(fm, B, L, gen, min_len=0):
    """(batch_dict, item_dict, mask) as LongCTRDataLoader's collator yields them: pre-padded histories of at least
    min_len items (row 0 holds exactly min_len, row 1 is full), the target last in each sample's block of L + 1 item
    rows."""
    lens = torch.randint(max(min_len, 1), L + 1, (B,), generator=gen)
    lens[0], lens[1] = min_len, L
    hist = torch.zeros(B, L, dtype=torch.long)
    for b in range(B):
        n = int(lens[b])
        if n:
            hist[b, L - n:] = torch.randint(1, 80, (n,), generator=gen)
    target = torch.randint(1, 80, (B, 1), generator=gen)
    items = torch.cat([hist, target], dim=1).flatten()
    item_dict = {"item_id": items}
    if "cate_id" in fm.features:
        item_dict["cate_id"] = torch.where(items > 0, items % 11 + 1, torch.zeros_like(items))
    batch_dict = {"user_id": torch.randint(1, 30, (B,), generator=gen),
                  "label": (torch.rand(B, generator=gen) < 0.4).double()}
    return batch_dict, item_dict, (hist > 0).float()


def min_len(model):
    """ETA with k < L: at least k valid items, so that no tie among masked positions crosses the k boundary.  An empty
    history is then covered by the configurations with k >= L, and by SDIM."""
    k = min(getattr(model, "topk", L_HIST), L_HIST)
    return k if k < L_HIST else 0


def item_emb(model, item_dict, B):
    return model.embedding_layer(item_dict, flatten_emb=True).view(B, -1, model.item_info_dim)


def interest(model, name, x, mask, R):
    """The reference's interest block on x with the rotations R (a per-batch draw is fed through torch.randn)."""
    real = torch.randn
    if not model.reuse_hash:
        torch.randn = lambda *a, **k: R.clone()
    try:
        target = x[:, -1, :]
        s = model.short_seq_len
        short = model.short_attention(target, x[:, -s:-1, :], mask[:, -s:-1])
        hist = x[:, 0:-1, :]
        if name == "ETA":
            topk_emb, topk_mask = model.topk_retrieval(model.random_rotations, target, hist, mask, model.topk)
            long = model.long_attention(target, topk_emb, topk_mask)
        else:
            long = model.lsh_attentioin(model.random_rotations, target, hist, mask)
    finally:
        torch.randn = real
    return target, short, long


def eta_positions(model, x, mask, R):
    """The chosen positions as a set, sorted ascending (well_posed makes the set unique)."""
    Rf = R.double().expand(x.shape[0], *R.shape[1:])
    proj = torch.einsum("bld,bdh->blh", x.detach().double(), Rf)
    code = proj > 0
    dist = (code[:, :-1] ^ code[:, -1:]).sum(-1)
    dist = torch.where(mask != 0, dist, torch.full_like(dist, model.hash_bits + 1))
    k = min(model.topk, mask.shape[1])
    key = dist * (mask.shape[1] + 1) + torch.arange(mask.shape[1])     # (distance, position)
    return key.argsort(dim=1)[:, :k].sort(dim=1).values.to(torch.int32)


def case_init(M, name):
    init = {"models": {}}
    for case, kwargs in CASES[name].items():
        fm, model = build(M, name, case, 777)
        init["models"][case] = {"seed": 777, "specs": G.specs_json(fm), "labels": fm.labels, "kwargs": kwargs,
                                "state_dict": digests(model)}
    path = os.path.join(G.HERE, name.lower() + "_init.json")
    with open(path, "w") as fd:
        json.dump(init, fd, indent=1, sort_keys=True)
    print("wrote", path)


def case_next(M, name):
    gen = torch.Generator().manual_seed(61)
    B = 9
    for case in CASES[name]:
        fm, model = build(M, name, case, 71)
        model.train()
        for attempt in range(200):
            with torch.no_grad():
                for m in model.modules():
                    if isinstance(m, torch.nn.Embedding):
                        m.weight[1:].copy_(torch.randn(m.weight[1:].shape, generator=gen) * 0.5)
            _, item_dict, mask = triple(fm, B, L_HIST, gen, min_len(model))
            x = item_emb(model, item_dict, B).detach()
            R = rotations_for(model, B, model.item_info_dim, gen)
            if well_posed(model, x, mask, R):
                break
        else:
            raise RuntimeError("no well-posed draw for %s %s" % (name, case))
        x = x.clone().requires_grad_(True)
        model.zero_grad()
        target, short, long = interest(model, name, x, mask, R)
        gt, gs, gl = (torch.randn(t.shape, generator=gen) for t in (target, short, long))
        ((target * gt).sum() + (short * gs).sum() + (long * gl).sum()).backward()
        att = ("short_attention.", "long_attention.")
        w = {k: v for k, v in G.sd(model).items() if k.startswith(att)}
        g = {k: v for k, v in G.grads(model).items() if k.startswith(att)}
        out = {"target": target, "short": short, "long": long}
        if name == "ETA":
            out["pos"] = eta_positions(model, x, mask, R)
        G.save("next_%s_%s" % (name, case), {"B": B, "L": L_HIST, "case": case, "kwargs": CASES[name][case]},
               **{"in": {"x": x.detach(), "mask": mask, "R": R, "g_target": gt, "g_short": gs, "g_long": gl},
                  "out": out, "w": w, "g": g, "gin": {"x": x.grad}})


def case_models(M, name):
    gen = torch.Generator().manual_seed(67)
    B = 8
    for case, kwargs in CASES[name].items():
        if not kwargs["reuse_hash"]:
            continue
        fm, model = build(M, name, case, 2023)
        model._max_gradient_norm = 10.0
        model._batch_index = 0
        model.train()
        # three batches on which the states of every recorded step keep the block well posed
        for attempt in range(2000):
            with torch.no_grad():
                for m in model.modules():
                    if isinstance(m, torch.nn.Embedding):
                        m.weight[1:].copy_(torch.randn(m.weight[1:].shape, generator=gen) * 0.5)
            state0 = G.sd(model)
            batches = [triple(fm, B, L_HIST, gen, min_len(model)) for _ in range(3)]
            ok = True
            for i in range(3):
                bd, idict, mask = batches[i]
                if not well_posed(model, item_emb(model, dict(idict), B).detach(), mask,
                                  model.random_rotations.detach()):
                    ok = False
                    break
                if i < 2:
                    model.train_step((bd, dict(idict), mask))
            model.load_state_dict(state0)
            model.optimizer = torch.optim.Adam(model.parameters(), lr=1e-3)
            if ok:
                break
        else:
            raise RuntimeError("no well-posed draw for %s %s" % (name, case))
        w0 = G.sd(model)
        model.optimizer.zero_grad()
        bd, idict, mask = batches[0]
        ret = model.forward((bd, dict(idict), mask))
        loss = model.compute_loss(ret, model.get_labels((bd, idict, mask)))
        loss.backward()
        g = G.grads(model)
        outs = {"y_pred": ret["y_pred"], "loss": loss}
        model.optimizer.zero_grad()
        states, losses = {}, []
        for i in range(3):
            losses.append(model.train_step((batches[i][0], dict(batches[i][1]), batches[i][2])).detach())
            if i in (0, 2):
                states[i + 1] = G.sd(model)
        outs["step_losses"] = torch.stack(losses)
        ins = {}
        for i, (bd, idict, mask) in enumerate(batches):
            ins["%d/mask" % i] = mask
            ins["%d/label" % i] = bd["label"]
            ins["%d/user_id" % i] = bd["user_id"]
            for k, v in idict.items():
                ins["%d/%s" % (i, k)] = v
        meta = {"case": case, "kwargs": kwargs, "seed": 2023, "specs": G.specs_json(fm), "labels": fm.labels,
                "batch": B, "L": L_HIST, "item_fields": sorted(batches[0][1].keys())}
        G.save("model_%s_%s" % (name, case), meta,
               **{"in": ins, "w": w0, "out": outs, "g": g, "w1": states[1], "w3": states[3]})


if __name__ == "__main__":
    for name in ("ETA", "SDIM"):
        M = load(name)
        case_init(M, name)
        case_next(M, name)
        case_models(M, name)

"""Generates the MIRRN fixtures by running the REAL reference (model_zoo/LongCTR/MIRRN/MIRRN.py, imported by path),
with make_golden.py's helpers and settings (reference import stubs, one thread, deterministic algorithms) and
make_longctr_golden.py's batch generator, so no other fixture changes.  Run in the build container only:

    python tests/golden/make_mirrn_golden.py

Writes
  mirrn_init.json        state_dict keys, dtypes, shapes and SHA-256 of each tensor right after construction under
                         torch.manual_seed(777), for every configuration below;
  next_MIRRN_<c>.npz     the interest block on a (B, L + 1, d) item_feat_emb leaf: in/x, in/mask, in/R (the rotations
                         the block used: (d, bits), or (3, d, bits) for the three per-call draws target, short,
                         global), in/g_target, in/g_short, in/g_long; out/short, out/long, out/interests (B, 3, d),
                         out/pos (B, 3, k) (the chosen positions, ascending); gin/x; w and g the weights and gradients
                         of the two attentions, pos and the three FilterLayer2 blocks (complex_weight's off-diagonal
                         gradients included, which are zero);
  model_MIRRN_<c>.npz    (reuse_hash=True configurations) the LongCTR triples of three batches (in/<feature>, in/mask,
                         in/label), w the state after construction, out/y_pred and out/loss of batch 0 and g its
                         gradients, w1 / w3 the state after 1 and 3 train_step()s.
Every FilterLayer2's out_dropout.p is set to 0 on the reference instance: its mask is torch's and cannot be replayed.
The maker asserts, for every recorded step, that no SimHash projection of a valid row, the target or a non-empty mean
query lies within 1e-4 |v| |R_j| of its hyperplane, and that no query has a distance tie across its k boundary; it
re-draws the embeddings and the ids until both hold.
"""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_golden as G  # noqa: E402  (imports the reference)
import make_longctr_golden as LG  # noqa: E402

torch = G.torch

COMMON = dict(dnn_hidden_units=[16, 8], dnn_activations="ReLU", attention_dim=8, num_heads=2, use_scale=True,
              net_dropout=0, batch_norm=False, max_len=24)
# name: (kwargs, L)
CASES = {
    "k5_L8_reuse_b16": (dict(embedding_dim=4, reuse_hash=True, hash_bits=16, topk=5, short_seq_len=4, **COMMON), 8),
    "k4_L20_percall_b64": (dict(embedding_dim=4, reuse_hash=False, hash_bits=64, topk=4, short_seq_len=5, **COMMON),
                           20),
    "k2_L20_reuse_b48_one_field": (dict(embedding_dim=8, reuse_hash=True, hash_bits=48, topk=2, short_seq_len=3,
                                       **dict(COMMON, num_heads=1)), 20),
    "k1_L8_percall_b7": (dict(embedding_dim=4, reuse_hash=False, hash_bits=7, topk=1, short_seq_len=3, **COMMON), 8),
    "k12_L6_reuse_b33": (dict(embedding_dim=4, reuse_hash=True, hash_bits=33, topk=12, short_seq_len=4, **COMMON), 6),
}


def specs_of(case):
    return LG.ONE_ITEM_SPECS if case.endswith("one_field") else LG.SPECS


def build(M, case, seed):
    kwargs = CASES[case][0]
    torch.manual_seed(seed)
    fm = G.synthetic_fm(specs_of(case), emb_dim=kwargs["embedding_dim"])
    model = M.MIRRN(fm, **G.model_params(**kwargs))
    for blk in model.MHFT_block:
        blk.out_dropout.p = 0.0
    return fm, model


def rotations_for(model, d, gen):
    """The shared (d, bits) parameter, or three fresh (d, bits) draws (target, short, global) stacked."""
    if model.reuse_hash:
        return model.random_rotations.detach()
    return torch.stack([torch.randn(d, model.hash_bits, generator=gen) for _ in range(3)])


def well_posed(model, x, mask, R):
    x = x.detach().double()
    hist = x[:, :-1] * (mask != 0).unsqueeze(-1).double()
    counts = [(mask[:, -16:] != 0).sum(1), (mask != 0).sum(1)]
    queries = [x[:, -1], hist[:, -16:].sum(1), hist.sum(1)]
    Rs = [R] * 3 if R.dim() == 2 else list(R)
    L = mask.shape[1]
    k = min(model.topk, L)
    for q in range(3):
        Rq = Rs[q].double()
        rn = Rq.norm(dim=0)
        proj = x[:, :-1] @ Rq
        close = (proj.abs() <= 1e-4 * x[:, :-1].norm(dim=-1, keepdim=True) * rn) & (mask != 0).unsqueeze(-1) \
            & (x[:, :-1].norm(dim=-1, keepdim=True) > 0)
        qv = queries[q]
        qp = qv @ Rq
        live = torch.ones(x.shape[0], dtype=torch.bool) if q == 0 else counts[q - 1] > 0
        qclose = (qp.abs() <= 1e-4 * qv.norm(dim=-1, keepdim=True) * rn) & live.unsqueeze(-1)
        if bool(close.any()) or bool(qclose.any()):
            return False
        dist = ((proj > 0) ^ (qp > 0).unsqueeze(1)).sum(-1)
        dist = torch.where(mask != 0, dist, torch.full_like(dist, model.hash_bits + 1))
        if k < L:
            s = dist.sort(dim=1).values
            if bool((s[:, k - 1] == s[:, k]).any()):
                return False
    return True


def positions(model, x, mask, R):
    """(B, 3, k) chosen positions per query, ascending (well_posed makes each set unique)."""
    x = x.detach().double()
    hist = x[:, :-1] * (mask != 0).unsqueeze(-1).double()
    queries = [x[:, -1], hist[:, -16:].sum(1), hist.sum(1)]
    Rs = [R] * 3 if R.dim() == 2 else list(R)
    L = mask.shape[1]
    out = []
    for q in range(3):
        Rq = Rs[q].double()
        dist = (((x[:, :-1] @ Rq) > 0) ^ ((queries[q] @ Rq) > 0).unsqueeze(1)).sum(-1)
        dist = torch.where(mask != 0, dist, torch.full_like(dist, model.hash_bits + 1))
        key = dist * (L + 1) + torch.arange(L)
        out.append(key.argsort(dim=1)[:, :min(model.topk, L)].sort(dim=1).values)
    return torch.stack(out, dim=1).to(torch.int32)


def interest(model, x, mask, R):
    """MIRRN.forward's interest block (MIRRN.py:149-196) on x with the rotations R (per-call draws fed through
    torch.randn in the order target, short, global)."""
    real = torch.randn
    if not model.reuse_hash:
        draws = iter(R.clone())
        torch.randn = lambda *a, **k: next(draws).clone()
    try:
        target = x[:, -1, :]
        s = model.short_seq_len
        short = model.short_attention(target, x[:, -s:-1, :], mask[:, -s:-1])
        seq = x[:, 0:-1, :]
        embs, idxs = [], []
        for query in (target, model.masked_mean(seq[:, -16:], mask[:, -16:], dim=1),
                      model.masked_mean(seq, mask, dim=1)):
            emb, _, idx = model.topk_retrieval(model.random_rotations, query, seq, mask, model.topk)
            embs.append(emb)
            idxs.append(idx)
        ints = []
        for q in range(3):
            emb = embs[q] + model.pos(seq.shape[1] - idxs[q]) * 0.02
            ints.append(model.MHFT_block[q](emb).mean(1))
        interests = torch.stack(ints, 1)
        long = model.long_attention(target, interests)
    finally:
        torch.randn = real
    return target, short, long, interests


def case_init(M):
    init = {"models": {}}
    for case, (kwargs, _) in CASES.items():
        fm, model = build(M, case, 777)
        init["models"][case] = {"seed": 777, "specs": G.specs_json(fm), "labels": fm.labels, "kwargs": kwargs,
                                "state_dict": LG.digests(model)}
    path = os.path.join(G.HERE, "mirrn_init.json")
    with open(path, "w") as fd:
        json.dump(init, fd, indent=1, sort_keys=True)
    print("wrote", path)


def min_len(model, L):
    """With k < L at least k valid items, so that no tie among masked positions crosses the k boundary; an empty
    history is covered by the configuration with k >= L."""
    k = min(model.topk, L)
    return k if k < L else 0


def _perturb(model, gen):
    with torch.no_grad():
        for m in model.modules():
            if isinstance(m, torch.nn.Embedding) and m is not model.pos:
                m.weight[1:].copy_(torch.randn(m.weight[1:].shape, generator=gen) * 0.5)
        for blk in model.MHFT_block:     # filter weights large enough that the filter shows in the outputs
            blk.complex_weight.copy_(torch.randn(blk.complex_weight.shape, generator=gen) * 0.5)
            blk.LayerNorm.weight.copy_(1 + 0.2 * torch.randn(blk.LayerNorm.weight.shape, generator=gen))
            blk.LayerNorm.bias.copy_(0.1 * torch.randn(blk.LayerNorm.bias.shape, generator=gen))


def case_next(M):
    gen = torch.Generator().manual_seed(61)
    B = 6
    for case, (kwargs, L) in CASES.items():
        fm, model = build(M, case, 71)
        model.train()
        for attempt in range(5000):
            _perturb(model, gen)
            _, item_dict, mask = LG.triple(fm, B, L, gen, min_len(model, L))
            x = LG.item_emb(model, item_dict, B).detach()
            R = rotations_for(model, model.item_info_dim, gen)
            if well_posed(model, x, mask, R):
                break
        else:
            raise RuntimeError("no well-posed draw for MIRRN %s" % case)
        x = x.clone().requires_grad_(True)
        model.zero_grad()
        target, short, long, interests = interest(model, x, mask, R)
        gt, gs, gl = (torch.randn(t.shape, generator=gen) for t in (target, short, long))
        ((target * gt).sum() + (short * gs).sum() + (long * gl).sum()).backward()
        keep = ("short_attention.", "long_attention.", "pos.", "MHFT_block.")
        w = {k: v for k, v in G.sd(model).items() if k.startswith(keep)}
        g = {k: v for k, v in G.grads(model).items() if k.startswith(keep)}
        out = {"target": target, "short": short, "long": long, "interests": interests,
               "pos": positions(model, x, mask, R)}
        G.save("next_MIRRN_%s" % case, {"B": B, "L": L, "case": case, "kwargs": kwargs},
               **{"in": {"x": x.detach(), "mask": mask, "R": R, "g_target": gt, "g_short": gs, "g_long": gl},
                  "out": out, "w": w, "g": g, "gin": {"x": x.grad}})


def case_models(M):
    gen = torch.Generator().manual_seed(67)
    B = 6
    for case, (kwargs, L) in CASES.items():
        if not kwargs["reuse_hash"]:
            continue
        fm, model = build(M, case, 2023)
        model._max_gradient_norm = 10.0
        model._batch_index = 0
        model.train()
        # each batch drawn until the block is well posed at the state the steps before it leave
        _perturb(model, gen)
        state0 = G.sd(model)
        batches = []
        for i in range(3):
            for attempt in range(5000):
                bd, idict, mask = LG.triple(fm, B, L, gen, min_len(model, L))
                if well_posed(model, LG.item_emb(model, dict(idict), B).detach(), mask,
                              model.random_rotations.detach()):
                    break
            else:
                raise RuntimeError("no well-posed draw for MIRRN %s" % case)
            batches.append((bd, idict, mask))
            if i < 2:
                model.train_step((bd, dict(idict), mask))
        model.load_state_dict(state0)
        model.optimizer = torch.optim.Adam(model.parameters(), lr=1e-3)
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
                "batch": B, "L": L, "item_fields": sorted(batches[0][1].keys())}
        G.save("model_MIRRN_%s" % case, meta, **{"in": ins, "w": w0, "out": outs, "g": g, "w1": states[1],
                                                 "w3": states[3]})


if __name__ == "__main__":
    M = LG.load("MIRRN")
    case_init(M)
    case_next(M)
    case_models(M)

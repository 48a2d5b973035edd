"""Generates the SIM and TWIN fixtures by running the REAL reference (model_zoo/LongCTR/SIM/SIM.py and
model_zoo/LongCTR/TWIN/TWIN.py, imported by path), with make_golden.py's and make_longctr_golden.py's helpers and
settings (reference import stubs, one thread, deterministic algorithms, the LongCTR triples), so no other fixture
changes.  Run in the build container only:

    python tests/golden/make_sim_twin_golden.py

Writes
  sim_init.json / twin_init.json   state_dict keys, dtypes, shapes and SHA-256 of each tensor right after construction
                                   under torch.manual_seed(777), for every configuration below;
  next_<SIM|TWIN>_<c>.npz          the interest block of the reference's own forward on a (B, L + 1, d) item_feat_emb
                                   leaf (fed through a hook on embedding_layer; the blocks' outputs are read off the
                                   DNN inputs): in/x, in/mask, in/g_target, in/g_short, in/g_long (SIM: in/g_pooled);
                                   out/short, out/long (SIM: out/pooled), out/pos (the chosen positions, sorted
                                   ascending; TWIN (B, H, k)); gin/x; w and g every interest weight and its gradient;
  model_<SIM|TWIN>_<c>.npz         the LongCTR triples of three batches (in/<feature>, in/mask, in/label), w the state
                                   after construction, out/y_pred (SIM: out/y_aux) and out/loss of batch 0 and g its
                                   gradients, w1 / w3 the state after 1 and 3 train_step()s.
Each batch holds a full history (row 1) and a shortest one (row 0): empty where k >= L, else exactly k items; the rest
are pre-padded with random lengths.  Padding ids embed to zero rows.  The maker re-draws the embeddings and ids until,
on every recorded step, no valid score lies within 1e-4 of the largest |score| of its row (per head) of the k-th
selected one, and no SIM valid score lies that near 0: the reference's CPU topk then picks a well-defined set.  A SIM
row may still hold fewer positive valid scores than k, and then its masked rows (score 0) fill the selection.
"""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_golden as G  # noqa: E402  (imports the reference)
import make_longctr_golden as LG  # noqa: E402

torch = G.torch

COMMON = dict(dnn_hidden_units=[16, 8], dnn_activations="ReLU", attention_dim=8, net_dropout=0, batch_norm=False)
CASES = {
    "SIM": {
        "h2_k5": dict(embedding_dim=4, num_heads=2, topk=5, short_seq_len=4, alpha=0.7, beta=1.3, **COMMON),
        "h1_k8_one_field": dict(embedding_dim=8, num_heads=1, topk=8, short_seq_len=5, alpha=1, beta=1, **COMMON),
        "h2_k12": dict(embedding_dim=4, num_heads=2, topk=12, short_seq_len=3, alpha=1.5, beta=0.5, **COMMON),
    },
    "TWIN": {
        "h2_k5": dict(embedding_dim=4, num_heads=2, topk=5, short_seq_len=4, **COMMON),
        "h1_k8_one_field": dict(embedding_dim=8, num_heads=1, topk=8, short_seq_len=5, **COMMON),
        "h2_k12": dict(embedding_dim=4, num_heads=2, topk=12, short_seq_len=3, **COMMON),
    },
}
L_HIST = LG.L_HIST
MARGIN = 1e-4


def specs_of(case):
    return LG.ONE_ITEM_SPECS if case.endswith("one_field") else LG.SPECS


def build(M, name, case, seed):
    kwargs = CASES[name][case]
    torch.manual_seed(seed)
    fm = G.synthetic_fm(specs_of(case), emb_dim=kwargs["embedding_dim"])
    return fm, getattr(M, name)(fm, **G.model_params(**kwargs))


def scores(model, name, x, mask):
    """Float64 scores (SIM (B, 1, L), masked 0; TWIN (B, H, L), masked -1e9) from the model's weights."""
    x = x.detach().double()
    t, hist = x[:, -1], x[:, :-1]
    B, L, _ = hist.shape
    if name == "SIM":
        qk = torch.einsum("ba,bla->bl", t @ model.W_a.weight.double().t(), hist @ model.W_b.weight.double().t())
        return (qk * mask.double()).unsqueeze(1)
    att = model.long_attention
    H, hd = att.num_heads, att.head_dim
    q = (t @ att.W_q.weight.double().t()).view(B, H, 1, hd)
    k = (hist @ att.W_h.weight.double().t()).view(B, L, H, hd).transpose(1, 2)
    s = (q @ k.transpose(-1, -2)).squeeze(2) / hd ** 0.5
    return s.masked_fill(mask.view(B, 1, L) == 0, -1e9)


def well_posed(model, name, x, mask):
    s = scores(model, name, x, mask)
    valid = (mask != 0).unsqueeze(1).expand_as(s)
    scale = s.masked_fill(~valid, 0).abs().amax(dim=-1, keepdim=True).clamp_min(1e-12)
    if name == "SIM" and bool(((s.abs() <= MARGIN * scale) & valid).any()):
        return False
    k = min(model.topk, mask.shape[1])
    if k < mask.shape[1]:
        srt = s.sort(dim=-1, descending=True).values
        if bool(((srt[..., k - 1] - srt[..., k]).abs() <= MARGIN * scale[..., 0]).any()):
            return False
    return True


def positions(model, name, x, mask):
    """The chosen positions as a set, sorted ascending (well_posed makes the set unique); SIM (B, k), TWIN (B, H, k)."""
    s = scores(model, name, x, mask)
    k = min(model.topk, mask.shape[1])
    pos = s.argsort(dim=-1, descending=True)[..., :k].sort(dim=-1).values.to(torch.int32)
    return pos[:, 0] if name == "SIM" else pos


def min_len(model):
    k = min(model.topk, L_HIST)
    return k if k < L_HIST else 0


def run_forward(model, name, x, triple):
    """The reference's forward on the triple with item_feat_emb replaced by the leaf x; returns (ret, target, short,
    long, pooled or None), the blocks' outputs read off the DNN inputs."""
    bd, idict, mask = triple
    B, d = mask.shape[0], model.item_info_dim
    seen = {}

    def emb_hook(mod, args, out):
        return x.reshape(out.shape) if out.shape[0] == x.shape[0] * x.shape[1] else out

    def grab(key):
        def hook(mod, args):
            seen[key] = args[0]
        return hook
    hooks = [model.embedding_layer.register_forward_hook(emb_hook),
             model.dnn.register_forward_pre_hook(grab("dnn"))]
    if name == "SIM":
        hooks.append(model.dnn_aux.register_forward_pre_hook(grab("aux")))
    try:
        ret = model.forward((bd, dict(idict), mask))
    finally:
        for h in hooks:
            h.remove()
    h = seen["dnn"]
    target, short, long = h[:, -3 * d:-2 * d], h[:, -2 * d:-d], h[:, -d:]
    pooled = seen["aux"][:, -d:] if name == "SIM" else None
    return ret, target, short, long, pooled


def case_init(M, name):
    init = {"models": {}}
    for case, kwargs in CASES[name].items():
        fm, model = build(M, name, case, 777)
        init["models"][case] = {"seed": 777, "specs": G.specs_json(fm), "labels": fm.labels, "kwargs": kwargs,
                                "state_dict": LG.digests(model)}
    path = os.path.join(G.HERE, name.lower() + "_init.json")
    with open(path, "w") as fd:
        json.dump(init, fd, indent=1, sort_keys=True)
    print("wrote", path)


def _redraw_tables(model, gen):
    with torch.no_grad():
        for m in model.modules():
            if isinstance(m, torch.nn.Embedding):
                m.weight[1:].copy_(torch.randn(m.weight[1:].shape, generator=gen) * 0.5)


def case_next(M, name):
    gen = torch.Generator().manual_seed(61)
    B = 9
    for case in CASES[name]:
        fm, model = build(M, name, case, 71)
        model.train()
        for attempt in range(500):
            _redraw_tables(model, gen)
            triple = LG.triple(fm, B, L_HIST, gen, min_len(model))
            x = LG.item_emb(model, dict(triple[1]), B).detach()
            if well_posed(model, name, x, triple[2]):
                break
        else:
            raise RuntimeError("no well-posed draw for %s %s" % (name, case))
        mask = triple[2]
        x = x.clone().requires_grad_(True)
        model.zero_grad()
        _, target, short, long, pooled = run_forward(model, name, x, triple)
        outs = {"target": target, "short": short, "long": long}
        if pooled is not None:
            outs["pooled"] = pooled
        gouts = {k: torch.randn(v.shape, generator=gen) for k, v in outs.items()}
        sum((outs[k] * gouts[k]).sum() for k in outs).backward()
        keep = ("W_a.", "W_b.", "short_attention.", "long_attention.")
        w = {k: v for k, v in G.sd(model).items() if k.startswith(keep)}
        g = {k: v for k, v in G.grads(model).items() if k.startswith(keep)}
        out = {k: v.detach() for k, v in outs.items()}
        out["pos"] = positions(model, name, x, mask)
        G.save("next_%s_%s" % (name, case), {"B": B, "L": L_HIST, "case": case, "kwargs": CASES[name][case]},
               **{"in": dict({"x": x.detach(), "mask": mask}, **{"g_" + k: v for k, v in gouts.items()}),
                  "out": out, "w": w, "g": g, "gin": {"x": x.grad}})


def case_models(M, name):
    gen = torch.Generator().manual_seed(67)
    B = 8
    for case, kwargs in CASES[name].items():
        fm, model = build(M, name, case, 2023)
        model._max_gradient_norm = 10.0
        model._batch_index = 0
        model.train()
        for attempt in range(2000):
            _redraw_tables(model, gen)
            state0 = G.sd(model)
            batches = [LG.triple(fm, B, L_HIST, gen, min_len(model)) for _ in range(3)]
            ok = True
            for i in range(3):
                bd, idict, mask = batches[i]
                if not well_posed(model, name, LG.item_emb(model, dict(idict), B).detach(), mask):
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
        if "y_aux" in ret:
            outs["y_aux"] = ret["y_aux"]
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
    for name in ("SIM", "TWIN"):
        M = LG.load(name)
        case_init(M, name)
        case_next(M, name)
        case_models(M, name)

"""Generates the WuKong fixtures by running the REAL reference (model_zoo/WuKong), with make_golden.py's helpers and
settings (reference import stubs, one thread, deterministic algorithms) and its own generators, so no other fixture
changes.  Run in the build container only:

    python tests/golden/make_wukong_golden.py

Writes
  wukong_init.json        state_dict keys, dtypes, shapes and the SHA-256 of each tensor of the reference's WuKongLayer
                          right after construction under torch.manual_seed(4747), for five configurations (projection
                          residual, identity residual, layer_norm=False, empty fmb_mlp_units, dropout); and of WuKong
                          on a 6-field map right after construction (which ends in reset_parameters) under
                          torch.manual_seed(777), for the three model configurations below;
  next_WuKongLayer.npz    forward output, input gradient and every parameter gradient of three layers: F 5 -> 6 with a
                          projection, F 6 -> 6 with the identity, F 7 -> 5 without the output LayerNorm; every LayerNorm
                          weight and bias drawn away from 1 and 0 (groups w_<c>, g_<c>; in/x_<c>, in/gout_<c>,
                          out/y_<c>, gin/x_<c>);
  model_WuKong_bn.npz, model_WuKong_nobn.npz, model_WuKong_noln.npz
                          make_golden.run_model_case on the reference models (10-field map): inputs, weights,
                          y_pred, loss, gradients, the state after 1 and 3 train_step()s.
"""
import hashlib
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_golden as G  # noqa: E402  (imports the reference)

torch = G.torch

# (name, input_features, lcb, fmb, embedding_dim, rank_k, fmb_mlp_units, fmb_dropout, layer_norm)
LAYER_INIT = [("proj", 5, 3, 4, 8, 3, [16], 0.0, True), ("identity", 8, 4, 4, 8, 4, [16, 8], 0.0, True),
              ("noln", 6, 2, 3, 4, 2, [8], 0.0, False), ("nomlp", 6, 3, 3, 4, 2, [], 0.0, True),
              ("dropout", 6, 3, 3, 4, 2, [8, 8], 0.2, True)]
LAYER_CASES = [("proj", 5, 2, 4, 8, 3, [12], True), ("identity", 6, 3, 3, 4, 4, [8, 8], True),
               ("noln", 7, 2, 3, 5, 2, [], False)]
MODEL_KWARGS = {
    "bn": dict(embedding_dim=8, num_wukong_layers=3, lcb_features=4, fmb_features=4, fmb_mlp_units=[16, 16],
               fmp_rank_k=4, mlp_hidden_units=[16, 16], mlp_batch_norm=True),
    "nobn": dict(embedding_dim=8, num_wukong_layers=2, lcb_features=6, fmb_features=4, fmb_mlp_units=[24],
                 fmp_rank_k=3, mlp_hidden_units=[16], mlp_batch_norm=False),
    "noln": dict(embedding_dim=4, num_wukong_layers=2, lcb_features=3, fmb_features=5, fmb_mlp_units=[16],
                 fmp_rank_k=2, mlp_hidden_units=[12, 8], mlp_batch_norm=False, layer_norm=False),
}


def wukong_module():
    cls = G.load_model_class("WuKong", "WuKong")
    return sys.modules[cls.__module__]


def digests(module):
    return [[k, str(v.dtype), list(v.shape), hashlib.sha256(v.detach().contiguous().numpy().tobytes()).hexdigest()]
            for k, v in module.state_dict().items()]


def layer_norms(layer, gen):
    with torch.no_grad():
        for m in layer.modules():
            if isinstance(m, torch.nn.LayerNorm):
                m.weight.copy_(torch.rand(m.weight.shape, generator=gen) + 0.5)
                m.bias.copy_(torch.rand(m.bias.shape, generator=gen) * 0.6 - 0.3)


def case_init(M):
    init = {"layers": {}, "models": {}}
    for (name, nf, lcb, fmb, D, k, units, p, ln) in LAYER_INIT:
        torch.manual_seed(4747)
        m = M.WuKongLayer(nf, lcb, fmb, D, k, units, "relu", p, ln)
        init["layers"][name] = {"args": [nf, lcb, fmb, D, k, units, p, ln], "seed": 4747, "state_dict": digests(m)}
    specs = G.criteo_like_specs(6, 20)
    for name, kwargs in MODEL_KWARGS.items():
        torch.manual_seed(777)
        fm = G.synthetic_fm(specs, emb_dim=kwargs["embedding_dim"])
        model = M.WuKong(fm, **G.model_params(**kwargs))
        init["models"][name] = {"seed": 777, "specs": G.specs_json(fm), "labels": fm.labels, "kwargs": kwargs,
                                "state_dict": digests(model)}
    path = os.path.join(G.HERE, "wukong_init.json")
    with open(path, "w") as fd:
        json.dump(init, fd, indent=1, sort_keys=True)
    print("wrote", path)


def case_layer(M):
    gen = torch.Generator().manual_seed(81)
    B = 6
    groups = {"in": {}, "out": {}, "gin": {}}
    for (c, nf, lcb, fmb, D, k, units, ln) in LAYER_CASES:
        torch.manual_seed(81)
        layer = M.WuKongLayer(nf, lcb, fmb, D, k, units, "relu", 0.0, ln)
        layer_norms(layer, gen)
        x = (torch.randn(B, nf, D, generator=gen) * 0.7).requires_grad_(True)
        groups["w_" + c] = G.sd(layer)
        out = layer(x)
        gout = torch.randn(out.shape, generator=gen)
        (out * gout).sum().backward()
        groups["in"]["x_" + c], groups["in"]["gout_" + c] = x.detach(), gout
        groups["out"]["y_" + c] = out
        groups["gin"]["x_" + c] = x.grad
        groups["g_" + c] = G.grads(layer)
    G.save("next_WuKongLayer", {"B": B, "cases": [list(c) for c in LAYER_CASES]}, **groups)


def case_models(M):
    gen = torch.Generator().manual_seed(83)
    for name, kwargs in MODEL_KWARGS.items():
        torch.manual_seed(2023)
        fm = G.synthetic_fm(G.criteo_like_specs(10, 40), emb_dim=kwargs["embedding_dim"])
        model = M.WuKong(fm, **G.model_params(**kwargs))
        with torch.no_grad():
            for m in model.modules():
                if isinstance(m, torch.nn.Embedding):
                    m.weight[1:].copy_(torch.randn(m.weight[1:].shape, generator=gen) * 0.3)
        mat = G.synthetic_matrix(fm, 3 * 32, gen)
        G.run_model_case("model_WuKong_" + name, model, fm, mat, {"case": name, "kwargs": kwargs, "seed": 2023})


if __name__ == "__main__":
    M = wukong_module()
    case_init(M)
    case_layer(M)
    case_models(M)

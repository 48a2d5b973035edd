"""Generates the AutoInt fixtures by running the REAL reference (model_zoo/AutoInt), with make_golden.py's helpers and
settings (reference import stubs, one thread, deterministic algorithms) and its own generators, so no other fixture
changes.  Run in the build container only:

    python tests/golden/make_autoint_golden.py

Writes
  autoint_init.json       state_dict keys, dtypes, shapes and the SHA-256 of each tensor of the reference's
                          MultiHeadSelfAttention right after construction under torch.manual_seed(4747), for five
                          configurations (W_res, identity residual, use_residual=False, layer_norm, dropout); and of
                          AutoInt on a 6-field map right after construction (which ends in reset_parameters) under
                          torch.manual_seed(777), for the three model configurations below;
  next_MultiHeadSelfAttention.npz
                          forward output, input gradient and every parameter gradient of three layers: d_in 4 != A 8
                          with 2 heads (W_res); A 12 with 3 heads and use_scale; A 10 with 2 heads and layer_norm, its
                          weight and bias drawn away from 1 and 0 (groups w_<c>, g_<c>; in/x_<c>, in/gout_<c>,
                          out/y_<c>, gin/x_<c>);
  model_AutoInt_test.npz, model_AutoInt_wide.npz, model_AutoInt_nodnn.npz
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

# (name, input_dim, attention_dim, num_heads, dropout_rate, use_residual, use_scale, layer_norm)
LAYER_INIT = [("wres", 4, 8, 2, 0.0, True, False, False), ("identity", 16, 16, 2, 0.0, True, False, False),
              ("nores", 4, 8, 2, 0.0, False, False, False), ("ln", 10, 10, 2, 0.0, True, True, True),
              ("dropout", 8, 8, 1, 0.2, True, True, False)]
LAYER_CASES = [("wres", 4, 8, 2, True, False, False), ("h3_scale", 12, 12, 3, True, True, False),
               ("ln", 10, 10, 2, True, False, True)]
MODEL_KWARGS = {
    "test": dict(embedding_dim=4, attention_dim=8, num_heads=2, attention_layers=3, dnn_hidden_units=[64, 32]),
    "wide": dict(embedding_dim=8, attention_dim=8, num_heads=2, attention_layers=2, dnn_hidden_units=[24, 16],
                 use_wide=True, layer_norm=True, use_scale=True),
    "nodnn": dict(embedding_dim=4, attention_dim=12, num_heads=3, attention_layers=2, dnn_hidden_units=[]),
}


def autoint_module():
    cls = G.load_model_class("AutoInt", "AutoInt")
    return sys.modules[cls.__module__]


def digests(module):
    return [[k, str(v.dtype), list(v.shape), hashlib.sha256(v.detach().contiguous().numpy().tobytes()).hexdigest()]
            for k, v in module.state_dict().items()]


def case_init(M):
    init = {"layers": {}, "models": {}}
    for (name, din, A, H, p, res, scale, ln) in LAYER_INIT:
        torch.manual_seed(4747)
        m = M.MultiHeadSelfAttention(din, attention_dim=A, num_heads=H, dropout_rate=p, use_residual=res,
                                     use_scale=scale, layer_norm=ln)
        init["layers"][name] = {"args": [din, A, H, p, res, scale, ln], "seed": 4747, "state_dict": digests(m)}
    specs = G.criteo_like_specs(6, 20)
    for name, kwargs in MODEL_KWARGS.items():
        torch.manual_seed(777)
        fm = G.synthetic_fm(specs, emb_dim=kwargs["embedding_dim"])
        model = M.AutoInt(fm, **G.model_params(**kwargs))
        init["models"][name] = {"seed": 777, "specs": G.specs_json(fm), "labels": fm.labels, "kwargs": kwargs,
                                "state_dict": digests(model)}
    path = os.path.join(G.HERE, "autoint_init.json")
    with open(path, "w") as fd:
        json.dump(init, fd, indent=1, sort_keys=True)
    print("wrote", path)


def case_layer(M):
    gen = torch.Generator().manual_seed(81)
    B, F = 6, 5
    groups = {"in": {}, "out": {}, "gin": {}}
    for (c, din, A, H, res, scale, ln) in LAYER_CASES:
        torch.manual_seed(81)
        layer = M.MultiHeadSelfAttention(din, attention_dim=A, num_heads=H, use_residual=res, use_scale=scale,
                                         layer_norm=ln)
        if ln:
            with torch.no_grad():
                layer.layer_norm.weight.copy_(torch.rand(A, generator=gen) + 0.5)
                layer.layer_norm.bias.copy_(torch.rand(A, generator=gen) * 0.6 - 0.3)
        x = (torch.randn(B, F, din, generator=gen) * 0.7).requires_grad_(True)
        groups["w_" + c] = G.sd(layer)
        out = layer(x)
        gout = torch.randn(out.shape, generator=gen)
        (out * gout).sum().backward()
        groups["in"]["x_" + c], groups["in"]["gout_" + c] = x.detach(), gout
        groups["out"]["y_" + c] = out
        groups["gin"]["x_" + c] = x.grad
        groups["g_" + c] = G.grads(layer)
    cases = [list(c) for c in LAYER_CASES]
    G.save("next_MultiHeadSelfAttention", {"B": B, "F": F, "cases": cases}, **groups)


def case_models(M):
    gen = torch.Generator().manual_seed(83)
    for name, kwargs in MODEL_KWARGS.items():
        torch.manual_seed(2023)
        fm = G.synthetic_fm(G.criteo_like_specs(10, 40), emb_dim=kwargs["embedding_dim"])
        model = M.AutoInt(fm, **G.model_params(**kwargs))
        with torch.no_grad():
            for m in model.modules():
                if isinstance(m, torch.nn.Embedding):
                    m.weight[1:].copy_(torch.randn(m.weight[1:].shape, generator=gen) * 0.3)
        mat = G.synthetic_matrix(fm, 3 * 32, gen)
        G.run_model_case("model_AutoInt_" + name, model, fm, mat, {"case": name, "kwargs": kwargs, "seed": 2023})


if __name__ == "__main__":
    M = autoint_module()
    case_init(M)
    case_layer(M)
    case_models(M)

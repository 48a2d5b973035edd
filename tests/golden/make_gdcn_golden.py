"""Generates the GDCN fixtures by running the REAL reference (model_zoo/GDCN), with make_golden.py's helpers and
settings (reference import stubs, one thread, deterministic algorithms) and its own generators, so no other fixture
changes.  Run in the build container only:

    python tests/golden/make_gdcn_golden.py

Writes
  gdcn_init.json          state_dict keys, dtypes, shapes and the SHA-256 of each tensor of the reference's
                          GateCorssLayer right after construction under torch.manual_seed(4747), for four
                          (input_dim, cn_layers); and of GDCN and GDCNP on a 6-field map right after construction
                          (which ends in reset_parameters) under torch.manual_seed(777);
  next_GateCorssLayer.npz forward output, input gradient and every parameter gradient of a 3-layer GateCorssLayer
                          at d 20 and d 13 (groups w_d<d>, g_d<d>; in/x_d<d>, in/gout_d<d>, out/y_d<d>, gin/x_d<d>);
  model_GDCN.npz, model_GDCNP.npz
                          make_golden.run_model_case on the reference models (10-field map): inputs, weights,
                          y_pred, loss, gradients, the state after 1 and 3 train_step()s.  GDCN's kwargs carry the
                          GDCN_test YAML's `crossing_layers`, which the reference ignores (3 layers are built).
"""
import hashlib
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_golden as G  # noqa: E402  (imports the reference)

torch = G.torch

LAYER_CONFIGS = [(20, 3), (13, 1), (40, 2), (624, 3)]          # (input_dim, cn_layers)
MODEL_KWARGS = {
    "GDCN": dict(embedding_dim=4, dnn_hidden_units=[24, 16], dnn_activations="relu", crossing_layers=5),
    "GDCNP": dict(embedding_dim=4, dnn_hidden_units=[24, 16], dnn_activations="relu", num_cross_layers=2),
}


def gdcn_module():
    cls = G.load_model_class("GDCN", "GDCN")
    return sys.modules[cls.__module__]


def digests(module):
    return [[k, str(v.dtype), list(v.shape), hashlib.sha256(v.detach().contiguous().numpy().tobytes()).hexdigest()]
            for k, v in module.state_dict().items()]


def case_init(M):
    init = {"layers": {}, "models": {}}
    for (d, nl) in LAYER_CONFIGS:
        torch.manual_seed(4747)
        init["layers"]["d%d_L%d" % (d, nl)] = {"args": [d, nl], "seed": 4747,
                                               "state_dict": digests(M.GateCorssLayer(d, nl))}
    specs = G.criteo_like_specs(6, 20)
    for name, kwargs in MODEL_KWARGS.items():
        torch.manual_seed(777)
        fm = G.synthetic_fm(specs, emb_dim=4)
        model = getattr(M, name)(fm, **G.model_params(**dict(kwargs, embedding_dim=4)))
        init["models"][name] = {"seed": 777, "specs": G.specs_json(fm), "labels": fm.labels,
                                "kwargs": dict(kwargs, embedding_dim=4), "state_dict": digests(model)}
    path = os.path.join(G.HERE, "gdcn_init.json")
    with open(path, "w") as fd:
        json.dump(init, fd, indent=1, sort_keys=True)
    print("wrote", path)


def case_layer(M):
    gen = torch.Generator().manual_seed(71)
    B, nl = 6, 3
    groups = {"in": {}, "out": {}, "gin": {}}
    for d in (20, 13):
        torch.manual_seed(71)
        layer = M.GateCorssLayer(d, nl)
        x = (torch.randn(B, d, generator=gen) * 0.7).requires_grad_(True)
        groups["w_d%d" % d] = G.sd(layer)
        out = layer(x)
        gout = torch.randn(out.shape, generator=gen)
        (out * gout).sum().backward()
        groups["in"]["x_d%d" % d], groups["in"]["gout_d%d" % d] = x.detach(), gout
        groups["out"]["y_d%d" % d] = out
        groups["gin"]["x_d%d" % d] = x.grad
        groups["g_d%d" % d] = G.grads(layer)
    G.save("next_GateCorssLayer", {"B": B, "cn_layers": nl, "dims": [20, 13]}, **groups)


def case_models(M):
    gen = torch.Generator().manual_seed(73)
    for name, kwargs in MODEL_KWARGS.items():
        torch.manual_seed(2023)
        fm = G.synthetic_fm(G.criteo_like_specs(10, 40), emb_dim=4)
        model = getattr(M, name)(fm, **G.model_params(**kwargs))
        with torch.no_grad():
            for m in model.modules():
                if isinstance(m, torch.nn.Embedding):
                    m.weight[1:].copy_(torch.randn(m.weight[1:].shape, generator=gen) * 0.1)
        mat = G.synthetic_matrix(fm, 3 * 32, gen)
        G.run_model_case("model_" + name, model, fm, mat, {"case": name, "kwargs": kwargs, "seed": 2023})


if __name__ == "__main__":
    M = gdcn_module()
    case_init(M)
    case_layer(M)
    case_models(M)

"""Generates the FinalMLP fixtures by running the REAL reference (model_zoo/FinalMLP), with make_golden.py's helpers
and settings (reference import stubs, one thread, deterministic algorithms) and its own generators, so no other
fixture changes.  Run in the build container only:

    python tests/golden/make_finalmlp_golden.py

Writes
  finalmlp_init.json       state_dict keys, dtypes, shapes and the SHA-256 of each tensor right after construction:
                           the reference's InteractionAggregation under torch.manual_seed(4747) for AGG_CONFIGS, its
                           FeatureSelection (with and without context) under torch.manual_seed(4848), and every
                           model of MODEL_CASES on a 6-field map (construction ends in reset_parameters) under
                           torch.manual_seed(777);
  next_InteractionAggregation.npz
                           forward output and every gradient of InteractionAggregation (output_dim 1) for AGG_CONFIGS
                           (groups w_<tag>, g_<tag>; in/x_<tag>, in/y_<tag>, in/gout_<tag>, out/<tag>, gin/x_<tag>,
                           gin/y_<tag>);
  next_FeatureSelection.npz
                           both streams and every gradient of FeatureSelection without and with context features on
                           a 10-field map (tags noctx, ctx; in/matrix holds the batch, in/emb_<tag> the flattened
                           embedding fed in, in/gout1_<tag>, in/gout2_<tag> the streams' upstream gradients);
  model_<case>.npz         make_golden.run_model_case on the reference models of MODEL_CASES (10-field map): inputs,
                           weights, y_pred, loss, gradients, the state after 1 and 3 train_step()s.
"""
import hashlib
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_golden as G  # noqa: E402  (imports the reference)

torch = G.torch

# (tag, x_dim, y_dim, num_heads): head widths 12 | 20, 13 | 7, 10 | 6 and 32 | 16
AGG_CONFIGS = [("h1", 20, 12, 1), ("h2", 26, 14, 2), ("h3", 30, 18, 3), ("h2w", 64, 32, 2)]
FS_CONTEXTS = {"noctx": ([], []), "ctx": (["C0"], ["C1", "C2"])}
MODEL_CASES = {
    "FinalMLP": ("FinalMLP", dict(embedding_dim=4, mlp1_hidden_units=[24, 16], mlp2_hidden_units=[32, 24, 12],
                                  fs_hidden_units=[16, 8], num_heads=2)),
    # FinalMLP_test's layout: one context field for the first gate, two for the second
    "FinalMLP_ctx": ("FinalMLP", dict(embedding_dim=4, mlp1_hidden_units=[24, 16], mlp2_hidden_units=[32, 24, 12],
                                      fs_hidden_units=[16, 16], fs1_context=["C0"], fs2_context=["C1", "C2"],
                                      num_heads=2)),
    "FinalMLP_nofs": ("FinalMLP", dict(embedding_dim=4, mlp1_hidden_units=[24, 16], mlp2_hidden_units=[20, 12],
                                       use_fs=False, num_heads=4)),
    "DualMLP": ("DualMLP", dict(embedding_dim=4, mlp1_hidden_units=[24, 16], mlp2_hidden_units=[32, 16, 8])),
}


def finalmlp_module():
    cls = G.load_model_class("FinalMLP", "FinalMLP")
    return sys.modules[cls.__module__]


def model_class(cls_name):
    return G.load_model_class("FinalMLP", cls_name)


def digests(module):
    return [[k, str(v.dtype), list(v.shape), hashlib.sha256(v.detach().contiguous().numpy().tobytes()).hexdigest()]
            for k, v in module.state_dict().items()]


def case_init(M):
    init = {"aggregation": {}, "feature_selection": {}, "models": {}}
    for tag, dx, dy, h in AGG_CONFIGS:
        torch.manual_seed(4747)
        init["aggregation"][tag] = {"args": [dx, dy, 1, h], "seed": 4747,
                                    "state_dict": digests(M.InteractionAggregation(dx, dy, output_dim=1, num_heads=h))}
    specs = G.criteo_like_specs(6, 20)
    fm = G.synthetic_fm(specs, emb_dim=4)
    for tag, (c1, c2) in FS_CONTEXTS.items():
        torch.manual_seed(4848)
        args = [24, 4, [16, 8], c1, c2]
        init["feature_selection"][tag] = {"args": args, "seed": 4848, "specs": G.specs_json(fm), "labels": fm.labels,
                                          "state_dict": digests(M.FeatureSelection(fm, *args))}
    for case, (cls_name, kwargs) in MODEL_CASES.items():
        torch.manual_seed(777)
        fm = G.synthetic_fm(specs, emb_dim=4)
        model = model_class(cls_name)(fm, **G.model_params(**kwargs))
        init["models"][case] = {"model": cls_name, "seed": 777, "specs": G.specs_json(fm), "labels": fm.labels,
                                "kwargs": kwargs, "state_dict": digests(model)}
    path = os.path.join(G.HERE, "finalmlp_init.json")
    with open(path, "w") as fd:
        json.dump(init, fd, indent=1, sort_keys=True)
    print("wrote", path)


def case_aggregation(M):
    gen = torch.Generator().manual_seed(81)
    B = 7
    groups = {"in": {}, "out": {}, "gin": {}}
    for tag, dx, dy, h in AGG_CONFIGS:
        torch.manual_seed(81)
        layer = M.InteractionAggregation(dx, dy, output_dim=1, num_heads=h)
        with torch.no_grad():       # non-zero biases and weights of the scale a trained model has
            for p in layer.parameters():
                p.copy_(torch.randn(p.shape, generator=gen) * 0.3)
        x = torch.randn(B, dx, generator=gen).requires_grad_(True)
        y = torch.randn(B, dy, generator=gen).requires_grad_(True)
        groups["w_" + tag] = G.sd(layer)
        out = layer(x, y)
        gout = torch.randn(out.shape, generator=gen)
        (out * gout).sum().backward()
        groups["in"].update({"x_" + tag: x.detach(), "y_" + tag: y.detach(), "gout_" + tag: gout})
        groups["out"][tag] = out
        groups["gin"].update({"x_" + tag: x.grad, "y_" + tag: y.grad})
        groups["g_" + tag] = G.grads(layer)
    G.save("next_InteractionAggregation", {"B": B, "configs": AGG_CONFIGS}, **groups)


def case_feature_selection(M):
    gen = torch.Generator().manual_seed(83)
    B, D = 9, 4
    torch.manual_seed(83)
    fm = G.synthetic_fm(G.criteo_like_specs(10, 40), emb_dim=D)
    mat = G.synthetic_matrix(fm, B, gen)
    X = {k: v for k, v in G.batch_dict(fm, mat).items() if k not in fm.labels}
    groups = {"in": {"matrix": mat}, "out": {}, "gin": {}}
    d = D * fm.num_fields
    for tag, (c1, c2) in FS_CONTEXTS.items():
        torch.manual_seed(83)
        layer = M.FeatureSelection(fm, d, D, [16, 8], c1, c2)
        with torch.no_grad():       # gate inputs away from zero, context rows of a trained scale
            for name, p in layer.named_parameters():
                if "ctx_bias" in name or "embedding_layers" in name:
                    p.copy_(torch.randn(p.shape, generator=gen) * 0.5)
        emb = (torch.randn(B, d, generator=gen) * 0.5).requires_grad_(True)
        groups["w_" + tag] = G.sd(layer)
        f1, f2 = layer(X, emb)
        gout1, gout2 = torch.randn(f1.shape, generator=gen), torch.randn(f2.shape, generator=gen)
        ((f1 * gout1).sum() + (f2 * gout2).sum()).backward()
        groups["in"].update({"emb_" + tag: emb.detach(), "gout1_" + tag: gout1, "gout2_" + tag: gout2})
        groups["out"].update({"f1_" + tag: f1, "f2_" + tag: f2})
        groups["gin"]["emb_" + tag] = emb.grad
        groups["g_" + tag] = G.grads(layer)
    G.save("next_FeatureSelection", {"B": B, "embedding_dim": D, "fs_hidden_units": [16, 8],
                                     "contexts": FS_CONTEXTS, "specs": G.specs_json(fm), "labels": fm.labels},
           **groups)


def case_models():
    gen = torch.Generator().manual_seed(85)
    for case, (cls_name, kwargs) in MODEL_CASES.items():
        torch.manual_seed(2023)
        fm = G.synthetic_fm(G.criteo_like_specs(10, 40), emb_dim=4)
        model = model_class(cls_name)(fm, **G.model_params(**kwargs))
        with torch.no_grad():
            for m in model.modules():
                if isinstance(m, torch.nn.Embedding):
                    m.weight[1:].copy_(torch.randn(m.weight[1:].shape, generator=gen) * 0.1)
        mat = G.synthetic_matrix(fm, 3 * 32, gen)
        G.run_model_case("model_" + case, model, fm, mat,
                         {"case": case, "model": cls_name, "kwargs": kwargs, "seed": 2023})


if __name__ == "__main__":
    M = finalmlp_module()
    case_init(M)
    case_aggregation(M)
    case_feature_selection(M)
    case_models()

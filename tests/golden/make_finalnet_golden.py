"""Generates the FinalNet fixtures by running the REAL reference (model_zoo/FinalNet), with make_golden.py's helpers and
settings (reference import stubs, one thread, deterministic algorithms) and its own generators, so no other fixture
changes.  Run in the build container only:

    python tests/golden/make_finalnet_golden.py

Writes
  finalnet_init.json      state_dict keys, dtypes, shapes and the SHA-256 of each tensor of the reference's FinalBlock
                          and FeatureGating right after construction under torch.manual_seed(4848) (block configurations
                          with both residuals, batch norm on and off, a dropout and mixed per-layer rates, which show the
                          dropout index quirk in the `dropout` keys), and of FinalNet on a 6-field map right after
                          construction (which ends in reset_parameters) under torch.manual_seed(777), for the three
                          model configurations below;
  next_FinalBlock.npz     forward output, input gradient, every parameter gradient and the state after the forward
                          (running statistics, num_batches_tracked) of five blocks: concat and sum, batch norm on and off,
                          train and eval (eval with running statistics drawn away from 0 and 1), every BatchNorm weight
                          and bias drawn away from 1 and 0 (groups w_<c>, g_<c>, s_<c>; in/x_<c>, in/gout_<c>,
                          out/y_<c>, gin/x_<c>);
  next_FeatureGating.npz  the same for FeatureGating on (B, F, D) with the gate's weight drawn away from 0;
  model_FinalNet_2B.npz, model_FinalNet_1B_sum.npz, model_FinalNet_nobn.npz
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

# (name, input_dim, hidden_units, hidden_activations, dropout_rates, batch_norm, residual_type)
BLOCK_INIT = [("concat_bn", 12, [8, 6], None, 0, True, "concat"), ("sum_bn", 12, [5, 7], "ReLU", 0, True, "sum"),
              ("nobn", 10, [6], None, 0, False, "concat"), ("dropout", 10, [6, 4], None, 0.2, True, "concat"),
              ("mixed_dropout", 10, [6, 4, 4], ["ReLU", None, "Sigmoid"], [0, 0.5, 0], True, "concat")]
GATE_INIT = [("f5", 5), ("f39", 39)]
# (name, input_dim, hidden_units, hidden_activations, batch_norm, residual_type, training)
BLOCK_CASES = [("concat_bn_train", 12, [8, 6], None, True, "concat", True),
               ("sum_bn_train", 12, [5, 7], ["ReLU", "Sigmoid"], True, "sum", True),
               ("concat_nobn", 10, [6, 4], "ReLU", False, "concat", True),
               ("sum_nobn", 9, [3], None, False, "sum", True),
               ("concat_bn_eval", 12, [8, 6], ["Sigmoid", None], True, "concat", False)]
GATE_CASES = [("f5_d4", 5, 4), ("f7_d3", 7, 3)]
MODEL_KWARGS = {
    "2B": dict(embedding_dim=8, block_type="2B", batch_norm=True, use_feature_gating=True,
               block1_hidden_units=[16, 8], block2_hidden_units=[12, 8], residual_type="concat"),
    "1B_sum": dict(embedding_dim=6, block_type="1B", batch_norm=True, use_feature_gating=False,
                   block1_hidden_units=[12, 8], block1_hidden_activations="ReLU", residual_type="sum"),
    "nobn": dict(embedding_dim=4, block_type="2B", batch_norm=False, use_feature_gating=True,
                 block1_hidden_units=[8, 8], block1_hidden_activations=["ReLU", None],
                 block2_hidden_units=[16], block2_hidden_activations=["Sigmoid"], residual_type="concat"),
}


def finalnet_module():
    cls = G.load_model_class("FinalNet", "FinalNet")
    return sys.modules[cls.__module__]


def digests(module):
    return [[k, str(v.dtype), list(v.shape), hashlib.sha256(v.detach().contiguous().numpy().tobytes()).hexdigest()]
            for k, v in module.state_dict().items()]


def batch_norms(module, gen, running):
    with torch.no_grad():
        for m in module.modules():
            if isinstance(m, torch.nn.BatchNorm1d):
                m.weight.copy_(torch.rand(m.weight.shape, generator=gen) + 0.5)
                m.bias.copy_(torch.rand(m.bias.shape, generator=gen) * 0.6 - 0.3)
                if running:
                    m.running_mean.copy_(torch.randn(m.running_mean.shape, generator=gen) * 0.3)
                    m.running_var.copy_(torch.rand(m.running_var.shape, generator=gen) + 0.5)


def case_init(M):
    init = {"blocks": {}, "gates": {}, "models": {}}
    for (name, din, units, acts, drop, bn, res) in BLOCK_INIT:
        torch.manual_seed(4848)
        m = M.FinalBlock(din, units, acts, drop, bn, res)
        init["blocks"][name] = {"args": [din, units, acts, drop, bn, res], "seed": 4848, "state_dict": digests(m),
                                "dropout": [[k, mod.p] for k, mod in m.dropout.named_children()]}
    for (name, nf) in GATE_INIT:
        torch.manual_seed(4848)
        m = M.FeatureGating(nf)
        init["gates"][name] = {"args": [nf], "seed": 4848, "state_dict": digests(m)}
    specs = G.criteo_like_specs(6, 20)
    for name, kwargs in MODEL_KWARGS.items():
        torch.manual_seed(777)
        fm = G.synthetic_fm(specs, emb_dim=kwargs["embedding_dim"])
        model = M.FinalNet(fm, **G.model_params(**kwargs))
        init["models"][name] = {"seed": 777, "specs": G.specs_json(fm), "labels": fm.labels, "kwargs": kwargs,
                                "state_dict": digests(model)}
    path = os.path.join(G.HERE, "finalnet_init.json")
    with open(path, "w") as fd:
        json.dump(init, fd, indent=1, sort_keys=True)
    print("wrote", path)


def case_blocks(M):
    gen = torch.Generator().manual_seed(91)
    B = 8
    groups = {"in": {}, "out": {}, "gin": {}}
    for (c, din, units, acts, bn, res, training) in BLOCK_CASES:
        torch.manual_seed(91)
        block = M.FinalBlock(din, units, acts, 0, bn, res)
        batch_norms(block, gen, running=not training)
        block.train(training)
        x = (torch.randn(B, din, generator=gen) * 0.7).requires_grad_(True)
        groups["w_" + c] = G.sd(block)
        out = block(x)
        gout = torch.randn(out.shape, generator=gen)
        (out * gout).sum().backward()
        groups["in"]["x_" + c], groups["in"]["gout_" + c] = x.detach(), gout
        groups["out"]["y_" + c] = out
        groups["gin"]["x_" + c] = x.grad
        groups["g_" + c] = G.grads(block)
        groups["s_" + c] = G.sd(block)
    G.save("next_FinalBlock", {"B": B, "cases": [list(c) for c in BLOCK_CASES]}, **groups)


def case_gates(M):
    gen = torch.Generator().manual_seed(93)
    B = 6
    groups = {"in": {}, "out": {}, "gin": {}}
    for (c, nf, D) in GATE_CASES:
        torch.manual_seed(93)
        gate = M.FeatureGating(nf)
        with torch.no_grad():
            gate.linear.weight.copy_(torch.randn(nf, nf, generator=gen) * 0.4)
            gate.linear.bias.copy_(torch.rand(nf, generator=gen) + 0.5)
        x = (torch.randn(B, nf, D, generator=gen) * 0.7).requires_grad_(True)
        groups["w_" + c] = G.sd(gate)
        out = gate(x)
        gout = torch.randn(out.shape, generator=gen)
        (out * gout).sum().backward()
        groups["in"]["x_" + c], groups["in"]["gout_" + c] = x.detach(), gout
        groups["out"]["y_" + c] = out
        groups["gin"]["x_" + c] = x.grad
        groups["g_" + c] = G.grads(gate)
    G.save("next_FeatureGating", {"B": B, "cases": [list(c) for c in GATE_CASES]}, **groups)


def case_models(M):
    gen = torch.Generator().manual_seed(97)
    for name, kwargs in MODEL_KWARGS.items():
        torch.manual_seed(2023)
        fm = G.synthetic_fm(G.criteo_like_specs(10, 40), emb_dim=kwargs["embedding_dim"])
        model = M.FinalNet(fm, **G.model_params(**kwargs))
        with torch.no_grad():
            for m in model.modules():
                if isinstance(m, torch.nn.Embedding):
                    m.weight[1:].copy_(torch.randn(m.weight[1:].shape, generator=gen) * 0.3)
            if kwargs["use_feature_gating"]:
                model.feature_gating.linear.weight.copy_(torch.randn(10, 10, generator=gen) * 0.2)
        mat = G.synthetic_matrix(fm, 3 * 32, gen)
        G.run_model_case("model_FinalNet_" + name, model, fm, mat, {"case": name, "kwargs": kwargs, "seed": 2023})


if __name__ == "__main__":
    M = finalnet_module()
    case_init(M)
    case_blocks(M)
    case_gates(M)
    case_models(M)

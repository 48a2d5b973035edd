"""Generates the MaskNet fixtures by running the REAL reference (model_zoo/MaskNet), with make_golden.py's helpers and
settings (reference import stubs, one thread, deterministic algorithms) and its own generators, so no other fixture
changes.  Run in the build container only:

    python tests/golden/make_masknet_golden.py

Writes
  masknet_init.json   state_dict keys, dtypes, shapes and the SHA-256 of each tensor right after construction: the
                      reference's MaskBlock under torch.manual_seed(4747) for three configurations (a float
                      reduction_ratio, no LayerNorm, dropout), and MaskNet on a 6-field map (construction ends in
                      reset_parameters) under torch.manual_seed(777) for SerialMaskNet, ParallelMaskNet with dropout
                      and a float reduction_ratio, and a ParallelMaskNet without hidden units;
  next_MaskBlock.npz  forward output, both input gradients (V_emb and V_hidden) and every parameter gradient of one
                      MaskBlock at output width 20 (ReLU) and 13 (Sigmoid), with the LayerNorm's weight and bias
                      drawn away from 1 and 0 (groups w_n<n>, g_n<n>; in/{emb,hid,gout}_n<n>, out/y_n<n>,
                      gin/{emb,hid}_n<n>);
  model_MaskNet_serial.npz, model_MaskNet_parallel.npz, model_MaskNet_noln.npz
                      make_golden.run_model_case on the reference models (10-field map): inputs, weights, y_pred,
                      loss, gradients, the state after 1 and 3 train_step()s.
"""
import hashlib
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_golden as G  # noqa: E402  (imports the reference)

torch = G.torch

BLOCK_CONFIGS = {                # MaskBlock(input_dim, hidden_dim, output_dim, act, reduction_ratio, dropout, ln)
    "float_ratio": [40, 24, 16, "relu", 1.5, 0, True],
    "no_ln": [40, 40, 13, "sigmoid", 1, 0, False],
    "dropout": [24, 24, 8, "relu", 0.5, 0.2, True],
}
MODEL_KWARGS = {
    "serial": dict(embedding_dim=4, dnn_hidden_units=[24, 16], dnn_hidden_activations="relu",
                   model_type="SerialMaskNet", reduction_ratio=1),
    "parallel": dict(embedding_dim=4, dnn_hidden_units=[16], dnn_hidden_activations="relu",
                     model_type="ParallelMaskNet", parallel_num_blocks=3, parallel_block_dim=8, reduction_ratio=0.5),
    "noln": dict(embedding_dim=4, dnn_hidden_units=[20, 12], dnn_hidden_activations="relu",
                 model_type="SerialMaskNet", emb_layernorm=False, net_layernorm=False),
}
INIT_MODELS = {
    "serial": MODEL_KWARGS["serial"],
    "parallel_dropout": dict(MODEL_KWARGS["parallel"], net_dropout=0.1, reduction_ratio=1.25),
    "parallel_head": dict(embedding_dim=4, dnn_hidden_units=[], model_type="ParallelMaskNet", parallel_num_blocks=2,
                          parallel_block_dim=8),
}


def masknet_module():
    cls = G.load_model_class("MaskNet", "MaskNet")
    return sys.modules[cls.__module__]


def digests(module):
    return [[k, str(v.dtype), list(v.shape), hashlib.sha256(v.detach().contiguous().numpy().tobytes()).hexdigest()]
            for k, v in module.state_dict().items()]


def case_init(M):
    init = {"blocks": {}, "models": {}}
    for name, args in BLOCK_CONFIGS.items():
        torch.manual_seed(4747)
        init["blocks"][name] = {"args": args, "seed": 4747, "state_dict": digests(M.MaskBlock(*args))}
    specs = G.criteo_like_specs(6, 20)
    for name, kwargs in INIT_MODELS.items():
        torch.manual_seed(777)
        fm = G.synthetic_fm(specs, emb_dim=4)
        model = M.MaskNet(fm, **G.model_params(**kwargs))
        init["models"][name] = {"seed": 777, "specs": G.specs_json(fm), "labels": fm.labels, "kwargs": kwargs,
                                "state_dict": digests(model)}
    path = os.path.join(G.HERE, "masknet_init.json")
    with open(path, "w") as fd:
        json.dump(init, fd, indent=1, sort_keys=True)
    print("wrote", path)


def case_block(M):
    gen = torch.Generator().manual_seed(91)
    B, d, hd = 6, 12, 16
    groups = {"in": {}, "out": {}, "gin": {}}
    for n, act in ((20, "relu"), (13, "sigmoid")):
        torch.manual_seed(91)
        blk = M.MaskBlock(d, hd, n, act, 1.5, 0, True)
        with torch.no_grad():
            ln = blk.hidden_layer[1]
            ln.weight.copy_(1.0 + 0.5 * torch.randn(n, generator=gen))
            ln.bias.copy_(0.3 * torch.randn(n, generator=gen))
        emb = (torch.randn(B, d, generator=gen) * 0.7).requires_grad_(True)
        hid = (torch.randn(B, hd, generator=gen) * 0.7 + 0.2).requires_grad_(True)
        groups["w_n%d" % n] = G.sd(blk)
        out = blk(emb, hid)
        gout = torch.randn(out.shape, generator=gen)
        (out * gout).sum().backward()
        groups["in"]["emb_n%d" % n], groups["in"]["hid_n%d" % n] = emb.detach(), hid.detach()
        groups["in"]["gout_n%d" % n] = gout
        groups["out"]["y_n%d" % n] = out
        groups["gin"]["emb_n%d" % n], groups["gin"]["hid_n%d" % n] = emb.grad, hid.grad
        groups["g_n%d" % n] = G.grads(blk)
    G.save("next_MaskBlock", {"B": B, "input_dim": d, "hidden_dim": hd, "reduction_ratio": 1.5,
                              "widths": {"20": "relu", "13": "sigmoid"}}, **groups)


def case_models(M):
    gen = torch.Generator().manual_seed(93)
    for name, kwargs in MODEL_KWARGS.items():
        torch.manual_seed(2023)
        fm = G.synthetic_fm(G.criteo_like_specs(10, 40), emb_dim=4)
        model = M.MaskNet(fm, **G.model_params(**kwargs))
        with torch.no_grad():
            for m in model.modules():
                if isinstance(m, torch.nn.Embedding):
                    m.weight[1:].copy_(torch.randn(m.weight[1:].shape, generator=gen) * 0.1)
                if isinstance(m, torch.nn.LayerNorm):       # away from 1 and 0, so the affine path counts
                    m.weight.copy_(1.0 + 0.3 * torch.randn(m.weight.shape, generator=gen))
                    m.bias.copy_(0.2 * torch.randn(m.bias.shape, generator=gen))
        mat = G.synthetic_matrix(fm, 3 * 32, gen)
        G.run_model_case("model_MaskNet_" + name, model, fm, mat, {"case": name, "kwargs": kwargs, "seed": 2023})


if __name__ == "__main__":
    M = masknet_module()
    case_init(M)
    case_block(M)
    case_models(M)

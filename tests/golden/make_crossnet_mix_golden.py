"""Generates the CrossNetMix fixtures (DCNv2's use_low_rank_mixture=True) by running the REAL reference, with
make_golden.py's helpers and settings (reference import stubs, one thread, deterministic algorithms) and its
own generators, so no other fixture changes.  Run in the build container only:

    python tests/golden/make_crossnet_mix_golden.py

Writes
  crossnet_mix_init.json  state_dict keys, dtypes, shapes and the SHA-256 of each tensor of the reference's
                          CrossNetMix right after construction under torch.manual_seed(4343), for four
                          (in_features, layer_num, low_rank, num_experts) configurations;
  model_DCNv2_mix.npz     make_golden.run_model_case on the reference DCNv2 with the mixture (10-field map):
                          inputs, weights, y_pred, loss, gradients, the state after 1 and 3 train_step()s.
"""
import hashlib
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_golden as G  # noqa: E402  (imports the reference)

torch = G.torch

INIT_CONFIGS = [(20, 2, 4, 3), (12, 1, 8, 1), (40, 3, 32, 4), (16, 2, 64, 4)]   # (d, L, r, E)


def case_init():
    init = {}
    for (d, nl, r, E) in INIT_CONFIGS:
        torch.manual_seed(4343)
        layer = G.L.CrossNetMix(d, layer_num=nl, low_rank=r, num_experts=E)
        init["d%d_L%d_r%d_E%d" % (d, nl, r, E)] = {
            "args": [d, nl, r, E], "seed": 4343,
            "state_dict": [[k, str(v.dtype), list(v.shape),
                            hashlib.sha256(v.detach().contiguous().numpy().tobytes()).hexdigest()]
                           for k, v in layer.state_dict().items()]}
    path = os.path.join(G.HERE, "crossnet_mix_init.json")
    with open(path, "w") as fd:
        json.dump(init, fd, indent=1, sort_keys=True)
    print("wrote", path)


def case_model():
    gen = torch.Generator().manual_seed(61)
    kwargs = dict(embedding_dim=8, model_structure="parallel", num_cross_layers=2, use_low_rank_mixture=True,
                  low_rank=4, num_experts=3, parallel_dnn_hidden_units=[24, 16], dnn_activations="relu")
    torch.manual_seed(2023)
    fm = G.synthetic_fm(G.criteo_like_specs(10, 40), emb_dim=8)
    model = G.load_model_class("DCNv2", "DCNv2")(fm, **G.model_params(**kwargs))
    with torch.no_grad():
        for m in model.modules():
            if isinstance(m, torch.nn.Embedding):
                m.weight[1:].copy_(torch.randn(m.weight[1:].shape, generator=gen) * 0.1)
        for k, p in model.named_parameters():
            if k.startswith("crossnet.bias."):          # zeros at init: give the bias path something to carry
                p.copy_(torch.randn(p.shape, generator=gen) * 0.1)
    mat = G.synthetic_matrix(fm, 3 * 32, gen)
    G.run_model_case("model_DCNv2_mix", model, fm, mat, {"case": "DCNv2_mix", "kwargs": kwargs, "seed": 2023})


if __name__ == "__main__":
    case_init()
    case_model()

"""Generates the DIEN fixtures by running the REAL reference (model_zoo/DIEN), with make_golden.py's helpers and settings
(reference import stubs, one thread, deterministic algorithms) and its own generators, so no other fixture changes.
Run in the build container only:

    python tests/golden/make_dien_golden.py

Writes
  dien_init.json          state_dict keys, dtypes, shapes and the SHA-256 of each tensor of DIEN on the sequence map below
                          right after construction (which ends in reset_parameters) under torch.manual_seed(777), for
                          the model configurations below;
  next_DIEN_<c>.npz       the interest stack of pair 0 (DIEN.interest_extraction, the attention and interest_evolution,
                          then get_unmasked_tensor) on ragged histories: in/seq (B, L, H), in/target (B, H), in/mask,
                          in/gout; out/h_out; gin/seq, gin/target; w and g the stack's parameters and their gradients;
  model_DIEN_<c>.npz      make_golden.run_model_case on the reference models: inputs, weights, y_pred, loss, gradients,
                          the state after 1 and 3 train_step()s.
Every history matrix holds, in each batch of 32 rows, an empty row, a full row, a row of length 1 and a row with a zero
id inside its history (rows 0 to 3); the rest are post-padded with random lengths.
"""
import hashlib
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_golden as G  # noqa: E402  (imports the reference)

torch = G.torch

SEQ_SPECS = [("user_id", {"type": "categorical", "source": "", "padding_idx": 0, "vocab_size": 30}),
             ("item_id", {"type": "categorical", "source": "", "padding_idx": 0, "vocab_size": 60}),
             ("cate_id", {"type": "categorical", "source": "", "padding_idx": 0, "vocab_size": 12}),
             ("click_history", {"type": "sequence", "source": "", "padding_idx": 0, "vocab_size": 60, "max_len": 7,
                                "share_embedding": "item_id", "feature_encoder": None}),
             ("cate_history", {"type": "sequence", "source": "", "padding_idx": 0, "vocab_size": 12, "max_len": 7,
                               "share_embedding": "cate_id", "feature_encoder": None})]
ONE_SEQ_SPECS = SEQ_SPECS[:4]       # every sequence field must be some pair's: the reference's DNN width counts the rest
TUPLE = dict(dien_target_field=[("item_id", "cate_id")], dien_sequence_field=[("click_history", "cate_history")])
MODEL_KWARGS = {
    "augru_bilinear": dict(embedding_dim=4, gru_type="AUGRU", attention_type="bilinear_attention",
                           use_attention_softmax=True, dnn_hidden_units=[16, 8], dnn_activations="ReLU",
                           batch_norm=False, dien_neg_seq_field=[], **TUPLE),
    "agru_dot": dict(embedding_dim=8, gru_type="AGRU", attention_type="dot_attention", use_attention_softmax=False,
                     dnn_hidden_units=[16], dnn_activations="ReLU", batch_norm=False, dien_target_field="item_id",
                     dien_sequence_field="click_history", dien_neg_seq_field=[]),
    "augru_din_sumpool": dict(embedding_dim=4, gru_type="AUGRU", attention_type="din_attention",
                              attention_hidden_units=[8, 4], attention_activation="ReLU", enable_sum_pooling=True,
                              dnn_hidden_units=[16, 8], dnn_activations="ReLU", batch_norm=False,
                              dien_neg_seq_field=[], **TUPLE),
    "gru_dice_bn": dict(embedding_dim=4, gru_type="GRU", dnn_hidden_units=[16, 8], dnn_activations="Dice",
                        batch_norm=True, dien_neg_seq_field=[], **TUPLE),
}
STACK_PREFIXES = ("extraction_modules.", "evolving_modules.", "attention_modules.")


def model_specs(name):
    return ONE_SEQ_SPECS if name == "agru_dot" else SEQ_SPECS


def digests(module):
    return [[k, str(v.dtype), list(v.shape), hashlib.sha256(v.detach().contiguous().numpy().tobytes()).hexdigest()]
            for k, v in module.state_dict().items()]


def history_kinds(mat, fm, B):
    """Rows 0..3 of each batch: empty, full, length 1, a zero inside the history (ids at 0..5 but position 2)."""
    for name, spec in fm.features.items():
        if spec["type"] != "sequence":
            continue
        cols = fm.get_column_index(name)
        c0, L = cols[0], len(cols)
        for i in range(mat.shape[0] // B):
            r = i * B
            ids = torch.arange(1, L + 1, dtype=mat.dtype) % (spec["vocab_size"] - 1) + 1
            mat[r, c0:c0 + L] = 0
            mat[r + 1, c0:c0 + L] = ids
            mat[r + 2, c0:c0 + L] = 0
            mat[r + 2, c0] = ids[3]
            mat[r + 3, c0:c0 + L] = ids
            mat[r + 3, c0 + 2] = 0
            mat[r + 3, c0 + 6:c0 + L] = 0
    return mat


def build(M, name, seed):
    kwargs = MODEL_KWARGS[name]
    torch.manual_seed(seed)
    fm = G.synthetic_fm(model_specs(name), emb_dim=kwargs["embedding_dim"])
    return fm, M.DIEN(fm, **G.model_params(**kwargs))


def case_init(M):
    init = {"models": {}}
    for name, kwargs in MODEL_KWARGS.items():
        fm, model = build(M, name, 777)
        init["models"][name] = {"seed": 777, "specs": G.specs_json(fm), "labels": fm.labels, "kwargs": kwargs,
                                "state_dict": digests(model)}
    path = os.path.join(G.HERE, "dien_init.json")
    with open(path, "w") as fd:
        json.dump(init, fd, indent=1, sort_keys=True)
    print("wrote", path)


def case_stacks(M):
    gen = torch.Generator().manual_seed(95)
    B, L = 9, 7
    lens = torch.tensor([0, 7, 1, 4, 0, 3, 6, 2, 5])
    for name, kwargs in MODEL_KWARGS.items():
        fm, model = build(M, name, 91)
        model.train()
        with torch.no_grad():       # nonzero GRU biases and a non-identity W_kernel, so every gradient is exercised
            for k, p in model.named_parameters():
                if k.startswith(STACK_PREFIXES) and ("bias" in k or "W_kernel" in k):
                    p.add_(torch.randn(p.shape, generator=gen) * 0.2)
        H = model.extraction_modules[0].hidden_size
        mask = torch.arange(L).view(1, -1) < lens.view(-1, 1)
        mask[3, 1] = False          # a zero inside the history: length 3, position 3 still unmasked
        seq = (torch.randn(B, L, H, generator=gen) * 0.7 * mask.unsqueeze(-1)).requires_grad_(True)
        tgt = (torch.randn(B, H, generator=gen) * 0.7).requires_grad_(True)
        nz = mask.sum(dim=1) > 0
        packed, interest = model.interest_extraction(0, seq[nz], mask[nz])
        h_out = model.interest_evolution(0, packed, interest, tgt[nz], mask[nz])
        out = model.get_unmasked_tensor(h_out, nz)
        gout = torch.randn(out.shape, generator=gen)
        (out * gout).sum().backward()
        w = {k: v for k, v in G.sd(model).items() if k.startswith(STACK_PREFIXES)}
        g = {k: v for k, v in G.grads(model).items() if k.startswith(STACK_PREFIXES)}
        G.save("next_DIEN_" + name, {"B": B, "L": L, "H": H, "case": name, "kwargs": kwargs},
               **{"in": {"seq": seq.detach(), "target": tgt.detach(), "mask": mask.to(torch.uint8), "gout": gout},
                  "out": {"h_out": out}, "w": w, "g": g,
                  "gin": {"seq": seq.grad, "target": torch.zeros_like(tgt) if tgt.grad is None else tgt.grad}})


def case_models(M):
    gen = torch.Generator().manual_seed(93)
    for name in MODEL_KWARGS:
        fm, model = build(M, name, 2023)
        with torch.no_grad():
            for m in model.modules():
                if isinstance(m, torch.nn.Embedding):
                    m.weight[1:].copy_(torch.randn(m.weight[1:].shape, generator=gen) * 0.3)
        mat = history_kinds(G.synthetic_matrix(fm, 3 * 32, gen, seq_min=0), fm, 32)
        G.run_model_case("model_DIEN_" + name, model, fm, mat,
                         {"case": name, "kwargs": MODEL_KWARGS[name], "seed": 2023})


if __name__ == "__main__":
    M = sys.modules[G.load_model_class("DIEN", "DIEN").__module__]
    case_init(M)
    case_stacks(M)
    case_models(M)

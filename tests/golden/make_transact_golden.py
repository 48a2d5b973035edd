"""Generates the TransAct fixtures by running the REAL reference (model_zoo/TransAct), with make_golden.py's helpers and
settings (reference import stubs, one thread, deterministic algorithms) and its own generators, so no other fixture
changes.  Run in the build container only:

    python tests/golden/make_transact_golden.py

Writes
  transact_init.json      state_dict keys, dtypes, shapes and the SHA-256 of each tensor of the reference's
                          TransActTransformer (the configurations of MODULE_CASES) right after construction under
                          torch.manual_seed(4747), and of TransAct on the sequence maps below right after construction
                          (which ends in reset_parameters) under torch.manual_seed(777), for MODEL_KWARGS;
  next_TransActTransformer_<c>.npz
                          forward output, input gradients and every parameter gradient of one module on
                          (target_emb, sequence_emb, mask = ids == 0): in/seq (B, L, ns D), in/tgt (B, nt D), in/ids,
                          in/gout, out/y, gin/seq, gin/tgt, w, g.  Each batch holds an empty history (row 0), a full
                          one (row 1), left- and right-padded ragged ones, and a history whose first two items repeat
                          (row 2), so the max-pool has exact ties;
  model_TransAct_<c>.npz  make_golden.run_model_case on the reference models: inputs, weights, y_pred, loss, gradients,
                          the state after 1 and 3 train_step()s.
"""
import hashlib
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_golden as G  # noqa: E402  (imports the reference)

torch = G.torch

# (name, L, D, ns, nt, num_heads, layers, dim_feedforward, first_k_cols, concat_max_pool)
MODULE_CASES = [("h1_k1_pool", 7, 4, 1, 1, 1, 1, 16, 1, True),
                ("h2_l2_k3_pool_tuple", 9, 4, 2, 2, 2, 2, 12, 3, True),
                ("h4_k2_nopool", 6, 4, 1, 1, 4, 1, 8, 2, False),
                ("h1_l2_k1_pool_ties", 8, 3, 1, 2, 1, 2, 10, 1, True)]

SEQ_SPECS = [("user_id", {"type": "categorical", "source": "", "padding_idx": 0, "vocab_size": 30}),
             ("item_id", {"type": "categorical", "source": "", "padding_idx": 0, "vocab_size": 60}),
             ("cate_id", {"type": "categorical", "source": "", "padding_idx": 0, "vocab_size": 12}),
             ("click_history", {"type": "sequence", "source": "", "padding_idx": 0, "vocab_size": 60, "max_len": 7,
                                "share_embedding": "item_id", "feature_encoder": None}),
             ("cate_history", {"type": "sequence", "source": "", "padding_idx": 0, "vocab_size": 12, "max_len": 7,
                               "share_embedding": "cate_id", "feature_encoder": None})]
ONE_SEQ_SPECS = SEQ_SPECS[:4]       # every sequence field must be some pair's: the reference concatenates the rest
MODEL_KWARGS = {
    "tuple_k1_pool": dict(embedding_dim=4, num_heads=1, transformer_layers=1, dim_feedforward=16, dcn_cross_layers=2,
                          dcn_hidden_units=[16, 8], mlp_hidden_units=[], first_k_cols=1, concat_max_pool=True,
                          target_item_field=[("item_id", "cate_id")],
                          sequence_item_field=[("click_history", "cate_history")]),
    "two_pairs_k2_nopool": dict(embedding_dim=4, num_heads=2, transformer_layers=2, dim_feedforward=8,
                                dcn_cross_layers=1, dcn_hidden_units=[16], mlp_hidden_units=[8], first_k_cols=2,
                                concat_max_pool=False, target_item_field=["item_id", "cate_id"],
                                sequence_item_field=["click_history", "cate_history"]),
    "h4_k3_bn": dict(embedding_dim=8, num_heads=4, transformer_layers=1, dim_feedforward=16, dcn_cross_layers=2,
                     dcn_hidden_units=[16, 8], mlp_hidden_units=[8], first_k_cols=3, concat_max_pool=True,
                     batch_norm=True, target_item_field="item_id", sequence_item_field="click_history"),
}


def model_specs(name):
    return ONE_SEQ_SPECS if name == "h4_k3_bn" else SEQ_SPECS


def transact_module():
    cls = G.load_model_class("TransAct", "TransAct")
    return sys.modules[cls.__module__]


def digests(module):
    return [[k, str(v.dtype), list(v.shape), hashlib.sha256(v.detach().contiguous().numpy().tobytes()).hexdigest()]
            for k, v in module.state_dict().items()]


def history_ids(B, L, vocab, gen):
    """(B, L) ids: row 0 empty, row 1 full, row 2 with its first two items equal, the rest ragged, odd rows padded on
    the left (TransAct's layout) and even rows on the right."""
    ids = torch.randint(1, vocab, (B, L), generator=gen)
    lens = torch.randint(1, L + 1, (B,), generator=gen)
    lens[0], lens[1], lens[2] = 0, L, max(2, int(lens[2]))
    pos = torch.arange(L).view(1, -1)
    keep = pos < lens.view(-1, 1)
    left = (torch.arange(B) % 2 == 1).view(-1, 1)
    keep = torch.where(left, pos >= (L - lens).view(-1, 1), keep)
    ids = ids * keep
    ids[2, 1] = ids[2, 0]
    return ids


def case_init(M):
    init = {"modules": {}, "models": {}}
    for (name, L, D, ns, nt, H, n, ffn, k, pool) in MODULE_CASES:
        torch.manual_seed(4747)
        m = M.TransActTransformer(D * (ns + nt), dim_feedforward=ffn, num_heads=H, transformer_layers=n,
                                  first_k_cols=k, concat_max_pool=pool)
        init["modules"][name] = {"args": [D * (ns + nt), ffn, H, n, k, pool], "seed": 4747, "state_dict": digests(m)}
    for name, kwargs in MODEL_KWARGS.items():
        torch.manual_seed(777)
        fm = G.synthetic_fm(model_specs(name), emb_dim=kwargs["embedding_dim"])
        model = M.TransAct(fm, **G.model_params(**kwargs))
        init["models"][name] = {"seed": 777, "specs": G.specs_json(fm), "labels": fm.labels, "kwargs": kwargs,
                                "state_dict": digests(model)}
    path = os.path.join(G.HERE, "transact_init.json")
    with open(path, "w") as fd:
        json.dump(init, fd, indent=1, sort_keys=True)
    print("wrote", path)


def case_modules(M):
    gen = torch.Generator().manual_seed(91)
    B = 6
    for (c, L, D, ns, nt, H, n, ffn, k, pool) in MODULE_CASES:
        md = D * (ns + nt)
        torch.manual_seed(91)
        mod = M.TransActTransformer(md, dim_feedforward=ffn, num_heads=H, transformer_layers=n, first_k_cols=k,
                                    concat_max_pool=pool)
        with torch.no_grad():       # nonzero biases and LayerNorm affines, so every gradient is exercised
            for lyr in mod.transformer_encoder.layers:
                lyr.self_attn.in_proj_bias.copy_(torch.randn(3 * md, generator=gen) * 0.1)
                lyr.self_attn.out_proj.bias.copy_(torch.randn(md, generator=gen) * 0.1)
                for norm in (lyr.norm1, lyr.norm2):
                    norm.weight.copy_(torch.rand(md, generator=gen) + 0.5)
                    norm.bias.copy_(torch.rand(md, generator=gen) * 0.6 - 0.3)
        ids = history_ids(B, L, 50, gen)
        seq = torch.randn(B, L, ns * D, generator=gen) * 0.7
        seq[2, 1] = seq[2, 0]                       # a repeated item: bit-identical tokens, ties in the max-pool
        seq = seq.requires_grad_(True)
        tgt = (torch.randn(B, nt * D, generator=gen) * 0.7).requires_grad_(True)
        w = G.sd(mod)
        mod.train()
        y = mod(tgt, seq, mask=(ids == 0))
        gout = torch.randn(y.shape, generator=gen)
        (y * gout).sum().backward()
        G.save("next_TransActTransformer_" + c, {"B": B, "L": L, "case": [c, L, D, ns, nt, H, n, ffn, k, pool]},
               **{"in": {"seq": seq.detach(), "tgt": tgt.detach(), "ids": ids, "gout": gout}, "out": {"y": y},
                  "gin": {"seq": seq.grad, "tgt": tgt.grad}, "w": w, "g": G.grads(mod)})


def case_models(M):
    gen = torch.Generator().manual_seed(93)
    for name, kwargs in MODEL_KWARGS.items():
        torch.manual_seed(2023)
        fm = G.synthetic_fm(model_specs(name), emb_dim=kwargs["embedding_dim"])
        model = M.TransAct(fm, **G.model_params(**kwargs))
        with torch.no_grad():
            for m in model.modules():
                if isinstance(m, torch.nn.Embedding):
                    m.weight[1:].copy_(torch.randn(m.weight[1:].shape, generator=gen) * 0.3)
        mat = G.synthetic_matrix(fm, 3 * 32, gen, seq_min=0)
        B = 32
        for i in range(3):                          # per batch: the history layouts of history_ids, both fields alike
            rows = slice(i * B, (i + 1) * B)
            first = None
            for f, spec in fm.features.items():
                if spec["type"] != "sequence":
                    continue
                col = fm.get_column_index(f)
                cur = mat[rows, col[0]:col[-1] + 1]
                h = history_ids(B, spec["max_len"], spec["vocab_size"], gen).double()
                if first is None:
                    first = h != 0
                else:
                    h = h.clamp_min(1) * first
                    h[2, 1] = h[2, 0]
                cur.copy_(h)
        G.run_model_case("model_TransAct_" + name, model, fm, mat, {"case": name, "kwargs": kwargs, "seed": 2023})


if __name__ == "__main__":
    M = transact_module()
    case_init(M)
    case_modules(M)
    case_models(M)

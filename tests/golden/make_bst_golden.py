"""Generates the BST fixtures by running the REAL reference (model_zoo/BST), with make_golden.py's helpers and settings
(reference import stubs, one thread, deterministic algorithms) and its own generators, so no other fixture changes.
Run in the build container only:

    python tests/golden/make_bst_golden.py

Writes
  bst_init.json           state_dict keys, dtypes, shapes and the SHA-256 of each tensor of the reference's
                          TransformerBlock (four configurations) and BehaviorTransformer (two) right after construction
                          under torch.manual_seed(4747); and of BST on the sequence map below right after construction
                          (which ends in reset_parameters) under torch.manual_seed(777), for the model configurations
                          below;
  next_TransformerBlock_<c>.npz
                          forward output, input gradient and every parameter gradient of one block on x (B, L, md) with
                          the reference's mask (BST.get_mask) from a ragged history (in/x, in/valid, in/gout, out/y,
                          gin/x, w, g), for the block configurations of BLOCK_CASES;
  model_BST_<c>.npz       make_golden.run_model_case on the reference models: inputs, weights, y_pred, loss, gradients,
                          the state after 1 and 3 train_step()s.
"""
import hashlib
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_golden as G  # noqa: E402  (imports the reference)

torch = G.torch

# (name, model_dim, num_heads, attn_dropout, net_dropout, layer_norm, use_residual)
BLOCK_INIT = [("ln_h4", 8, 4, 0.0, 0.0, True, True), ("noln_h3", 12, 3, 0.0, 0.0, False, True),
              ("nores_h1", 6, 1, 0.0, 0.0, True, False), ("dropout", 16, 2, 0.1, 0.2, True, True)]
# (name, seq_len, model_dim, num_heads, stacked, position_dim, use_position_emb)
TRANSFORMER_INIT = [("pos", 6, 8, 4, 1, 4, True), ("nopos_2", 9, 12, 3, 2, 4, False)]
# (name, model_dim, num_heads, layer_norm, use_residual, causal)
BLOCK_CASES = [("ln_h4", 8, 4, True, True, False), ("noln_h3_causal", 12, 3, False, True, True),
               ("nores_h1", 6, 1, True, False, False), ("ln_h2_causal", 16, 2, True, True, True)]

SEQ_SPECS = [("user_id", {"type": "categorical", "source": "", "padding_idx": 0, "vocab_size": 30}),
             ("item_id", {"type": "categorical", "source": "", "padding_idx": 0, "vocab_size": 60}),
             ("cate_id", {"type": "categorical", "source": "", "padding_idx": 0, "vocab_size": 12}),
             ("click_history", {"type": "sequence", "source": "", "padding_idx": 0, "vocab_size": 60, "max_len": 7,
                                "share_embedding": "item_id", "feature_encoder": None}),
             ("cate_history", {"type": "sequence", "source": "", "padding_idx": 0, "vocab_size": 12, "max_len": 7,
                               "share_embedding": "cate_id", "feature_encoder": None})]
ONE_SEQ_SPECS = SEQ_SPECS[:4]       # every sequence field must be some pair's: the reference concatenates the rest
MODEL_KWARGS = {
    "tuple_mean": dict(embedding_dim=4, num_heads=2, dnn_hidden_units=[24, 16], dnn_activations="relu",
                       bst_target_field=[("item_id", "cate_id")],
                       bst_sequence_field=[("click_history", "cate_history")], seq_pooling_type="mean",
                       use_position_emb=True),
    "sum_nopos_causal": dict(embedding_dim=8, num_heads=2, stacked_transformer_layers=2, dnn_hidden_units=[16],
                             dnn_activations="relu", bst_target_field="item_id", bst_sequence_field="click_history",
                             seq_pooling_type="sum", use_position_emb=False, use_causal_mask=True),
    "target_two_pairs": dict(embedding_dim=4, num_heads=4, dnn_hidden_units=[16, 8], dnn_activations="relu",
                             bst_target_field=["item_id", "cate_id"],
                             bst_sequence_field=["click_history", "cate_history"], seq_pooling_type="target"),
    "concat_noln": dict(embedding_dim=4, num_heads=3, dnn_hidden_units=[16], dnn_activations="relu",
                        bst_target_field=[("item_id", "cate_id")],
                        bst_sequence_field=[("click_history", "cate_history")], seq_pooling_type="concat",
                        layer_norm=False, use_residual=False),
}


def model_specs(name):
    return ONE_SEQ_SPECS if name == "sum_nopos_causal" else SEQ_SPECS


def bst_module():
    cls = G.load_model_class("BST", "BST")
    return sys.modules[cls.__module__]


def digests(module):
    return [[k, str(v.dtype), list(v.shape), hashlib.sha256(v.detach().contiguous().numpy().tobytes()).hexdigest()]
            for k, v in module.state_dict().items()]


def ref_mask(valid, heads, causal):
    """BST.get_mask on a (B, L - 1) validity mask: the (B H, L, L) bool attn_mask."""
    B = valid.shape[0]
    padding = torch.cat([~valid, torch.zeros(B, 1, dtype=torch.bool)], dim=-1)
    L = padding.shape[1]
    m = padding.unsqueeze(1).repeat(1, L, 1) & ~torch.eye(L, dtype=torch.bool).unsqueeze(0)
    if causal:
        m = m | torch.triu(torch.ones(L, L), 1).bool().unsqueeze(0)
    return m.unsqueeze(1).repeat(1, heads, 1, 1).flatten(end_dim=1)


def case_init(M):
    init = {"blocks": {}, "transformers": {}, "models": {}}
    for (name, md, H, pa, pn, ln, res) in BLOCK_INIT:
        torch.manual_seed(4747)
        m = M.TransformerBlock(model_dim=md, ffn_dim=md, num_heads=H, attn_dropout=pa, net_dropout=pn, layer_norm=ln,
                               use_residual=res)
        init["blocks"][name] = {"args": [md, H, pa, pn, ln, res], "seed": 4747, "state_dict": digests(m)}
    for (name, L, md, H, n, pd, pos) in TRANSFORMER_INIT:
        torch.manual_seed(4747)
        m = M.BehaviorTransformer(seq_len=L, model_dim=md, num_heads=H, stacked_transformer_layers=n,
                                  position_dim=pd, use_position_emb=pos)
        init["transformers"][name] = {"args": [L, md, H, n, pd, pos], "seed": 4747, "state_dict": digests(m)}
    for name, kwargs in MODEL_KWARGS.items():
        torch.manual_seed(777)
        fm = G.synthetic_fm(model_specs(name), emb_dim=kwargs["embedding_dim"])
        model = M.BST(fm, **G.model_params(**kwargs))
        init["models"][name] = {"seed": 777, "specs": G.specs_json(fm), "labels": fm.labels, "kwargs": kwargs,
                                "state_dict": digests(model)}
    path = os.path.join(G.HERE, "bst_init.json")
    with open(path, "w") as fd:
        json.dump(init, fd, indent=1, sort_keys=True)
    print("wrote", path)


def case_blocks(M):
    gen = torch.Generator().manual_seed(91)
    B, L = 5, 7
    for (c, md, H, ln, res, causal) in BLOCK_CASES:
        torch.manual_seed(91)
        blk = M.TransformerBlock(model_dim=md, ffn_dim=md, num_heads=H, layer_norm=ln, use_residual=res)
        with torch.no_grad():       # nonzero biases and LayerNorm affines, so every gradient is exercised
            blk.attention.in_proj_bias.copy_(torch.randn(3 * md, generator=gen) * 0.1)
            blk.attention.out_proj.bias.copy_(torch.randn(md, generator=gen) * 0.1)
            if ln:
                for norm in (blk.layer_norm1, blk.layer_norm2):
                    norm.weight.copy_(torch.rand(md, generator=gen) + 0.5)
                    norm.bias.copy_(torch.rand(md, generator=gen) * 0.6 - 0.3)
        lens = torch.tensor([0, 6, 3, 1, 5])
        valid = torch.arange(L - 1).view(1, -1) < lens.view(-1, 1)
        x = (torch.randn(B, L, md, generator=gen) * 0.7).requires_grad_(True)
        w = G.sd(blk)
        y = blk(x, attn_mask=ref_mask(valid, H, causal))
        gout = torch.randn(y.shape, generator=gen)
        (y * gout).sum().backward()
        G.save("next_TransformerBlock_" + c, {"B": B, "L": L, "case": [c, md, H, ln, res, causal]},
               **{"in": {"x": x.detach(), "valid": valid.to(torch.uint8), "gout": gout}, "out": {"y": y},
                  "gin": {"x": x.grad}, "w": w, "g": G.grads(blk)})


def case_models(M):
    gen = torch.Generator().manual_seed(93)
    for name, kwargs in MODEL_KWARGS.items():
        torch.manual_seed(2023)
        fm = G.synthetic_fm(model_specs(name), emb_dim=kwargs["embedding_dim"])
        model = M.BST(fm, **G.model_params(**kwargs))
        with torch.no_grad():
            for m in model.modules():
                if isinstance(m, torch.nn.Embedding):
                    m.weight[1:].copy_(torch.randn(m.weight[1:].shape, generator=gen) * 0.3)
        mat = G.synthetic_matrix(fm, 3 * 32, gen, seq_min=0)
        G.run_model_case("model_BST_" + name, model, fm, mat, {"case": name, "kwargs": kwargs, "seed": 2023})


if __name__ == "__main__":
    M = bst_module()
    case_init(M)
    case_blocks(M)
    case_models(M)

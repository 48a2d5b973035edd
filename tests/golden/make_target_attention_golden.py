"""Generates the MultiHeadTargetAttention construction fixture by running the REAL reference, with
make_golden.py's helpers and settings (reference import stubs, one thread, deterministic algorithms), so no
other fixture changes.  Run in the build container only:

    python tests/golden/make_target_attention_golden.py

Writes
  target_attention_init.json  state_dict keys, dtypes, shapes and the SHA-256 of each tensor of the reference's
                              MultiHeadTargetAttention right after construction under torch.manual_seed(4747),
                              for five (input_dim, attention_dim, num_heads, use_qkvo) configurations.
"""
import hashlib
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_golden as G  # noqa: E402  (imports the reference)

torch = G.torch

INIT_CONFIGS = [(12, 12, 1, True), (12, 12, 3, True), (12, 12, 2, False), (64, 64, 4, True), (16, 40, 5, True)]


def case_init():
    init = {}
    for (d, A, H, qkvo) in INIT_CONFIGS:
        torch.manual_seed(4747)
        layer = G.L.MultiHeadTargetAttention(input_dim=d, attention_dim=A, num_heads=H, use_qkvo=qkvo)
        init["d%d_A%d_H%d_qkvo%d" % (d, A, H, int(qkvo))] = {
            "args": [d, A, H, qkvo], "seed": 4747,
            "state_dict": [[k, str(v.dtype), list(v.shape),
                            hashlib.sha256(v.detach().contiguous().numpy().tobytes()).hexdigest()]
                           for k, v in layer.state_dict().items()],
            "children": [name for name, _ in layer.named_children()]}
    path = os.path.join(G.HERE, "target_attention_init.json")
    with open(path, "w") as fd:
        json.dump(init, fd, indent=1, sort_keys=True)
    print("wrote", path)


if __name__ == "__main__":
    case_init()

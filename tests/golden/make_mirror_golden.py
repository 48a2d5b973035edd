"""Generates tests/golden/mirror_init.json: for every constructor case of
tests/test_host_logic.py::_MIRROR_CASES, what the REAL reference model class builds under
torch.manual_seed(4242) — state_dict keys in order, dtype, shape and a SHA-256 of each tensor's bytes,
and the module tree (names, and the torch type of every stock module).  Needs the reference
installed under oracle/_ref (python oracle/install_ref.py); the tests read only the JSON.

    python tests/golden/make_mirror_golden.py
"""
import hashlib
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import torch  # noqa: E402

from baseline import refenv  # noqa: E402
from test_host_logic import _MIRROR_CASES, mirror_case_id  # noqa: E402


def tensor_digest(t):
    return hashlib.sha256(t.detach().contiguous().cpu().numpy().tobytes()).hexdigest()


def main():
    refenv.import_reference()
    out = {}
    for i, (name, specs, kwargs) in enumerate(_MIRROR_CASES):
        cls = refenv.load_model_class(name)
        torch.manual_seed(4242)
        ref = cls(refenv.synthetic_feature_map(specs, embedding_dim=kwargs["embedding_dim"]),
                  model_root="/tmp/b2_mirror/", metrics=["AUC"], verbose=0, gpu=-1, optimizer="adam",
                  loss="binary_crossentropy", **kwargs)
        out[mirror_case_id(i)] = {
            "state_dict": [[k, str(v.dtype), list(v.shape), tensor_digest(v)] for k, v in ref.state_dict().items()],
            "modules": {m: (type(mod).__module__ + "." + type(mod).__name__
                            if type(mod).__module__.startswith("torch.") else None)
                        for m, mod in ref.named_modules()},
        }
    with open(os.path.join(HERE, "mirror_init.json"), "w") as fd:
        json.dump(out, fd, indent=1, sort_keys=True)


if __name__ == "__main__":
    main()

import json
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


class Golden(object):
    """One tests/golden/<name>.npz produced by the real reference (make_golden.py)."""

    def __init__(self, name):
        import torch
        blob = np.load(os.path.join(GOLDEN, name + ".npz"), allow_pickle=False)
        self.meta = json.loads(str(blob["meta"]))
        self.groups = {}
        for key in blob.files:
            if key == "meta":
                continue
            group, _, rest = key.partition("/")
            self.groups.setdefault(group, {})[rest] = torch.from_numpy(np.array(blob[key]))

    def __getitem__(self, group):
        return self.groups.get(group, {})

    def specs(self):
        from collections import OrderedDict
        return OrderedDict((k, v) for k, v in self.meta["specs"])


@pytest.fixture
def golden():
    return Golden


def rel_err(a, b):
    """max |a-b| / max(|b|_inf, tiny): the 1e-5 'relative fp32' bar of BASELINE.json's north_star."""
    import torch
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    denom = max(float(b.abs().max()), 1e-30)
    return float((a - b).abs().max()) / denom


def close(a, b, rtol, atol=1e-6):
    """|a-b|_inf <= rtol * |b|_inf + atol.  atol covers quantities that are mathematically zero
    (e.g. the last-bias gradient under a softmax) where only rounding noise remains."""
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).abs().max()) <= rtol * float(b.abs().max()) + atol

"""The LongCTR data loader on the H100: the device triple of b2_longctr_collate bit for bit against the reference
collator's goldens; ETA, SDIM, SIM, TWIN and MIRRN trained by the loader against the same models trained on the golden
triples; a LongCTRPipeline epoch with the captured step against an eager loop; evaluate / predict over the loader."""
import os
import sys

import numpy as np
import pytest
import torch

from conftest import close, rel_err

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_longctr_loader_host import MK, feature_map, load_golden, make_loader  # noqa: E402

pytestmark = pytest.mark.gpu

COMMON = dict(dnn_hidden_units=[16, 8], dnn_activations="ReLU", attention_dim=8, net_dropout=0, batch_norm=False)
# the configurations of each model's reference-trajectory test, and that test's tolerance on the weights after 3 steps
MODELS = {
    "ETA": (dict(embedding_dim=4, reuse_hash=True, hash_bits=32, topk=5, short_seq_len=4, num_heads=2, use_scale=True,
                 **COMMON), 2e-5, 1e-7),
    "SDIM": (dict(embedding_dim=4, reuse_hash=True, num_hashes=3, hash_bits=3, l2_norm=True, use_qkvo=True,
                  short_seq_len=4, num_heads=2, use_scale=True, **COMMON), 2e-5, 1e-7),
    "SIM": (dict(embedding_dim=4, num_heads=2, topk=5, short_seq_len=4, alpha=0.7, beta=1.3, **COMMON), 2e-5, 1e-7),
    "TWIN": (dict(embedding_dim=4, num_heads=2, topk=5, short_seq_len=4, **COMMON), 2e-5, 1e-7),
    "MIRRN": (dict(embedding_dim=4, reuse_hash=True, hash_bits=16, topk=5, short_seq_len=4, num_heads=2,
                   use_scale=True, max_len=24, **COMMON), 5e-5, 1e-6),
}


@pytest.fixture(scope="module", autouse=True)
def _built():
    import __graft_entry__
    __graft_entry__.build()
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"


@pytest.fixture(autouse=True)
def _fp32():
    from fuxictr_b200 import functional as F2
    F2.set_matmul_precision("fp32")
    yield
    F2.set_matmul_precision("fp32")


def golden_triples(case, device="cuda"):
    out = []
    for b in load_golden(case)[1]:
        out.append(({k: torch.from_numpy(v).to(device) for k, v in b["bd"].items()},
                    {k: torch.from_numpy(v).to(device) for k, v in b["item"].items()},
                    torch.from_numpy(b["mask"]).to(device)))
    return out


@pytest.mark.parametrize("case", list(MK.CASES))
def test_device_triples_are_bit_exact(case):
    meta, batches = load_golden(case)
    loader = make_loader(case)
    torch.manual_seed(7)
    got = list(loader)
    assert len(got) == len(batches) == len(loader)
    for (bd, items, mask), ref in zip(got, batches):
        assert list(bd) == meta["batch_keys"] and list(items) == meta["item_keys"]
        assert mask.is_cuda and mask.dtype == torch.float32 and tuple(mask.shape) == ref["mask"].shape
        assert torch.equal(mask.cpu(), torch.from_numpy(ref["mask"]))
        for group, want in (("bd", bd), ("item", items)):
            for k, v in ref[group].items():
                r = torch.from_numpy(v)
                t = want[k]
                assert t.is_cuda and t.dtype == r.dtype and t.shape == r.shape, (group, k, t.dtype, t.shape)
                assert torch.equal(t.cpu(), r), (group, k)


def _model(name, fm, seed=777):
    from fuxictr_b200 import zoo
    kw = MODELS[name][0]
    torch.manual_seed(seed)
    model = getattr(zoo, name)(fm, gpu=0, **kw)
    if name == "MIRRN":         # the filter dropout off, as MIRRN's trajectory test has it
        for blk in model.MHFT_block:
            blk.out_dropout.p = 0.0
    with torch.no_grad():
        for m in model.modules():
            if isinstance(m, torch.nn.Embedding):
                m.weight[1:].normal_(0, 0.1)
    model.train()
    model.use_fused_optimizer()
    return model


@pytest.mark.parametrize("name", list(MODELS))
def test_models_trained_by_the_loader_follow_the_golden_triples(name):
    case = "train_pre_shuffled_ml12"
    _, rtol, atol = MODELS[name]
    fm = feature_map(embedding_dim=4)
    fed, ref = _model(name, fm), _model(name, fm)
    torch.manual_seed(7)
    got = []
    for i, triple in enumerate(make_loader(case)):
        if i == 3:
            break
        got.append(float(fed.fused_train_step(triple).detach()))
    want = [float(ref.fused_train_step(t).detach()) for t in golden_triples(case)[:3]]
    assert close(torch.tensor(got), torch.tensor(want), 1e-5), (got, want)
    sd, sd_ref = fed.state_dict(), ref.state_dict()
    for k, v in sd_ref.items():
        assert close(sd[k], v, rtol, atol=atol), (k, rel_err(sd[k], v))


@pytest.mark.parametrize("name", ["ETA", "TWIN"])
def test_pipeline_epoch_with_graph_matches_an_eager_loop(name):
    """train_pre_unshuffled_ml12 pads batches to L = 12, 12, 12, 6, 12, 12, 12 with a last batch of 11 rows: two
    eager full steps, the capture at the third, an eager L = 6 step, two replays and an eager partial batch."""
    from fuxictr_b200.pipeline import LongCTRPipeline
    case = "train_pre_unshuffled_ml12"
    fm = feature_map(embedding_dim=4)
    piped, ref = _model(name, fm), _model(name, fm)
    loader = make_loader(case)
    pipe = LongCTRPipeline(piped, loader, graph=True)
    got = pipe.epoch()
    assert pipe.graph is not None
    want = [float(ref.fused_train_step(t).detach()) for t in golden_triples(case)]
    assert len(got) == len(want) == 7
    assert close(torch.tensor(got), torch.tensor(want), 1e-5), (got, want)
    sd, sd_ref = piped.state_dict(), ref.state_dict()
    _, rtol, atol = MODELS[name]
    for k, v in sd_ref.items():
        assert close(sd[k], v, rtol, atol=atol), (k, rel_err(sd[k], v))
    got2 = pipe.epoch()                     # a second epoch replays the captured shape again
    want2 = [float(ref.fused_train_step(t).detach()) for t in golden_triples(case)]
    assert close(torch.tensor(got2), torch.tensor(want2), 1e-5), (got2, want2)


@pytest.mark.parametrize("case", ["valid_pre_unshuffled_ml64_one_col", "train_pre_shuffled_ml12"])
def test_evaluate_and_predict_over_the_loader(case):
    keep = MK.CASES[case][5]
    fm = feature_map(keep, embedding_dim=4)
    model = _model("ETA", fm)
    model.eval()
    torch.manual_seed(7)
    pred = model.predict(make_loader(case))
    want = model.predict(golden_triples(case))
    assert pred.dtype == np.float64 and np.array_equal(pred, want)
    torch.manual_seed(7)
    res = model.evaluate(make_loader(case), ["logloss", "AUC"])
    res_ref = model.evaluate(golden_triples(case), ["logloss", "AUC"])
    assert res == res_ref, (res, res_ref)

"""torchrun script (N GPUs, REAL ranks over NVLink peer memory + NCCL): evaluation of a row-sharded model.  After 2
training steps, every rank evaluates its shard of a validation split of k * batch_local * world + 3 rows
(MatrixDataLoader(shard=(rank, world), drop_last=False): a ragged last round, with 0 rows on some ranks when
world > 3).  The metrics must be identical on every rank, bit for bit, and equal the CPU ORACLE
(oracle/fuxictr_oracle.py) trained the same 2 steps and evaluated on the whole split, within 1e-5 relative;
predict() must return this rank's rows of the oracle's predictions.

    python -m torch.distributed.run --nproc-per-node 2 --master-addr 127.0.0.1 tools/dist_sharded_eval_check.py \
        [--model DLRM|DIN] [--precision fp32|tf32x3] [--batch-local 64]

Checker use of oracle/ only (tests/test_gpu_multirank_eval.py launches this script).
"""
import argparse
import os
import sys
from collections import OrderedDict

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
ap = argparse.ArgumentParser()
ap.add_argument("--model", default="DLRM", choices=["DLRM", "DIN"])
ap.add_argument("--precision", default="fp32", choices=["fp32", "tf32x3"])
ap.add_argument("--batch-local", type=int, default=64)
args = ap.parse_args()

rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
torch.cuda.set_device(local)
dist.init_process_group("nccl", device_id=torch.device("cuda", local))
import __graft_entry__  # noqa: E402

if rank == 0:
    __graft_entry__.build()
dist.barrier()
from fuxictr_b200 import zoo, sharded as SH, functional as F2  # noqa: E402
from fuxictr_b200.dataloader import MatrixDataLoader  # noqa: E402
from fuxictr_b200.schema import FeatureMap  # noqa: E402
from oracle import fuxictr_oracle as O  # noqa: E402

F2.set_matmul_precision(args.precision)
B_l, HIST, HID = args.batch_local, 10, [32, 16]
if args.model == "DIN":
    D = 8
    specs = [
        ("user", {"type": "categorical", "source": "", "padding_idx": 0, "vocab_size": 300}),
        ("item_id", {"type": "categorical", "source": "", "padding_idx": 0, "vocab_size": 500}),
        ("cate_id", {"type": "categorical", "source": "", "padding_idx": 0, "vocab_size": 40}),
        ("click_history", {"type": "sequence", "source": "", "padding_idx": 0, "vocab_size": 500, "max_len": HIST,
                           "share_embedding": "item_id"}),
        ("cate_history", {"type": "sequence", "source": "", "padding_idx": 0, "vocab_size": 40, "max_len": HIST,
                          "share_embedding": "cate_id"}),
    ]
else:
    D = 16
    specs = [("C%d" % i, {"type": "categorical", "source": "", "padding_idx": 0, "vocab_size": 50 + 37 * i})
             for i in range(26)]
spec_map = OrderedDict(specs)
fm = FeatureMap.from_specs(specs, embedding_dim=D)
DIN_FIELDS = dict(din_target_field=[("item_id", "cate_id")], din_sequence_field=[("click_history", "cate_history")])


def make_model():
    torch.manual_seed(7)
    if args.model == "DLRM":
        m = zoo.DLRM(fm, gpu=local, embedding_dim=D, top_mlp_units=HID, interaction_op="dot")
    else:
        m = zoo.DIN(fm, gpu=local, embedding_dim=D, dnn_hidden_units=HID, attention_hidden_units=[16],
                    attention_hidden_activations="Dice", **DIN_FIELDS)
    with torch.no_grad():
        for mod in m.modules():
            if isinstance(mod, torch.nn.Embedding):
                mod.weight[1:].normal_(0, 0.1)
    return m


def rows(gen, n):
    if args.model == "DIN":       # post-padded histories of random length (all-padding and full rows included)
        cols = [torch.randint(0, s["vocab_size"], (n, 1), generator=gen) for _, s in specs[:3]]
        keep = torch.arange(HIST).view(1, -1) < torch.randint(0, HIST + 1, (n, 1), generator=gen)
        for _, s in specs[3:]:
            h = torch.randint(1, s["vocab_size"], (n, HIST), generator=gen)
            cols.append(torch.where(keep, h, torch.zeros_like(h)))
        ids = torch.cat(cols, 1)
    else:
        ids = torch.cat([torch.randint(0, s["vocab_size"], (n, 1), generator=gen) for _, s in specs], 1)
    return torch.cat([ids.double(), (torch.rand(n, 1, generator=gen) < 0.3).double()], 1)


gen = torch.Generator().manual_seed(11)
# DIN's Dice attention keeps running statistics of each rank's LOCAL training batches, which the oracle trained on
# the global batch does not share: DIN is evaluated as initialised (both at the initial statistics), DLRM after
# 2 training steps
batches = [rows(gen, B_l * world) for _ in range(2 if args.model == "DLRM" else 0)]
valid = rows(gen, 2 * B_l * world + 3).numpy()

model = make_model()
state0 = OrderedDict((k, v.detach().cpu().clone()) for k, v in model.state_dict().items())
if args.model == "DLRM":
    pred = lambda s, X: O.dlrm_pred(spec_map, s, X, len(HID))                        # noqa: E731
else:                             # eval(): Dice normalises with its running statistics
    pred = lambda s, X: O.din_pred(spec_map, s, X, D, DIN_FIELDS["din_target_field"],  # noqa: E731
                                   DIN_FIELDS["din_sequence_field"], 1, len(HID), training=False)
trainer = O.OracleTrainer(state0, pred, spec_map, ["label"])
for b in batches:
    trainer.train_step(fm.batch_dict(b))
with torch.no_grad():
    y_pred, y_true = trainer.forward(fm.batch_dict(torch.from_numpy(valid)))
ref_pred = y_pred.detach().double().reshape(-1).numpy()
ref = O.evaluate_metrics(y_true.detach().double().reshape(-1).numpy(), ref_pred, ["logloss", "AUC"])

model.enable_sharding(SH.SymmPeerGroup(), B_l, fm.input_length + 1, torch.float64, want_fm=False)
model.use_fused_optimizer()
model.train()
for b in batches:
    model.fused_train_step(fm.batch_dict(b[rank * B_l:(rank + 1) * B_l].contiguous().cuda()))
loader = MatrixDataLoader(fm, valid, batch_size=B_l, shard=(rank, world), drop_last=False, pin=False)
got = model.evaluate(loader, ["logloss", "AUC"])
mine = model.predict(loader)
model.train()

ok = True
vals = torch.tensor([got["logloss"], got["AUC"]], dtype=torch.float64, device="cuda")
every = [torch.empty_like(vals) for _ in range(world)]
dist.all_gather(every, vals)
same = all(torch.equal(e, every[0]) for e in every)        # bit for bit on every rank
ok &= same
for k in ref:
    e = abs(got[k] - ref[k]) / abs(ref[k])
    ok &= e < 1e-5
    print("[r%d] %s %s %.10f oracle %.10f rel err %.2e" % (rank, args.model, k, got[k], ref[k], e), flush=True)
my_rows = np.concatenate([np.arange(lo, hi) for lo, hi in loader._spans()])
perr = float(np.abs(mine - ref_pred[my_rows]).max()) if my_rows.size else 0.0
ok &= mine.shape == (my_rows.size,) and perr < 1e-5
print("[r%d] identical on every rank: %s; %d own rows, predict err %.2e -> %s"
      % (rank, same, my_rows.size, perr, "OK" if ok else "FAIL"), flush=True)
flag = torch.tensor([0 if ok else 1], device="cuda")
dist.all_reduce(flag)
dist.barrier()
os._exit(0 if int(flag.item()) == 0 else 1)

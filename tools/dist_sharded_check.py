"""torchrun script (N GPUs, REAL ranks over NVLink peer memory + NCCL): a row-sharded model trained for 3
steps on its slice of the global batch must equal the CPU ORACLE (oracle/fuxictr_oracle.py, the
restatement of the reference's BaseModel.train_step) run on the whole global batch: per-step global
mean loss, this rank's table shards and the replicated dense weights, within 1e-5 relative.

    python -m torch.distributed.run --nproc-per-node 2 --master-addr 127.0.0.1 tools/dist_sharded_check.py \
        [--model DeepFM|DLRM|DCNv2|xDeepFM|DIN] [--precision fp32|tf32x3] [--batch-local 64] [--lazy]

--lazy evaluates the tables' dense Adam lazily (use_fused_optimizer(lazy_tables=True)): the push replays
stale rows, the pull enqueues touched rows, and state_dict() brings every shard row up to date.

DIN has two post-padded histories that share the item_id / cate_id tables.  Its Dice attention normalises
over the batch, and every rank uses its LOCAL batch's statistics, so its oracle step is the data-parallel one:
the oracle model on each rank's slice, loss scaled by 1/world, gradients summed, one step; the running
statistics follow each rank's own batches and are not compared.

Checker use of oracle/ only (tests/test_gpu_multirank.py launches this script).
"""
import argparse
import os
import sys
from collections import OrderedDict

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
ap = argparse.ArgumentParser()
ap.add_argument("--model", default="DeepFM", choices=["DeepFM", "DLRM", "DCNv2", "xDeepFM", "DIN"])
ap.add_argument("--precision", default="fp32", choices=["fp32", "tf32x3"])
ap.add_argument("--batch-local", type=int, default=64)
ap.add_argument("--lazy", action="store_true", help="lazily evaluated tables (dense Adam semantics, row-wise)")
args = ap.parse_args()

rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
torch.cuda.set_device(local)
dist.init_process_group("nccl", device_id=torch.device("cuda", local))
import __graft_entry__  # noqa: E402

if rank == 0:
    __graft_entry__.build()
dist.barrier()
from fuxictr_b200 import zoo, sharded as SH, functional as F2  # noqa: E402
from fuxictr_b200.schema import FeatureMap  # noqa: E402
from oracle import fuxictr_oracle as O  # noqa: E402

F2.set_matmul_precision(args.precision)
NF, D, B_l = (26, 16, args.batch_local) if args.model == "DLRM" else (12, 8, args.batch_local)
HIST = 10
if args.model == "DIN":
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
    specs = [("C%d" % i, {"type": "categorical", "source": "", "padding_idx": 0, "vocab_size": 50 + 37 * i})
             for i in range(NF)]
spec_map = OrderedDict(specs)
fm = FeatureMap.from_specs(specs, embedding_dim=D)
HID = [32, 16]
CIN = [8, 8]
DIN_FIELDS = dict(din_target_field=[("item_id", "cate_id")], din_sequence_field=[("click_history", "cate_history")])


def make_model():
    torch.manual_seed(7)
    if args.model == "DeepFM":
        m = zoo.DeepFM(fm, gpu=local, embedding_dim=D, hidden_units=HID)
    elif args.model == "DLRM":
        m = zoo.DLRM(fm, gpu=local, embedding_dim=D, top_mlp_units=HID, interaction_op="dot")
    elif args.model == "DCNv2":
        m = zoo.DCNv2(fm, gpu=local, embedding_dim=D, model_structure="parallel", num_cross_layers=2,
                      parallel_dnn_hidden_units=HID)
    elif args.model == "xDeepFM":
        m = zoo.xDeepFM(fm, gpu=local, embedding_dim=D, dnn_hidden_units=HID, cin_hidden_units=CIN)
    else:
        m = zoo.DIN(fm, gpu=local, embedding_dim=D, dnn_hidden_units=HID, attention_hidden_units=[16],
                    attention_hidden_activations="Dice", **DIN_FIELDS)
    with torch.no_grad():
        for mod in m.modules():
            if isinstance(mod, torch.nn.Embedding):
                mod.weight[1:].normal_(0, 0.1)
    return m


gen = torch.Generator().manual_seed(11)
batches = []
for step in range(3):
    n = B_l * world
    if args.model == "DIN":       # post-padded histories of random length (all-padding and full rows included)
        cols = [torch.randint(0, s["vocab_size"], (n, 1), generator=gen) for _, s in specs[:3]]
        keep = torch.arange(HIST).view(1, -1) < torch.randint(0, HIST + 1, (n, 1), generator=gen)
        for _, s in specs[3:]:
            h = torch.randint(1, s["vocab_size"], (n, HIST), generator=gen)
            cols.append(torch.where(keep, h, torch.zeros_like(h)))
        ids = torch.cat(cols, 1)
    else:
        ids = torch.cat([torch.randint(0, s["vocab_size"], (n, 1), generator=gen) for _, s in specs], 1)
    lab = (torch.rand(n, 1, generator=gen) < 0.3)
    batches.append(torch.cat([ids.double(), lab.double()], 1))

# the checker: the reference's train_step restated on CPU, on the GLOBAL batch
model = make_model()
state0 = OrderedDict((k, v.detach().cpu().clone()) for k, v in model.state_dict().items())
if args.model == "DeepFM":
    pred = lambda s, X: torch.sigmoid(O.deepfm_logit(spec_map, s, X, len(HID)))      # noqa: E731
elif args.model == "DLRM":
    pred = lambda s, X: O.dlrm_pred(spec_map, s, X, len(HID))                        # noqa: E731
elif args.model == "DCNv2":
    pred = lambda s, X: torch.sigmoid(O.dcnv2_logit(spec_map, s, X, 2, len(HID)))     # noqa: E731
elif args.model == "xDeepFM":
    pred = lambda s, X: torch.sigmoid(O.xdeepfm_logit(spec_map, s, X, CIN, len(HID)))  # noqa: E731
else:
    pred = lambda s, X: O.din_pred(spec_map, s, X, D, DIN_FIELDS["din_target_field"],  # noqa: E731
                                   DIN_FIELDS["din_sequence_field"], 1, len(HID))
trainer = O.OracleTrainer(state0, pred, spec_map, ["label"])


def data_parallel_step(b):
    """One oracle step from every rank's slice: loss / world per slice, gradients summed (Dice: local statistics)."""
    trainer.optimizer.zero_grad()
    total = 0.0
    for r in range(world):
        y_pred, y = trainer.forward(fm.batch_dict(b[r * B_l:(r + 1) * B_l]))
        loss = O.bce_mean(y_pred, y) / world
        loss.backward()
        total += float(loss)
    torch.nn.utils.clip_grad_norm_(trainer.params, trainer.max_norm)
    trainer.optimizer.step()
    return total


if args.model == "DIN":
    ref_losses = [data_parallel_step(b) for b in batches]
else:
    ref_losses = [float(trainer.train_step(fm.batch_dict(b))) for b in batches]

model.enable_sharding(SH.SymmPeerGroup(), B_l, fm.input_length + 1, torch.float64, want_fm=(args.model == "DeepFM"))
model.use_fused_optimizer(lazy_tables=args.lazy)
model.train()
losses = []
mine = [b[rank * B_l:(rank + 1) * B_l].contiguous().cuda() for b in batches]
for b in mine:
    losses.append(model.fused_train_step(fm.batch_dict(b)).detach().clone())
lt = torch.stack(losses)
dist.all_reduce(lt)
lt /= world          # global mean loss


def rel(a, b):
    return float((a - b).abs().max()) / max(float(b.abs().max()), 1e-30)


tol = 1e-5
ok = True
err = rel(lt.cpu(), torch.tensor(ref_losses))
ok &= err < tol
print("[r%d] %s%s loss err %.2e" % (rank, args.model, " lazy" if args.lazy else "", err), flush=True)
worst = 0.0
for k, v in model.state_dict().items():
    if args.model == "DIN" and ("running_" in k or "num_batches" in k):
        continue                # Dice's running statistics follow this rank's own batches
    r = trainer.state[k].detach()
    if not r.dtype.is_floating_point:       # frozen index buffers (triu masks): identical or wrong
        ok &= bool(torch.equal(v.cpu(), r))
        continue
    if "embedding_layers" in k:
        r = SH.shard_rows(r, rank, world)
    e = rel(v.cpu(), r)
    worst = max(worst, e)
    if e >= tol:
        print("[r%d] MISMATCH %s %.2e" % (rank, k, e), flush=True)
        ok = False
print("[r%d] worst weight err after 3 steps %.2e -> %s" % (rank, worst, "OK" if ok else "FAIL"), flush=True)
flag = torch.tensor([0 if ok else 1], device="cuda")
dist.all_reduce(flag)
dist.barrier()
os._exit(0 if int(flag.item()) == 0 else 1)

"""MultiHeadTargetAttention on the H100: the layer (pack, GEMM1, row kernel, GEMM2 and back) against the
reference's goldens and against the oracle in float64 across the row kernels' launch-plan branches in every
matmul mode; the unmodified reference layer in a small model on cuda:0 under patch.enable() against itself on
CPU through three Adam steps; and forward + backward captured in a CUDA graph."""
import copy
import sys

import pytest
import torch

from conftest import Golden, ROOT, close, rel_err

sys.path.insert(0, ROOT)
from oracle import fuxictr_oracle as O  # noqa: E402
from baseline import refenv  # noqa: E402

pytestmark = pytest.mark.gpu

RTOL = 1e-5
# single-pass modes: the Frobenius bars of test_gpu_parity.py::test_mlp_chain_matches_torch_autograd
FRO = {"tf32": (1e-2, 6e-2), "bf16": (3e-2, 1.5e-1)}


@pytest.fixture(scope="module", autouse=True)
def _built():
    import __graft_entry__
    __graft_entry__.build()
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"


@pytest.fixture
def mode_of():
    from fuxictr_b200 import functional as F2

    def set_mode(mode):
        F2.set_matmul_precision(mode)
    yield set_mode
    F2.set_matmul_precision("fp32")


def fro(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


@pytest.mark.parametrize("mode", ["fp32", "tf32x3"])
@pytest.mark.parametrize("name", ["h1_qkvo1", "h3_qkvo1", "h2_qkvo0"])
def test_layer_matches_reference_golden(name, mode, mode_of):
    from fuxictr_b200 import layers
    g = Golden("next_MHTA_" + name)
    m = g.meta
    d = g["in"]["target"].shape[1]
    layer = layers.MultiHeadTargetAttention(input_dim=d, attention_dim=d, num_heads=m["heads"],
                                            use_scale=m["use_scale"], use_qkvo=m["use_qkvo"])
    layer.load_state_dict(g["w"])
    layer = layer.cuda()
    mode_of(mode)
    t = g["in"]["target"].cuda().requires_grad_(True)
    x = g["in"]["history"].cuda().requires_grad_(True)
    out = layer(t, x, g["in"]["mask"].cuda())
    assert close(out, g["out"]["y"], RTOL), rel_err(out, g["out"]["y"])
    (out * g["in"]["gout"].cuda()).sum().backward()
    assert close(t.grad, g["gin"]["target"], RTOL), rel_err(t.grad, g["gin"]["target"])
    assert close(x.grad, g["gin"]["history"], RTOL), rel_err(x.grad, g["gin"]["history"])
    named = dict(layer.named_parameters())
    scale = max([float(v.abs().max()) for v in g["g"].values()] + [1e-30])
    for k, want in g["g"].items():
        assert close(named[k].grad, want, RTOL, atol=RTOL * scale), (k, rel_err(named[k].grad, want))


# (B, L, d, attention_dim, heads, use_qkvo, mask): L 1, below (31), at (32) and above (33) the 32-position
# chunk, and 200; hd 6 (sliced d 12 / 2 heads, d 30 / 5 heads without 16-byte loads, folded d 6); B not a multiple
# of the 8 rows per CTA and B 8192; all-masked rows ("padded": every third row only padding), bool and float masks
# and none; the width bound (folded 4 x 256, sliced 1024: one warp per CTA, over 48 KB of shared memory); SIMT
# GEMMs (d 12, the SIM / ETA item width) and tensor-core GEMMs (d 64).
SHAPES = [(5, 1, 12, 12, 2, True, "float"), (7, 31, 12, 12, 2, True, "padded"), (9, 32, 12, 64, 2, True, "bool"),
          (9, 33, 64, 64, 4, True, "padded"), (37, 200, 64, 64, 4, True, "bool"), (8192, 50, 12, 64, 2, True, "padded"),
          (6, 50, 12, 12, 2, False, "padded"), (11, 40, 12, 12, 3, False, None), (6, 45, 30, 30, 5, False, "float"),
          (4, 17, 6, 6, 1, True, None), (5, 20, 256, 256, 4, True, "float"), (3, 70, 1024, 1024, 2, False, "bool"),
          (8192, 50, 64, 64, 4, True, "padded"), (8192, 50, 12, 12, 2, False, "padded")]


def make_inputs(B, L, d, mask_kind, gen):
    t = torch.randn(B, d, generator=gen) * 0.5
    x = torch.randn(B, L, d, generator=gen) * 0.5
    mask = None
    if mask_kind is not None:
        lens = torch.randint(1, L + 1, (B,), generator=gen)
        mask = (torch.arange(L)[None, :] < lens[:, None])
        if mask_kind == "padded":
            mask[::3] = False
        mask = mask.float() if mask_kind in ("float", "padded") else mask
    return t, x, mask


@pytest.mark.parametrize("mode", ["fp32", "tf32x3", "tf32", "bf16"])
@pytest.mark.parametrize("B,L,d,A,H,qkvo,mask_kind", SHAPES)
def test_layer_matches_float64_oracle(mode, B, L, d, A, H, qkvo, mask_kind, mode_of):
    from fuxictr_b200 import layers
    torch.manual_seed(B + L + d + H)
    layer = layers.MultiHeadTargetAttention(input_dim=d, attention_dim=A, num_heads=H, use_qkvo=qkvo)
    state = {k: v.detach().double().cuda().requires_grad_(True) for k, v in layer.state_dict().items()}
    gen = torch.Generator().manual_seed(d * 7 + B + L)
    t, x, mask = make_inputs(B, L, d, mask_kind, gen)
    gout = torch.randn(B, d, generator=gen)
    mask_c = mask.cuda() if mask is not None else None
    tr, xr = t.double().cuda().requires_grad_(True), x.double().cuda().requires_grad_(True)
    yr = O.multi_head_target_attention(state, "", tr, xr, mask_c, H, True, qkvo)
    yr.backward(gout.double().cuda())
    layer = layer.cuda()
    mode_of(mode)
    tg, xg = t.cuda().requires_grad_(True), x.cuda().requires_grad_(True)
    yg = layer(tg, xg, mask_c)
    yg.backward(gout.cuda())
    named = dict(layer.named_parameters())
    pairs = [(tg.grad, tr.grad, "target"), (xg.grad, xr.grad, "history")] + \
        [(named[k].grad, ref.grad, k) for k, ref in state.items()]
    if L == 1:      # a softmax over one position is constant: the target, W_q and W_k get no gradient
        for got, ref, k in pairs[:1] + ([] if not qkvo else pairs[2:4]):
            assert float(ref.abs().max()) == 0.0 and float(got.abs().max()) <= 1e-6, k
        pairs = pairs[1:2] + (pairs[4:] if qkvo else [])
    if mode in ("fp32", "tf32x3") or not qkvo:       # no GEMM in the sliced form: fp32 in every mode
        assert close(yg, yr, RTOL), rel_err(yg, yr)
        for got, ref, k in pairs:
            assert close(got, ref, RTOL, atol=RTOL * float(ref.abs().max())), (k, rel_err(got, ref))
        return
    tol_y, tol = FRO[mode]
    assert fro(yg, yr) <= tol_y
    for got, ref, k in pairs:
        assert fro(got, ref) <= tol, k


def test_eval_mode_attention_dropout_runs_the_kernels():
    from fuxictr_b200 import layers
    torch.manual_seed(3)
    layer = layers.MultiHeadTargetAttention(input_dim=12, attention_dim=12, num_heads=2, dropout_rate=0.3).cuda()
    gen = torch.Generator().manual_seed(4)
    t, x, mask = make_inputs(6, 9, 12, "bool", gen)
    layer.eval()
    y = layer(t.cuda(), x.cuda(), mask.cuda())
    state = {k: v.detach().double() for k, v in layer.state_dict().items()}
    ref = O.multi_head_target_attention({k: v.cuda() for k, v in state.items()}, "", t.double().cuda(),
                                        x.double().cuda(), mask.cuda(), 2, True, True)
    assert close(y, ref, RTOL)


# ------------------------------------------------------------------ the unmodified reference layer under patch.enable()
def build_ref_model(R, d, vocab, L):
    class Tiny(torch.nn.Module):
        """An item embedding, the reference's MultiHeadTargetAttention over the history and an MLP_Block head."""

        def __init__(self):
            super().__init__()
            self.emb = torch.nn.Embedding(vocab, d, padding_idx=0)
            self.attention = R.layers.MultiHeadTargetAttention(input_dim=d, attention_dim=64, num_heads=2)
            self.mlp = R.layers.MLP_Block(input_dim=2 * d, output_dim=1, hidden_units=[32, 16],
                                          hidden_activations="ReLU")

        def forward(self, target_ids, history_ids):
            t, h = self.emb(target_ids), self.emb(history_ids)
            mask = history_ids != 0
            return self.mlp(torch.cat([t, self.attention(t, h, mask)], dim=1)).squeeze(1)

    return Tiny()


@pytest.mark.skipif(not refenv.available(), reason=refenv.why_unavailable())
@pytest.mark.parametrize("d", [12, 64])
def test_reference_target_attention_runs_on_the_kernels(d):
    from fuxictr_b200 import patch
    R = refenv.import_reference()
    B, L, vocab = 256, 50, 500
    torch.manual_seed(11)
    cpu_model = build_ref_model(R, d, vocab, L)
    with torch.no_grad():
        cpu_model.emb.weight[1:].normal_(0, 0.3)
    gpu_model = copy.deepcopy(cpu_model).cuda()
    gen = torch.Generator().manual_seed(12)
    batches = []
    for _ in range(3):
        lens = torch.randint(0, L + 1, (B,), generator=gen)          # 0: a history of padding only
        hist = torch.randint(1, vocab, (B, L), generator=gen) * (torch.arange(L)[None, :] < lens[:, None])
        batches.append((torch.randint(1, vocab, (B,), generator=gen), hist,
                        (torch.rand(B, generator=gen) < 0.3).float()))
    opts = [torch.optim.Adam(m.parameters(), lr=1e-3) for m in (cpu_model, gpu_model)]
    patch.enable()
    try:
        before = patch.call_counts().get("MultiHeadTargetAttention", 0)
        for step, (tid, hist, y) in enumerate(batches):
            losses, grads = [], []
            for m, opt, dev in ((cpu_model, opts[0], "cpu"), (gpu_model, opts[1], "cuda")):
                opt.zero_grad()
                out = m(tid.to(dev), hist.to(dev))
                loss = torch.nn.functional.binary_cross_entropy_with_logits(out, y.to(dev))
                loss.backward()
                if step == 0:
                    losses.append(out)
                grads.append({k: p.grad.detach().cpu() for k, p in m.named_parameters()})
                opt.step()
            if step == 0:
                assert losses[1].is_cuda and rel_err(losses[1], losses[0]) <= 1e-5, "forward differs"
            scale = max(float(g.abs().max()) for g in grads[0].values())
            for k, ref in grads[0].items():
                err = float((grads[1][k] - ref).abs().max())
                assert err <= 1e-5 * max(float(ref.abs().max()), 1e-3 * scale), "step %d grad %s: %g" % (step, k, err)
        assert patch.call_counts().get("MultiHeadTargetAttention", 0) - before == 3, "the kernel path was not taken"
        sd_ref, sd_gpu = cpu_model.state_dict(), gpu_model.state_dict()
        for k in sd_ref:
            err = float((sd_gpu[k].cpu() - sd_ref[k]).abs().max())
            assert err <= 1e-3 * 3e-3 + 1e-5 * float(sd_ref[k].abs().max()), "%s after 3 steps: %g" % (k, err)
    finally:
        patch.disable()


# ------------------------------------------------------------------ CUDA graph capture
@pytest.mark.parametrize("mode,d,qkvo", [("fp32", 12, True), ("tf32x3", 64, True), ("bf16", 64, True),
                                         ("fp32", 12, False)])
def test_cuda_graph_replay_matches_eager(mode, d, qkvo, mode_of):
    from fuxictr_b200 import layers
    mode_of(mode)
    torch.manual_seed(21)
    layer = layers.MultiHeadTargetAttention(input_dim=d, attention_dim=64 if qkvo else d, num_heads=2,
                                            use_qkvo=qkvo).cuda()
    gen = torch.Generator().manual_seed(22)
    t0, x0, mask = make_inputs(300, 50, d, "padded", gen)
    gout = torch.randn(300, d, generator=gen).cuda()
    t = t0.cuda().requires_grad_(True)
    x = x0.cuda().requires_grad_(True)
    mask = mask.cuda()
    params = [t, x] + list(layer.parameters())

    def step():
        for p in params:
            p.grad = None
        y = layer(t, x, mask)
        y.backward(gout)
        return y

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            want_y = step().detach().clone()
    torch.cuda.current_stream().wait_stream(side)
    want = [p.grad.detach().clone() for p in params]
    graph = torch.cuda.CUDAGraph()
    for p in params:
        p.grad = None
    with torch.cuda.graph(graph):
        y = layer(t, x, mask)
        y.backward(gout)
    with torch.no_grad():
        t.copy_(t0.cuda())
    graph.replay()
    torch.cuda.synchronize()
    assert close(y, want_y, 1e-6, atol=0.0)
    for p, w in zip(params, want):
        assert close(p.grad, w, 1e-6, atol=0.0)

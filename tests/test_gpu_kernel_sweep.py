"""The non-GEMM kernels against float64 at every branch of their launch plans.

Each test calls a kernel through its functional.py wrapper (or the C-ABI) and compares it with a plain
float64 restatement of the same operation: the oracle's restatement of the reference where it has one,
torch float64 autograd otherwise.  The bar is the C2 test's: run the restatement in float32 (what the
reference computes) and in float64 (the exact answer), then require for the output and every gradient
    err(ours, fp64) <= max(1e-5, 3 * err(reference fp32, fp64))          (max-norm, relative)
so a shape where fp32 arithmetic itself is unstable widens the bar by exactly that instability and no
more.  Operations that only copy data are held bit-exact."""
import sys
from collections import OrderedDict

import pytest
import torch

from conftest import rel_err, close, ROOT

sys.path.insert(0, ROOT)
pytestmark = pytest.mark.gpu

RTOL = 1e-5


@pytest.fixture(scope="module", autouse=True)
def _built():
    import __graft_entry__
    __graft_entry__.build()
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"


def bar(ours, ref32, ref64, what):
    e_ours, e_ref = rel_err(ours, ref64), rel_err(ref32, ref64)
    assert e_ours <= max(RTOL, 3 * e_ref), (what, e_ours, e_ref)


def grads_of(fn, inputs, gout, dtype, device="cpu"):
    """fn(*inputs) and the gradients of <fn, gout> w.r.t. every input, all in `dtype` on `device`."""
    xs = [x.detach().to(device=device, dtype=dtype).requires_grad_(True) for x in inputs]
    y = fn(*xs)
    y.backward(gout.to(device=device, dtype=dtype))
    return y.detach(), [x.grad for x in xs]


def check_against_fp64(fn, inputs, gout, y, grads, names, device="cpu"):
    y64, g64 = grads_of(fn, inputs, gout, torch.float64, device)
    y32, g32 = grads_of(fn, inputs, gout, torch.float32, device)
    bar(y, y32, y64, "out")
    for name, g, a, b in zip(names, grads, g32, g64):
        bar(g, a, b, name)


# ------------------------------------------------------------------ CrossNet (rank-1 cross, all layers fused)
def _crossnet_case(B, d, L, x_std=1.0, w_scale=1.0, b_std=0.1, seed=0):
    from fuxictr_b200 import layers
    from oracle import fuxictr_oracle as O
    gen = torch.Generator().manual_seed(seed * 7919 + d * 31 + L)
    x0 = torch.randn(B, d, generator=gen) * x_std
    w = torch.randn(L, d, generator=gen) * (w_scale / d ** 0.5)
    b = torch.randn(L, d, generator=gen) * b_std
    gout = torch.randn(B, d, generator=gen)
    layer = layers.CrossNet(d, L)
    with torch.no_grad():
        for i, m in enumerate(layer.cross_net):
            m.weight.weight.copy_(w[i:i + 1])
            m.bias.copy_(b[i])
    layer = layer.cuda()
    xg = x0.cuda().requires_grad_(True)
    y = layer(xg)
    y.backward(gout.cuda())
    gw = torch.cat([m.weight.weight.grad for m in layer.cross_net], 0)
    gb = torch.stack([m.bias.grad for m in layer.cross_net], 0)

    def ref(x, wt, bt):
        state = OrderedDict()
        for i in range(L):
            state["cross_net.%d.weight.weight" % i] = wt[i:i + 1]
            state["cross_net.%d.bias" % i] = bt[i]
        return O.crossnet(x, state, "", L)
    check_against_fp64(ref, [x0, w, b], gout, y, [xg.grad, gw, gb], ["gx0", "gw", "gb"])


# d crosses the register-chunk templates (CH = 4 | 8 | 20 | 32 chunks of 32 columns) and partial chunks
@pytest.mark.parametrize("d", [1, 31, 128, 129, 256, 257, 640, 641, 1024])
@pytest.mark.parametrize("L", [1, 3, 6])
def test_crossnet_sweep(d, L):
    _crossnet_case(300, d, L)


def test_crossnet_backward_over_48k_shared_memory():
    # 2 * L * d * 4 bytes = 56 KB of per-CTA gradient staging: the opt-in shared-memory launch
    _crossnet_case(300, 1024, 7)


def test_crossnet_batch_leaves_last_cta_partial():
    # 8 samples (warps) per CTA: 13 samples leave 3 warps of the second CTA without a sample
    _crossnet_case(13, 100, 3)


@pytest.mark.parametrize("B,d,x_std,w_scale", [(512, 416, 2.0, 2.0), (512, 624, 3.0, 3.0)])
def test_crossnet_backward_large_cross_scalars(B, d, x_std, w_scale):
    """|s_l| = |w_l . x_l| grows across layers.  The backward rebuilds x_l = alpha_l x_0 + beta_l from the
    saved scalars; alpha_l must be summed upward (1 + s_0 + ... + s_{l-1}), not peeled off alpha_L, or
    the subtraction cancels and gw loses digits."""
    _crossnet_case(B, d, 6, x_std=x_std, w_scale=w_scale, b_std=0.1, seed=1)


# ------------------------------------------------------------------ CIN (fused layers and the fallback)
def _cin_case(F_, units, D, B, seed=0):
    from fuxictr_b200 import layers
    from oracle import fuxictr_oracle as O
    torch.manual_seed(seed + F_ * 131 + D)
    layer = layers.CompressedInteractionNet(F_, units)
    with torch.no_grad():
        for p in layer.parameters():
            p.normal_(0, 0.2)
    names = [k for k, _ in layer.named_parameters()]
    params = [p.detach().clone() for p in layer.parameters()]
    gen = torch.Generator().manual_seed(B + D)
    emb = torch.randn(B, F_, D, generator=gen) * 0.5
    gout = torch.randn(B, 1, generator=gen)
    layer = layer.cuda()
    e = emb.cuda().requires_grad_(True)
    y = layer(e)
    y.backward(gout.cuda())
    named = dict(layer.named_parameters())

    def ref(x, *ps):
        return O.compressed_interaction_net(x, OrderedDict(zip(names, ps)), "", units)
    check_against_fp64(ref, [emb] + params, gout, y, [e.grad] + [named[k].grad for k in names],
                       ["gemb"] + names)


# H (the layer-1 input width, = F) crosses the dXk register templates HK = 16 | 40 | 64 and H' the
# accumulator templates HP = 8 | 16 | 32; the second layer (3 maps) runs with x_k != x_0, H = H'.
@pytest.mark.parametrize("H", [1, 16, 17, 40, 41, 64])
@pytest.mark.parametrize("HO", [1, 3, 8, 9, 16, 17, 32])
def test_cin_sweep(H, HO):
    D = [1, 7, 16, 33][(H + HO) % 4]
    _cin_case(H, [HO, 3], D, 37)           # B * D is never a multiple of the 256-column tile


@pytest.mark.parametrize("D", [1, 7, 16, 33])
def test_cin_embedding_dims(D):
    # F * H = 41 * 41 = 1681 weight columns: four k-slices of the weight-gradient kernel
    _cin_case(41, [17, 9, 32], D, 45)


@pytest.mark.parametrize("F_,units", [(8, [33, 8]), (65, [8])])
def test_cin_unfused_fallback(F_, units):
    from fuxictr_b200 import functional as F2
    assert not F2.cin_supported(F_, units)
    _cin_case(F_, units, 7, 37)


# ------------------------------------------------------------------ FM product_sum / bi_interaction / inner_product
@pytest.mark.parametrize("mode", [0, 1, 2])
@pytest.mark.parametrize("D", [1, 3, 10, 16, 17, 32, 33, 64, 100])
@pytest.mark.parametrize("F_", [2, 3, 39, 64])
def test_fm_sweep(mode, D, F_):
    """product_sum / bi_interaction: DP = 2^k lanes per sample (k capped at 5, so D > 32 loops);
    inner_product: a shared-memory tile of spb samples, spb halved from 8 until it fits 48 KB (F=64, D=100
    runs one sample per CTA)."""
    from fuxictr_b200 import functional as F2
    from oracle import fuxictr_oracle as O
    out_name = ["product_sum", "bi_interaction", "inner_product"][mode]
    B = 67
    gen = torch.Generator().manual_seed(mode * 1000 + D * 10 + F_)
    emb = torch.randn(B, F_, D, generator=gen) * 0.5
    P = F_ * (F_ - 1) // 2
    gout = torch.randn(*((B, 1) if mode == 0 else (B, D) if mode == 1 else (B, P)), generator=gen)
    e = emb.cuda().requires_grad_(True)
    y = F2.fm_interaction(e, mode)
    y.backward(gout.cuda())
    check_against_fp64(lambda x: O.inner_product_interaction(x, out_name), [emb], gout, y, [e.grad], ["gemb"])


def test_fm_inner_product_over_shared_memory_cap_is_refused():
    from fuxictr_b200 import functional as F2, _lib
    emb = torch.randn(4, 64, 200, device="cuda")      # one sample's tile alone is 51 KB > 48 KB
    with pytest.raises(_lib.B2Error):
        F2.fm_interaction(emb, 2)


# ------------------------------------------------------------------ Dice (train and eval)
def _dice_input(M, C, gen, special):
    x = torch.randn(M, C, generator=gen, dtype=torch.float64) * 1.5 + torch.randn(1, C, generator=gen,
                                                                                   dtype=torch.float64)
    if special:
        x[:, 0] = 1e3 + torch.randn(M, generator=gen, dtype=torch.float64)    # var = E[x^2] - mu^2 at mu = 1e3
        if C > 1:
            x[:, 1] = 0.3                                                       # var = 0: rstd = 1/sqrt(eps)
    return x.float()


def _dice_case(M, C, training, special=False):
    from fuxictr_b200 import layers
    gen = torch.Generator().manual_seed(M * 7 + C)
    x = _dice_input(M, C, gen, special)
    alpha = torch.randn(C, generator=gen) * 0.5
    gout = torch.randn(M, C, generator=gen)
    rm0 = torch.randn(C, generator=gen)
    rv0 = torch.rand(C, generator=gen) + 0.5
    layer = layers.Dice(C).cuda()
    with torch.no_grad():
        layer.alpha.copy_(alpha)
        layer.bn.running_mean.copy_(rm0)
        layer.bn.running_var.copy_(rv0)
    layer.train(training)
    xg = x.cuda().requires_grad_(True)
    y = layer(xg)
    y.backward(gout.cuda())

    def ref(dtype):
        bn = torch.nn.BatchNorm1d(C, affine=False, eps=1e-9, momentum=0.01).to(device="cuda", dtype=dtype)
        with torch.no_grad():
            bn.running_mean.copy_(rm0)
            bn.running_var.copy_(rv0)
        bn.train(training)
        xr = x.cuda().to(dtype).requires_grad_(True)
        ar = alpha.cuda().to(dtype).requires_grad_(True)
        p = torch.sigmoid(bn(xr))
        out = p * xr + ar * (1 - p) * xr                  # activations.py:49-50
        out.backward(gout.cuda().to(dtype))
        return out.detach(), xr.grad, ar.grad, bn.running_mean, bn.running_var
    r64, r32 = ref(torch.float64), ref(torch.float32)
    ours = (y, xg.grad, layer.alpha.grad, layer.bn.running_mean, layer.bn.running_var)
    for name, o, a, b in zip(["out", "gx", "galpha", "running_mean", "running_var"], ours, r32, r64):
        bar(o, a, b, name)


# C crosses the 32-column blocks of the statistics kernel; M crosses its 64-row splits (102,400 rows = C4)
@pytest.mark.parametrize("C", [1, 31, 32, 33, 64, 500])
@pytest.mark.parametrize("M", [2, 63, 64, 65, 4097, 102400])
@pytest.mark.parametrize("training", [True, False])
def test_dice_sweep(C, M, training):
    _dice_case(M, C, training)


@pytest.mark.parametrize("training", [True, False])
@pytest.mark.parametrize("M", [65, 4097])
def test_dice_offset_and_constant_columns(M, training):
    _dice_case(M, 33, training, special=True)


# ------------------------------------------------------------------ DIN attention glue
def _din_mask(B, L, kind, gen):
    if kind == "none":
        return None
    m = torch.rand(B, L, generator=gen) < 0.7
    m[:, 0] = True
    if kind == "row":
        m[1] = False                                     # one sample's history entirely masked
    return m


@pytest.mark.parametrize("d", [8, 32, 33, 64])
@pytest.mark.parametrize("L", [1, 31, 32, 33, 50, 200])
@pytest.mark.parametrize("mask_kind", ["none", "partial", "row"])
def test_din_glue_sweep(d, L, mask_kind):
    """att_in = [t, h, t-h, t*h], the masked softmax (one warp per row, L > 32 takes several lane passes)
    and the masked weighted sum (one warp per (b, l) in the backward, d > 32 loops), each forward and
    backward."""
    from fuxictr_b200 import functional as F2
    B = 37
    gen = torch.Generator().manual_seed(d * 1000 + L * 3 + len(mask_kind))
    t = torch.randn(B, d, generator=gen)
    h = torch.randn(B, L, d, generator=gen)
    w = torch.randn(B, L, generator=gen) * 2
    mask = _din_mask(B, L, mask_kind, gen)
    mask_u8 = mask.to(torch.uint8).cuda() if mask is not None else None
    mf = mask.double() if mask is not None else None

    # input construction (target_attention.py:80-82)
    g_in = torch.randn(B * L, 4 * d, generator=gen)
    tg, hg = t.cuda().requires_grad_(True), h.cuda().requires_grad_(True)
    att = F2._DinInput.apply(tg, hg)
    att.backward(g_in.cuda())
    att_ref = lambda t_, h_: torch.cat([t_.unsqueeze(1).expand(-1, L, -1), h_, t_.unsqueeze(1) - h_,
                                        t_.unsqueeze(1) * h_], dim=-1).view(-1, 4 * d)
    check_against_fp64(att_ref, [t, h], g_in, att, [tg.grad, hg.grad], ["gtarget", "ghist"])

    # masked softmax (target_attention.py:85-90)
    g_p = torch.randn(B, L, generator=gen)
    wg = w.cuda().requires_grad_(True)
    p = F2._DinSoftmax.apply(wg, mask_u8)
    p.backward(g_p.cuda())

    def softmax_ref(w_):
        if mf is None:
            return w_.softmax(dim=-1)
        m = mf.to(w_.dtype)
        return (w_ * m + -1.e9 * (1 - m)).softmax(dim=-1)
    check_against_fp64(softmax_ref, [w], g_p, p, [wg.grad], ["gw_softmax"])
    if mask_kind == "row":          # every score is the -1e9 fill: uniform weights, no gradient
        assert close(p[1], torch.full((L,), 1.0 / L), 1e-6)
        assert float(wg.grad[1].abs().max()) == 0.0

    # masked weighted sum (target_attention.py:85-86, 91)
    g_out = torch.randn(B, d, generator=gen)
    wg2, hg2 = w.cuda().requires_grad_(True), h.cuda().requires_grad_(True)
    out = F2._DinWeightedSum.apply(wg2, mask_u8, hg2)
    out.backward(g_out.cuda())

    def wsum_ref(w_, h_):
        if mf is not None:
            w_ = w_ * mf.to(w_.dtype)
        return (w_.unsqueeze(-1) * h_).sum(dim=1)
    check_against_fp64(wsum_ref, [w, h], g_out, out, [wg2.grad, hg2.grad], ["gw_wsum", "ghist_wsum"])


@pytest.mark.parametrize("d,L", [(8, 50), (33, 31), (64, 200)])
def test_din_input_backward_accumulates_history_gradient(d, L):
    """b2_din_input_bwd(accumulate_hist=1) adds the history gradient onto what ghist already holds."""
    from fuxictr_b200 import functional as F2, _lib
    B = 29
    gen = torch.Generator().manual_seed(d + L)
    t, h = torch.randn(B, d, generator=gen), torch.randn(B, L, d, generator=gen)
    g_in = torch.randn(B * L, 4 * d, generator=gen)
    prior = torch.randn(B, L, d, generator=gen)
    tc, hc, gc = t.cuda(), h.cuda(), g_in.cuda()
    gt = torch.empty(B, d, device="cuda")
    gh = prior.cuda()
    _lib.call("b2_din_input_bwd", F2._ptr(tc), F2._ptr(hc), F2._ptr(gc), B, L, d, F2._ptr(gt), F2._ptr(gh), 1,
              F2._stream())
    g4 = g_in.double().view(B, L, 4, d)
    want_h = prior.double() + g4[:, :, 1] - g4[:, :, 2] + g4[:, :, 3] * t.double().unsqueeze(1)
    want_t = (g4[:, :, 0] + g4[:, :, 2] + g4[:, :, 3] * h.double()).sum(1)
    assert close(gh, want_h, RTOL) and close(gt, want_t, RTOL)


# ------------------------------------------------------------------ embedding gather / scatter / LR
def _gather_setup(dims, B, idx_dtype, seed, seq=None, pad_every=7, oob=False):
    """Tables (padding row 0 zeroed), ids with padding and optionally out-of-range values, and a plan.
    `seq`: {field index: (seq_len, pool)}.  Out-of-range ids exercise the kernel's range check (the id is
    tested before any address is formed; the row reads as zeros and the status word names the field)."""
    from fuxictr_b200 import functional as F2
    seq = seq or {}
    gen = torch.Generator().manual_seed(seed)
    vocabs = [50 + 13 * i for i in range(len(dims))]
    tables = []
    for v, dm in zip(vocabs, dims):
        t = torch.randn(v, dm, generator=gen)
        t[0] = 0
        tables.append(t.cuda())
    idx, fields = [], []
    for i, (v, dm) in enumerate(zip(vocabs, dims)):
        L, pool = seq.get(i, (1, 0))
        ids = torch.randint(1, v, (B, L), generator=gen)
        ids[torch.rand(B, L, generator=gen) < 1.0 / pad_every] = 0
        if L > 1:
            ids[::5] = 0                                      # every position padding
            ids[1::5, L // 2:] = 0                            # padded tail
        if oob:
            ids[3::11, 0] = v + 4
            ids[4::13, -1] = -1
        idx.append((ids if L > 1 else ids[:, 0]).to(idx_dtype).cuda())
        fields.append(F2.GatherField("f%d" % i, i, dm, L, pool, padding_idx=0))
    return F2.GatherPlan(fields), tables, idx


def _gather_reference(plan, tables, idx, gout):
    """Forward (float64, out-of-range rows read as zeros) and the float64 index_add_ table gradients."""
    outs, grads = [], []
    B = idx[0].shape[0]
    go = gout.double().split(plan.widths, dim=1)
    for f, t, ids, g in zip(plan.fields, tables, idx, go):
        ids = ids.long().view(B, -1)
        ok = (ids >= 0) & (ids < t.shape[0])
        rows = torch.where(ok, ids, torch.zeros_like(ids))
        emb = t.double()[rows] * ok.unsqueeze(-1)                        # (B, L, dim)
        live = ok & (ids != f.padding_idx)
        if f.seq_len > 1 and f.pool != 0:
            out = emb.sum(1)
            scale = torch.ones(B, 1, dtype=torch.float64, device=t.device)
            if f.pool == 2:
                count = (emb.sum(-1) != 0).double().sum(-1, keepdim=True)
                out = out / (count + 1e-12)
                scale = 1.0 / (count + 1e-12)
            gpos = (g * scale).unsqueeze(1).expand(-1, f.seq_len, -1)
        else:
            out = emb.reshape(B, -1)
            gpos = g.view(B, f.seq_len, f.dim)
        gt = torch.zeros(t.shape, dtype=torch.float64, device=t.device)
        gt.index_add_(0, ids[live], gpos[live])
        outs.append(out)
        grads.append(gt)
    return torch.cat(outs, 1), grads


def _run_gather(plan, tables, idx, check_exact=True, status_want=None):
    from fuxictr_b200 import functional as F2
    tabs = [t.clone().requires_grad_(True) for t in tables]
    status = torch.zeros(1, dtype=torch.int32, device="cuda")
    out = F2.embed_gather(plan, idx, tabs, status=status)
    gout = torch.randn(out.shape, device="cuda", generator=torch.Generator(device="cuda").manual_seed(5))
    out.backward(gout)
    want, gwant = _gather_reference(plan, tables, idx, gout)
    for f, part, ref in zip(plan.fields, out.split(plan.widths, 1), want.split(plan.widths, 1)):
        if f.seq_len > 1 and f.pool != 0:
            assert rel_err(part, ref) <= 1e-6, (f.name, rel_err(part, ref))
        elif check_exact:
            assert torch.equal(part, ref.float()), f.name                # pure copies: bit for bit
    for f in plan.fields:
        g = tabs[f.table_slot].grad
        assert close(g, gwant[f.table_slot], RTOL), (f.name, rel_err(g, gwant[f.table_slot]))
        assert float(g[0].abs().max()) == 0.0                            # padding row: no gradient
    torch.cuda.synchronize()
    if status_want is not None:
        assert int(status.item()) == status_want
    return out


@pytest.mark.parametrize("idx_dtype", [torch.float64, torch.int64, torch.int32])
@pytest.mark.parametrize("dim", [1, 3, 4, 6, 16, 130, 200])
def test_gather_single_dim_vs_embedding(dim, idx_dtype):
    """Odd dims take 4-byte lanes (VEC=1), 6 takes VEC=2; 130 and 200 are wider than one pass of 32 lanes
    (the general kernel).  Forward equals F.embedding bit for bit."""
    plan, tables, idx = _gather_setup([dim] * 5, 333, idx_dtype, seed=dim)
    out = _run_gather(plan, tables, idx)
    for i, (t, ids) in enumerate(zip(tables, idx)):
        want = torch.nn.functional.embedding(ids.long(), t, padding_idx=0)
        assert torch.equal(out[:, i * dim:(i + 1) * dim], want)


@pytest.mark.parametrize("idx_dtype", [torch.float64, torch.int64, torch.int32])
def test_gather_mixed_dims_one_plan(idx_dtype):
    plan, tables, idx = _gather_setup([1, 3, 4, 6, 16, 130, 200, 16], 257, idx_dtype, seed=11)
    _run_gather(plan, tables, idx)


@pytest.mark.parametrize("idx_dtype", [torch.float64, torch.int64, torch.int32])
@pytest.mark.parametrize("dim", [3, 16, 130])
def test_gather_sequence_pooling(dim, idx_dtype):
    """Unpooled, sum-pooled and mean-pooled sequence fields next to a plain one, with rows whose every
    position is padding (mean of nothing = 0) and padded tails."""
    seq = {1: (8, 0), 2: (8, 1), 3: (50, 2), 4: (5, 2)}
    plan, tables, idx = _gather_setup([dim] * 5, 203, idx_dtype, seed=3 + dim, seq=seq)
    _run_gather(plan, tables, idx)


@pytest.mark.parametrize("pooled", [False, True])
def test_gather_out_of_range_ids_read_zero_and_flag(pooled):
    seq = {1: (6, 2)} if pooled else {}
    plan, tables, idx = _gather_setup([16, 16], 120, torch.int64, seed=21, seq=seq, oob=True)
    _run_gather(plan, tables, idx, status_want=2)


@pytest.mark.parametrize("dim,nf,hot", [(16, 4, 0), (16, 4, 16), (3, 1, 0), (6, 2, 0)])
def test_gather_deep_unroll(dim, nf, hot):
    """B * fields >= 2^20 work items: the fast kernel unrolls 8 rows per lane (with and without staging
    the hot rows in shared memory)."""
    B = (1 << 20) // nf + 3
    plan, tables, idx = _gather_setup([dim] * nf, B, torch.int64, seed=dim + nf)
    plan.hot_rows = hot
    out = _run_gather(plan, tables, idx)
    assert B * nf >= 1 << 20
    for i, (t, ids) in enumerate(zip(tables, idx)):
        assert torch.equal(out[:, i * dim:(i + 1) * dim], t[ids.long()])


@pytest.mark.parametrize("idx_dtype", [torch.float64, torch.int64, torch.int32])
@pytest.mark.parametrize("with_seq", [False, True])
def test_lr_forward_backward(idx_dtype, with_seq):
    """LogisticRegression gather-reduce: out[b] = sum over every (field, position) of w[id] + bias; the
    backward scatters gout to every non-padding row and sums it into the bias."""
    from fuxictr_b200 import functional as F2
    seq = {2: (50, 1), 3: (7, 1)} if with_seq else {}
    nf = 40 if not with_seq else 6
    plan, tables, idx = _gather_setup([1] * nf, 1000, idx_dtype, seed=7, seq=seq)
    bias = torch.randn(1, device="cuda").requires_grad_(True)
    tabs = [t.clone().requires_grad_(True) for t in tables]
    out = F2.lr_forward(plan, idx, tabs, bias)
    gout = torch.randn(out.shape, device="cuda", generator=torch.Generator(device="cuda").manual_seed(8))
    out.backward(gout)
    want = bias.detach().double().expand(out.shape[0]).clone()
    for t, ids in zip(tables, idx):
        want += t.double()[ids.long().view(out.shape[0], -1)].sum(dim=(1, 2))
    assert close(out.view(-1), want, RTOL)
    assert close(bias.grad, gout.double().sum().view(1), RTOL)
    for f, t, ids, tg in zip(plan.fields, tables, idx, tabs):
        ids = ids.long().view(out.shape[0], -1)
        live = ids != 0
        ref = torch.zeros(t.shape, dtype=torch.float64, device="cuda")
        ref.index_add_(0, ids[live], gout.double().expand(-1, ids.shape[1])[live].unsqueeze(-1))
        assert close(tg.grad, ref, RTOL), f.name


# ------------------------------------------------------------------ fused logit + sigmoid + BCE
# Saturating logits.  fp32 sigmoid rounds to 1 above ~16.6 (log(1-p) = -inf -> the -100 clamp, p(1-p) = 0 -> zero
# gradient); below ~-27.6 p(1-p) < 1e-12, so the clamp on it scales the gradient down (-30, -50, -80); exp
# overflows below ~-88.7 (p = 0 -> log p clamped at -100).
EXTREME_LOGITS = [17.0, -17.0, 30.0, -30.0, -50.0, -80.0, 90.0, -90.0, 1e4, -1e4]


def _logit_bce_refs(terms, y, B):
    """Per-row fp32 semantics of the reference (torch sigmoid + binary_cross_entropy in float32: p, the row
    losses, dL/dlogit) and the same formula in float64 with the same clamps (p, mean loss, dL/dlogit)."""
    ts = [t.detach().clone().float().requires_grad_(True) for t in terms]
    z = ts[0]
    for t in ts[1:]:
        z = z + t
    p32 = torch.sigmoid(z)
    rows32 = torch.nn.functional.binary_cross_entropy(p32, y, reduction="none").detach()
    torch.nn.functional.binary_cross_entropy(p32, y).backward()
    z64 = sum(t.double() for t in terms)
    p64 = torch.sigmoid(z64)
    yd = y.double()
    l64 = -(yd * torch.clamp(torch.log(p64), min=-100) + (1 - yd) * torch.clamp(torch.log(1 - p64), min=-100)).mean()
    pq = (1 - p64) * p64
    g64 = ((p64 - yd) / torch.clamp(pq, min=1e-12)) * pq / B
    return p32.detach(), rows32, ts[0].grad, p64, l64, g64


@pytest.mark.parametrize("nterms", [1, 2, 3, 4])
@pytest.mark.parametrize("B", [1, 255, 257])
def test_logit_bce_extremes(nterms, B):
    """Rows with a saturating logit are held to the reference's own fp32 semantics, element by element (their
    float64 values differ by design: -17 instead of the -100 clamp, 1/B instead of a zero gradient), so a kernel
    without the clamps, with other clamp values or with a zero gradient fails there.  The other rows get the fp64
    bar with the fp32 error measured on those rows only, and once more in a launch of their own for the loss."""
    from fuxictr_b200 import functional as F2
    gen = torch.Generator().manual_seed(B * 10 + nterms)
    ext = torch.tensor(EXTREME_LOGITS)
    E = len(ext)
    z0 = (torch.randn(B, 1, generator=gen) * 2).clamp(-8, 8)
    y = (torch.rand(B, 1, generator=gen) < 0.5).float()
    extreme = torch.rand(B, generator=gen) < 0.4
    if B >= 2 * E:                                   # every saturating logit with both labels
        extreme[:2 * E] = True
        y[:2 * E, 0] = torch.arange(2 * E).remainder(2).float()
        z0[:2 * E, 0] = ext.repeat_interleave(2)
    elif B == 1:
        extreme[0] = nterms % 2 == 1
    pos = torch.nonzero(extreme[2 * E:] if B >= 2 * E else extreme).view(-1) + (2 * E if B >= 2 * E else 0)
    z0[pos, 0] = ext[torch.randint(0, E, (pos.numel(),), generator=gen)]
    terms = [z0] + [torch.randn(B, 1, generator=gen) * 0.3 for _ in range(nterms - 1)]
    mod = ~extreme

    tc = [t.cuda().requires_grad_(True) for t in terms]
    loss, y_pred = F2.logit_bce(y.cuda(), *tc)
    loss.backward()
    p32, rows32, g32, p64, l64, g64 = _logit_bce_refs(terms, y, B)
    assert torch.isfinite(loss).all() and all(torch.isfinite(t.grad).all() for t in tc)

    # the loss of the whole batch: the fp32 row losses (clamps included), summed exactly
    want = float(rows32.double().sum()) / B
    assert abs(float(loss) - want) <= 2e-6 * abs(want), (float(loss), want)
    yp, gmax = y_pred.cpu(), float(g32.abs().max())
    if extreme.any():
        ex = extreme
        assert ((yp[ex] - p32[ex]).abs() <= 2e-6 * p32[ex].abs()).all(), (yp[ex], p32[ex])
        for i, t in enumerate(tc):
            g = t.grad.cpu()
            ok = (g[ex] - g32[ex]).abs() <= 1e-5 * g32[ex].abs() + 1e-7 * gmax
            assert ok.all(), ("glogit term %d" % i, z0[ex][~ok.view(-1)], g[ex][~ok], g32[ex][~ok])
    if mod.any():
        bar(yp[mod], p32[mod], p64[mod], "y_pred")
        for i, t in enumerate(tc):
            bar(t.grad.cpu()[mod], g32[mod], g64[mod], "glogit term %d" % i)
        m = mod.cuda()
        loss_m, _ = F2.logit_bce(y.cuda()[m], *[t.cuda()[m] for t in terms])
        _, rows32_m, _, _, l64_m, _ = _logit_bce_refs([t[mod] for t in terms], y[mod], int(mod.sum()))
        bar(loss_m, rows32_m.mean(), l64_m, "loss of the non-saturating rows")

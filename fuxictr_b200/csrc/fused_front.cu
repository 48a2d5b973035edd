// fused_front.cu — the whole "sparse front" of an FM-style model in one launch each way, sm_90a.
//
// Forward  (b2_front_fwd): for every sample, in ONE kernel
//   * the multi-field embedding gather, written as the stacked (B, F, D) tensor
//       FeatureEmbedding.forward            fuxictr/pytorch/layers/embeddings/feature_embedding.py:73-88
//   * the FM second-order term  0.5 * sum_d[(sum_f e)^2 - sum_f e^2]
//       InnerProductInteraction product_sum fuxictr/pytorch/layers/interactions/inner_product.py:56-62
//   * the first-order term  sum_f w_f[idx_f] + bias
//       LogisticRegression.forward          fuxictr/pytorch/layers/blocks/logistic_regression.py:55-58
//   (FactorizationMachine.forward = FM + LR, layers/blocks/factorization_machine.py:56-59)
// Backward (b2_front_bwd): one kernel turns the MLP's input gradient, the logit gradient and the
//   saved field sums into dense-table gradients:  g[b,f,:] = gx[b,f,:] + gl[b] * (S[b,:] - e[b,f,:]),
//   warp-aggregated `red.global.add.v4.f32` into the embedding-gradient tables, plus the D=1
//   scatter for the LR tables and the bias gradient.
//
// One warp owns one sample: LPR = 2^k lanes per table row (16-byte accesses), 32/LPR rows per
// pass, ceil(F / (32/LPR)) passes with all index loads, then all row loads, in flight together;
// field sums are xor-shuffle reductions over the (fields x emb_dim) register tile.
#include "embed_common.cuh"
#include "adam_common.cuh"

namespace {

// MAX_PASSES: rows of one sample handled per chunk of the pass loop = MAX_PASSES * (32 / LPR);
// a smaller value keeps the register arrays (and so the occupancy) matched to the field count.
template <typename IdxT, int MAX_PASSES>
__global__ void __launch_bounds__(256)
front_fwd_kernel(const __grid_constant__ B2FieldPack emb, const __grid_constant__ B2FieldPack lr,
                 const __grid_constant__ b2_lazy_ctx lz, int lazy,
                 int64_t batch, int dim, int lpr_log2, int has_lr, int want_fm,
                 const float* __restrict__ bias, float* __restrict__ logit_out,
                 float* __restrict__ sum_out, int32_t* __restrict__ status, int64_t small_delta) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const SmemFields sf = b2_stage_fields(emb, smem_raw);     // kernel parameters -> shared memory only
  SmemFields lf;
  lf.f = nullptr;
  lf.slot_start = nullptr;
  if (has_lr) lf = b2_stage_fields(lr, smem_raw + ((pack_smem_bytes(emb.nfields) + 15) & ~(size_t) 15));
  b2_pdl_trigger();
  b2_pdl_wait();
  const int F = emb.nfields;
  const int LPR = 1 << lpr_log2;
  const int rows_per_pass = 32 >> lpr_log2;
  const int lane = threadIdx.x & 31;
  const int sub = lane & (LPR - 1), rg = lane >> lpr_log2;
  const int e = sub * 4;
  const bool lane_on = e < dim;
  const int64_t warp = ((int64_t) blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t) gridDim.x * blockDim.x) >> 5;
  const float bv = (bias != nullptr) ? __ldg(bias) : 0.f;
  // lazy tables: steps completed so far; a row with last_step < done replays the missed
  // zero-gradient Adam updates in registers (never written back here)
  const int done = lazy ? (int) *lz.step_dev : 0;
  const B2AdamConst ac = {lz.w1, lz.beta2, lz.w2, lz.eps};
  const B2AdamSched* sched = reinterpret_cast<const B2AdamSched*>(lz.sched);

  for (int64_t b = warp; b < batch; b += nwarps) {
    float4 s = make_float4(0.f, 0.f, 0.f, 0.f), q = make_float4(0.f, 0.f, 0.f, 0.f);
    float lrsum = 0.f;
    for (int f0 = 0; f0 < F; f0 += rows_per_pass * MAX_PASSES) {
      int64_t row[MAX_PASSES];
      bool ok[MAX_PASSES];
#pragma unroll
      for (int u = 0; u < MAX_PASSES; ++u) {  // all index loads in flight
        const int f = f0 + u * rows_per_pass + rg;
        ok[u] = false;
        row[u] = 0;
        if (f < F) {
          const b2_field& fd = sf.f[f];
          row[u] = b2_load_index<IdxT>(fd.idx, b * fd.idx_stride);
          ok[u] = row[u] >= 0 && row[u] < fd.vocab;
          if (!ok[u] && status != nullptr && sub == 0) atomicMax(status, f + 1);
        }
      }
      float4 v[MAX_PASSES];
      float w[MAX_PASSES];
#pragma unroll
      for (int u = 0; u < MAX_PASSES; ++u) {  // all row loads in flight
        const int f = f0 + u * rows_per_pass + rg;
        v[u] = make_float4(0.f, 0.f, 0.f, 0.f);
        w[u] = 0.f;
        if (f < F && ok[u]) {
          if (lane_on)
            v[u] = __ldg(reinterpret_cast<const float4*>(reinterpret_cast<const float*>(sf.f[f].table) +
                                                         row[u] * dim + e));
          if (has_lr && sub == 0) w[u] = __ldg(reinterpret_cast<const float*>(lf.f[f].table) + row[u]);
        }
      }
      if (lazy) {
        int last_e[MAX_PASSES], last_l[MAX_PASSES];
#pragma unroll
        for (int u = 0; u < MAX_PASSES; ++u) {   // all last_step loads in flight
          const int f = f0 + u * rows_per_pass + rg;
          last_e[u] = done;
          last_l[u] = done;
          if (f < F && ok[u]) {
            if (lane_on) last_e[u] = __ldg(lz.last_step + lz.grow_emb[f] + row[u]);
            if (has_lr && sub == 0) last_l[u] = __ldg(lz.last_step + lz.grow_lr[f] + row[u]);
          }
        }
        float4 m4[MAX_PASSES], v4[MAX_PASSES];
        float m1[MAX_PASSES], v1[MAX_PASSES];
#pragma unroll
        for (int u = 0; u < MAX_PASSES; ++u) {   // all moment loads of stale rows in flight
          const int f = f0 + u * rows_per_pass + rg;
          m4[u] = v4[u] = make_float4(0.f, 0.f, 0.f, 0.f);
          m1[u] = v1[u] = 0.f;
          if (last_e[u] < done) {
            const float* pp = reinterpret_cast<const float*>(sf.f[f].table) + row[u] * dim + e;
            m4[u] = *reinterpret_cast<const float4*>(pp + lz.delta_m);
            v4[u] = *reinterpret_cast<const float4*>(pp + lz.delta_v);
          }
          if (last_l[u] < done) {
            const float* pp = reinterpret_cast<const float*>(lf.f[f].table) + row[u];
            m1[u] = pp[lz.delta_m];
            v1[u] = pp[lz.delta_v];
          }
        }
#pragma unroll
        for (int u = 0; u < MAX_PASSES; ++u) {   // replay the missed zero-gradient updates
          for (int k = last_e[u] + 1; k <= done; ++k) {
            const B2AdamSched sc = sched[k];
            b2_adam_apply(v[u].x, 0.f, m4[u].x, v4[u].x, ac, sc.x, sc.y);
            b2_adam_apply(v[u].y, 0.f, m4[u].y, v4[u].y, ac, sc.x, sc.y);
            b2_adam_apply(v[u].z, 0.f, m4[u].z, v4[u].z, ac, sc.x, sc.y);
            b2_adam_apply(v[u].w, 0.f, m4[u].w, v4[u].w, ac, sc.x, sc.y);
          }
          for (int k = last_l[u] + 1; k <= done; ++k) {
            const B2AdamSched sc = sched[k];
            b2_adam_apply(w[u], 0.f, m1[u], v1[u], ac, sc.x, sc.y);
          }
        }
      }
#pragma unroll
      for (int u = 0; u < MAX_PASSES; ++u) {
        const int f = f0 + u * rows_per_pass + rg;
        if (f < F) {
          if (lane_on) {
            const b2_field& fd = sf.f[f];
            float* op = reinterpret_cast<float*>(fd.out) + b * fd.out_stride + e;
            *reinterpret_cast<float4*>(op) = v[u];
            if (small_delta != 0)    // the 3xTF32 small part of the first GEMM's A operand, born with the rows
              *reinterpret_cast<float4*>(op + small_delta) = make_float4(b2_tf32_small(v[u].x), b2_tf32_small(v[u].y),
                                                                        b2_tf32_small(v[u].z), b2_tf32_small(v[u].w));
          }
          s.x += v[u].x; s.y += v[u].y; s.z += v[u].z; s.w += v[u].w;
          q.x = fmaf(v[u].x, v[u].x, q.x); q.y = fmaf(v[u].y, v[u].y, q.y);
          q.z = fmaf(v[u].z, v[u].z, q.z); q.w = fmaf(v[u].w, v[u].w, q.w);
          lrsum += w[u];
        }
      }
    }
    // field sums: reduce over the row groups (lanes with equal `sub`)
    for (int o = LPR; o < 32; o <<= 1) {
      s.x += __shfl_xor_sync(0xffffffffu, s.x, o); s.y += __shfl_xor_sync(0xffffffffu, s.y, o);
      s.z += __shfl_xor_sync(0xffffffffu, s.z, o); s.w += __shfl_xor_sync(0xffffffffu, s.w, o);
      q.x += __shfl_xor_sync(0xffffffffu, q.x, o); q.y += __shfl_xor_sync(0xffffffffu, q.y, o);
      q.z += __shfl_xor_sync(0xffffffffu, q.z, o); q.w += __shfl_xor_sync(0xffffffffu, q.w, o);
    }
    if (sum_out != nullptr && rg == 0 && lane_on)
      *reinterpret_cast<float4*>(sum_out + b * dim + e) = s;
    float total = 0.f;
    if (want_fm) {
      // 0.5 * ((sum e)^2 - sum e^2), then sum over the embedding dim (inner_product.py:56-62)
      float t = ((s.x * s.x - q.x) + (s.y * s.y - q.y) + (s.z * s.z - q.z) + (s.w * s.w - q.w)) * 0.5f;
      if (!lane_on) t = 0.f;
      for (int o = 1; o < LPR; o <<= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
      total = t;  // identical in every lane of a row group; take lane 0's
    }
    lrsum = b2_warp_sum(lrsum);
    if (lane == 0 && logit_out != nullptr) logit_out[b] = total + (lrsum + bv);
  }
}

template <typename IdxT>
__global__ void __launch_bounds__(256)
front_bwd_kernel(const __grid_constant__ B2FieldPack emb, const __grid_constant__ B2FieldPack lr,
                 const __grid_constant__ b2_lazy_ctx lz, int lazy,
                 int64_t batch, int dim, int lpr_log2, int has_lr, int want_fm,
                 const float* __restrict__ emb_saved, const float* __restrict__ gx_base,
                 const float* __restrict__ sums, const float* __restrict__ glogit,
                 float* __restrict__ gbias) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  __shared__ float red[32];
  const SmemFields sf = b2_stage_fields(emb, smem_raw);
  SmemFields lf;
  lf.f = nullptr;
  lf.slot_start = nullptr;
  if (has_lr) lf = b2_stage_fields(lr, smem_raw + ((pack_smem_bytes(emb.nfields) + 15) & ~(size_t) 15));
  b2_pdl_trigger();
  b2_pdl_wait();
  const int F = emb.nfields;
  const int LPR = 1 << lpr_log2;
  const int lane = threadIdx.x & 31;
  const int sub = lane & (LPR - 1);
  const int my_group = lane >> lpr_log2;
  const int groups_per_warp = 32 >> lpr_log2;
  const int e = sub * 4;
  const int64_t nitems = batch * (int64_t) F;
  const int64_t ngroups = ((int64_t) gridDim.x * blockDim.x) >> lpr_log2;
  const int64_t group = ((int64_t) blockIdx.x * blockDim.x + threadIdx.x) >> lpr_log2;
  const int64_t warp_first = group - my_group;
  float gb_acc = 0.f;
  const int tmark = lazy ? (int) *lz.step_dev + 1 : 0;   // the optimizer step this backward feeds

  for (int64_t wbase = warp_first; wbase < nitems; wbase += ngroups) {
    const int64_t item = wbase + my_group;
    float* drow = nullptr;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    int enq_e = -1, enq_l = -1;   // global rows this lane has to append to the worklist
    if (item < nitems) {
      const int64_t b = item / F;
      const int f = (int) (item - b * F);
      const b2_field& fd = sf.f[f];
      const int64_t row = b2_load_index<IdxT>(fd.idx, b * fd.idx_stride);
      const float gl = (glogit != nullptr) ? __ldg(glogit + b) : 0.f;
      if (f == 0 && sub == 0) gb_acc += gl;
      const bool ok = row >= 0 && row < fd.vocab && row != (int64_t) fd.padding_idx;
      if (ok) {
        if (fd.table != nullptr) drow = reinterpret_cast<float*>(const_cast<void*>(fd.table)) + row * dim;
        if (has_lr && sub == 0) {
          const b2_field& ld = lf.f[f];
          if (ld.table != nullptr && row != (int64_t) ld.padding_idx) {
            b2_red_add(reinterpret_cast<float*>(const_cast<void*>(ld.table)) + row, gl);
            if (lazy) {   // first toucher of the LR row this step enqueues it
              const int grow = (int) (lz.grow_lr[f] + row);
              if (atomicExch(lz.mark + grow, tmark) != tmark) enq_l = grow;
            }
          }
        }
        if (lazy && drow != nullptr && sub == 0) {   // first toucher of the embedding row enqueues it
          const int grow = (int) (lz.grow_emb[f] + row);
          if (atomicExch(lz.mark + grow, tmark) != tmark) enq_e = grow;
        }
      }
      if (drow != nullptr && e < dim) {
        // fd.out points into the incoming-gradient arena; the saved embeddings share its layout
        const float* grow = reinterpret_cast<const float*>(fd.out) + b * fd.out_stride + e;
        if (gx_base != nullptr) v = __ldg(reinterpret_cast<const float4*>(grow));
        if (want_fm) {
          const float4 ev = __ldg(reinterpret_cast<const float4*>(emb_saved + (grow - gx_base)));
          const float4 sv = __ldg(reinterpret_cast<const float4*>(sums + b * dim + e));
          v.x = fmaf(gl, sv.x - ev.x, v.x); v.y = fmaf(gl, sv.y - ev.y, v.y);
          v.z = fmaf(gl, sv.z - ev.z, v.z); v.w = fmaf(gl, sv.w - ev.w, v.w);
        }
      }
    }
    if (lazy) {
      // warp-aggregated append: one atomicAdd on the shared counter per warp, not per row
      const unsigned me = __ballot_sync(0xffffffffu, enq_e >= 0);
      const unsigned ml = __ballot_sync(0xffffffffu, enq_l >= 0);
      const int ne = __popc(me), nl = __popc(ml);
      if (ne + nl > 0) {
        int base = 0;
        if (lane == 0) base = atomicAdd(lz.counter, ne + nl);
        base = __shfl_sync(0xffffffffu, base, 0);
        const unsigned lt = (1u << lane) - 1u;
        if (enq_e >= 0) {
          const int pos = base + __popc(me & lt);
          if (pos < lz.worklist_capacity) lz.worklist[pos] = enq_e;
        }
        if (enq_l >= 0) {
          const int pos = base + ne + __popc(ml & lt);
          if (pos < lz.worklist_capacity) lz.worklist[pos] = enq_l;
        }
      }
    }
    // warp-level aggregation of duplicate destination rows (see scatter_bwd_kernel)
    const unsigned peers = __match_any_sync(0xffffffffu, (unsigned long long) drow);
    unsigned gset = 0;
    for (int g = 0; g < groups_per_warp; ++g) gset |= ((peers >> (g << lpr_log2)) & 1u) << g;
    const bool leader = (drow != nullptr) && ((gset & ((1u << my_group) - 1u)) == 0u);
    const bool has_dups = (drow != nullptr) && (gset != (1u << my_group));
    if (__ballot_sync(0xffffffffu, has_dups) != 0u) {
      float4 acc = v;
      for (int g = 0; g < groups_per_warp; ++g) {
        const int srcl = (g << lpr_log2) + sub;
        float4 o;
        o.x = __shfl_sync(0xffffffffu, v.x, srcl);
        o.y = __shfl_sync(0xffffffffu, v.y, srcl);
        o.z = __shfl_sync(0xffffffffu, v.z, srcl);
        o.w = __shfl_sync(0xffffffffu, v.w, srcl);
        if (g != my_group && ((gset >> g) & 1u)) { acc.x += o.x; acc.y += o.y; acc.z += o.z; acc.w += o.w; }
      }
      v = acc;
    }
    if (leader && e < dim) b2_red_add_v4(drow + e, v);
  }
  if (gbias != nullptr) {
    const float t = b2_block_sum(gb_acc, red);
    if (threadIdx.x == 0 && t != 0.f) b2_red_add(gbias, t);
  }
}

template <typename IdxT>
int launch_front_fwd(const B2FieldPack& emb, const B2FieldPack& lr, const b2_lazy_ctx& lz, int lazy,
                     int64_t batch, int dim, int has_lr,
                     int want_fm, const float* bias, float* logit_out, float* sum_out, int32_t* status,
                     int64_t small_delta, cudaStream_t st) {
  int lpr_log2 = next_pow2_log2((dim + 3) / 4);
  const size_t smem = ((pack_smem_bytes(emb.nfields) + 15) & ~(size_t) 15) + pack_smem_bytes(emb.nfields) + 16;
  const int grid = grid_for(batch * 32, 256);
  const int passes = (emb.nfields + (32 >> lpr_log2) - 1) / (32 >> lpr_log2);
  auto kfn = front_fwd_kernel<IdxT, 8>;
  if (passes <= 2) kfn = front_fwd_kernel<IdxT, 2>;
  else if (passes <= 5) kfn = front_fwd_kernel<IdxT, 5>;
  B2_LAUNCH(kfn, grid, 256, smem, st, emb, lr, lz, lazy, batch, dim, lpr_log2, has_lr, want_fm, bias, logit_out, sum_out, status, small_delta);
  B2_CUDA_LAUNCH_CHECK("b2_front_fwd");
  return B2_OK;
}

template <typename IdxT>
int launch_front_bwd(const B2FieldPack& emb, const B2FieldPack& lr, const b2_lazy_ctx& lz, int lazy,
                     int64_t batch, int dim, int has_lr,
                     int want_fm, const float* emb_saved, const float* gx, const float* sums,
                     const float* glogit, float* gbias, cudaStream_t st) {
  int lpr_log2 = next_pow2_log2((dim + 3) / 4);
  const size_t smem = ((pack_smem_bytes(emb.nfields) + 15) & ~(size_t) 15) + pack_smem_bytes(emb.nfields) + 16;
  const int grid = grid_for((batch * (int64_t) emb.nfields) << lpr_log2, 256);
  auto kfn = front_bwd_kernel<IdxT>;
  B2_LAUNCH(kfn, grid, 256, smem, st, emb, lr, lz, lazy, batch, dim, lpr_log2, has_lr, want_fm, emb_saved, gx, sums, glogit, gbias);
  B2_CUDA_LAUNCH_CHECK("b2_front_bwd");
  return B2_OK;
}

// Validates the "front" layout: F categorical fields of one common dim (multiple of 4, <= 128),
// stacked/concatenated into 16-byte aligned rows; the LR pack has the same fields with dim 1.
int check_front(const b2_field* emb, const b2_field* lr, int nfields, bool bwd) {
  B2_REQUIRE(emb != nullptr, "emb fields is NULL");
  B2_REQUIRE(nfields >= 1 && nfields <= B2_MAX_FIELDS, "nfields=%d outside [1,%d]", nfields, B2_MAX_FIELDS);
  const int dim = emb[0].dim;
  B2_REQUIRE(dim >= 4 && dim <= 128 && dim % 4 == 0, "front kernels need emb dim %% 4 == 0 and <= 128 (got %d)", dim);
  for (int i = 0; i < nfields; ++i) {
    const b2_field& f = emb[i];
    B2_REQUIRE(f.dim == dim && f.seq_len == 1, "field %d: front kernels need one common dim and no sequences", i);
    B2_REQUIRE(f.idx != nullptr && f.out != nullptr, "field %d: NULL idx/out", i);
    B2_REQUIRE(bwd || f.table != nullptr, "field %d: NULL table", i);
    B2_REQUIRE(((uintptr_t) f.out % 16) == 0 && (f.out_stride % 4) == 0 &&
               (f.table == nullptr || ((uintptr_t) f.table % 16) == 0), "field %d: rows must be 16-byte aligned", i);
    if (lr != nullptr) {
      B2_REQUIRE(lr[i].idx == f.idx && lr[i].idx_stride == f.idx_stride, "field %d: LR and embedding must share indices", i);
      B2_REQUIRE(bwd || lr[i].table != nullptr, "field %d: NULL LR table", i);
    }
  }
  return B2_OK;
}

void fill_pack(B2FieldPack& pack, const b2_field* fields, int nfields) {
  for (int i = 0; i < nfields; ++i) {
    pack.f[i] = fields[i];
    pack.slot_start[i] = i;
  }
  pack.slot_start[nfields] = nfields;
  pack.nfields = nfields;
  pack.nslots = nfields;
  pack.all_len1 = 1;
  pack.pad_ = 0;
}
}  // namespace

extern "C" B2_API int b2_front_fwd(const b2_field* emb_fields, const b2_field* lr_fields, int nfields,
                                   int64_t batch, int idx_dtype, int want_fm, const float* bias,
                                   float* logit_out, float* sum_out, int32_t* status,
                                   const b2_lazy_ctx* lazy, float* emb_small, void* stream) {
  int rc = check_front(emb_fields, lr_fields, nfields, false);
  if (rc != B2_OK) return rc;
  // emb_small mirrors the output arena: field i's rows land at emb_small + (emb_fields[i].out - emb_fields[0].out)
  int64_t small_delta = 0;
  if (emb_small != nullptr) {
    B2_REQUIRE(((uintptr_t) emb_small % 16) == 0, "emb_small must be 16-byte aligned");
    small_delta = emb_small - reinterpret_cast<float*>(emb_fields[0].out);
    B2_REQUIRE(small_delta != 0, "emb_small must not alias the output");
  }
  B2_REQUIRE(batch >= 0, "negative batch");
  B2_REQUIRE(!want_fm || sum_out != nullptr, "want_fm needs sum_out (saved for the backward)");
  if (batch == 0) return B2_OK;
  static thread_local B2FieldPack epack, lpack;
  fill_pack(epack, emb_fields, nfields);
  const int has_lr = lr_fields != nullptr;
  if (has_lr) fill_pack(lpack, lr_fields, nfields); else lpack.nfields = 0;
  cudaStream_t st = (cudaStream_t) stream;
  const int dim = emb_fields[0].dim;
  static thread_local b2_lazy_ctx lz_none;
  const b2_lazy_ctx& lz = lazy ? *lazy : lz_none;
  const int lzf = lazy ? 1 : 0;
  switch (idx_dtype) {
    case B2_F64: return launch_front_fwd<double>(epack, lpack, lz, lzf, batch, dim, has_lr, want_fm, bias, logit_out, sum_out, status, small_delta, st);
    case B2_I64: return launch_front_fwd<int64_t>(epack, lpack, lz, lzf, batch, dim, has_lr, want_fm, bias, logit_out, sum_out, status, small_delta, st);
    case B2_I32: return launch_front_fwd<int32_t>(epack, lpack, lz, lzf, batch, dim, has_lr, want_fm, bias, logit_out, sum_out, status, small_delta, st);
    default: return b2_fail(B2_E_INVALID, "idx_dtype %d unsupported", idx_dtype);
  }
}

extern "C" B2_API int b2_front_bwd(const b2_field* emb_fields, const b2_field* lr_fields, int nfields,
                                   int64_t batch, int idx_dtype, int want_fm, const float* emb_saved,
                                   const float* gx, const float* sums, const float* glogit, float* gbias,
                                   const b2_lazy_ctx* lazy, void* stream) {
  int rc = check_front(emb_fields, lr_fields, nfields, true);
  if (rc != B2_OK) return rc;
  B2_REQUIRE(batch >= 0, "negative batch");
  B2_REQUIRE(gx != nullptr, "gx (gradient arena base) is NULL");
  B2_REQUIRE(!want_fm || (emb_saved != nullptr && sums != nullptr && glogit != nullptr), "want_fm needs emb_saved, sums, glogit");
  B2_REQUIRE(lr_fields == nullptr || glogit != nullptr, "LR backward needs glogit");
  if (batch == 0) return B2_OK;
  static thread_local B2FieldPack epack, lpack;
  fill_pack(epack, emb_fields, nfields);
  const int has_lr = lr_fields != nullptr;
  if (has_lr) fill_pack(lpack, lr_fields, nfields); else lpack.nfields = 0;
  cudaStream_t st = (cudaStream_t) stream;
  const int dim = emb_fields[0].dim;
  static thread_local b2_lazy_ctx lz_none;
  const b2_lazy_ctx& lz = lazy ? *lazy : lz_none;
  const int lzf = lazy ? 1 : 0;
  switch (idx_dtype) {
    case B2_F64: return launch_front_bwd<double>(epack, lpack, lz, lzf, batch, dim, has_lr, want_fm, emb_saved, gx, sums, glogit, gbias, st);
    case B2_I64: return launch_front_bwd<int64_t>(epack, lpack, lz, lzf, batch, dim, has_lr, want_fm, emb_saved, gx, sums, glogit, gbias, st);
    case B2_I32: return launch_front_bwd<int32_t>(epack, lpack, lz, lzf, batch, dim, has_lr, want_fm, emb_saved, gx, sums, glogit, gbias, st);
    default: return b2_fail(B2_E_INVALID, "idx_dtype %d unsupported", idx_dtype);
  }
}

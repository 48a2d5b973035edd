// transact.cu — TransAct's sequence kernels (model_zoo/TransAct/src/TransAct.py), sm_90a.
//
// A TransActTransformer layer on the early-fusion tokens X (B L, md) is the in-projection GEMM, the masked
// self-attention below, the out-projection GEMM, bst.cu's residual + dropout + LayerNorm row kernel, the FFN as a
// two-layer MLP chain (ReLU and the inner dropout in the first epilogue) and the residual + LayerNorm kernel again.
// This file holds the token assembly (with the per-slot valid bytes), the attention and the output head (last k slots
// and the masked max over L).  Layouts and range: include/fuxictr_b200.h "TransAct".
//
// Attention: one CTA of TA_THREADS threads per (sample, head, block of TA_TILE queries).  K and V stream through
// shared memory in tiles of TA_TILE keys with an online softmax, so shared memory is O(TA_TILE dh), not O(L dh).
// Scores: thread t takes query t / 8 of the block and keys t % 8 + 8 u (u < 4) of the tile, so a row's max and sum are
// 8-lane shuffles.  Products with V (and, in the backward, with K, Q and dO): warp w takes queries 4 w .. 4 w + 3 and
// lane l columns l + 32 v (v < NV = ceil(dh / 32)), so a 128- or 256-wide head keeps every lane busy.  Tiles sit at
// a row pitch of dh + 1.  The forward saves the softmax max and sum per (b, h, i); the backward recomputes P from
// them in two deterministic passes, query-block outer for dQ (which also writes D_i = dO_i . O_i) and key-block outer
// for dK and dV.  Padded query rows are skipped (their output and gradients are 0): the model zeroes them, and as keys
// they are masked in every layer.  All arithmetic is fp32 on CUDA cores, expf (not __expf).
#include "row_common.cuh"
#include "philox.cuh"

#define TA_THREADS 256
#define TA_TILE 32
#define TA_TP (TA_TILE + 1)

struct ta_parts {
  const float* src[B2_TRANSACT_MAX_PARTS];    // ns sequence views, then nt target views
  int64_t ld[B2_TRANSACT_MAX_PARTS];
  float* dst[B2_TRANSACT_MAX_PARTS];          // their gradients
};

// ---------------------------------------------------------------------------------
// Tokens
// ---------------------------------------------------------------------------------
__device__ __forceinline__ bool ta_id_nonzero(const void* ids, int dtype, int64_t off) {
  if (dtype == B2_F64) return __ldg(reinterpret_cast<const double*>(ids) + off) != 0.0;
  if (dtype == B2_I64) return __ldg(reinterpret_cast<const long long*>(ids) + off) != 0;
  if (dtype == B2_I32) return __ldg(reinterpret_cast<const int*>(ids) + off) != 0;
  return __ldg(reinterpret_cast<const float*>(ids) + off) != 0.f;
}

// X[b L + t, :] = [seq_0[b, t] .. seq_{ns-1}[b, t] | tgt_0[b] .. tgt_{nt-1}[b]] "=" with its GEMM operand copy; then
// warp per sample: valid[b, t] = ids[b, t] != 0, and the last slot of an all-padding sample set to 1.
__global__ void __launch_bounds__(256)
ta_tokens_fwd_kernel(ta_parts p, int ns, int nt, const void* __restrict__ ids, int ids_dtype, int64_t ld_ids,
                     int64_t batch, int L, int D, float* __restrict__ tok, void* aux, int aux_dtype, int64_t ld_aux,
                     uint8_t* __restrict__ valid) {
  b2_pdl_wait();
  const int md = D * (ns + nt);
  const int64_t total = batch * L * md;
  for (int64_t e = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t) gridDim.x * blockDim.x) {
    const int64_t row = e / md;
    const int c = (int) (e - row * md);
    const int64_t b = row / L;
    const int t = (int) (row - b * L);
    const int f = c / D, d = c - f * D;
    const float v = f < ns ? __ldg(p.src[f] + b * p.ld[f] + (int64_t) t * D + d) : __ldg(p.src[f] + b * p.ld[f] + d);
    tok[e] = v;
    if (aux) {
      const float w[1] = {v};
      rk_store_aux<1>(aux, aux_dtype, row * ld_aux + c, w);
    }
  }
  const int lane = threadIdx.x & 31;
  const int64_t nwarps = (int64_t) gridDim.x * (blockDim.x >> 5);
  for (int64_t b = (int64_t) blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); b < batch; b += nwarps) {
    bool any = false;
    for (int t0 = 0; t0 < L; t0 += 32) {
      const int t = t0 + lane;
      const bool v = t < L && ta_id_nonzero(ids, ids_dtype, b * ld_ids + t);
      any |= __any_sync(0xffffffffu, v);
      if (t < L) valid[b * L + t] = (v || (t == L - 1 && !any)) ? 1 : 0;
    }
    // `any` of the last chunk already covers every earlier chunk
  }
  b2_pdl_trigger();
}

// From G (B L, md): dseq[f] (B, L, D) "=" its columns, dtgt[f] (B, D) "=" the sum over t of its columns (one thread
// per (b, column), t in order: deterministic).
__global__ void __launch_bounds__(256)
ta_tokens_bwd_kernel(const float* __restrict__ g, int64_t batch, int L, int D, int ns, int nt, ta_parts p) {
  b2_pdl_wait();
  const int md = D * (ns + nt);
  const int64_t nseq = batch * L * ns * D, ntgt = batch * nt * D;
  for (int64_t e = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; e < nseq + ntgt;
       e += (int64_t) gridDim.x * blockDim.x) {
    if (e < nseq) {
      const int64_t row = e / (ns * D);
      const int c = (int) (e - row * ns * D);
      const int f = c / D, d = c - f * D;
      p.dst[f][row * D + d] = __ldg(g + row * md + c);
    } else {
      const int64_t r = e - nseq;
      const int64_t b = r / (nt * D);
      const int c = (int) (r - b * nt * D);
      const int f = c / D, d = c - f * D;
      const float* gb = g + b * L * md + ns * D + c;
      float s = 0.f;
      for (int t = 0; t < L; ++t) s += __ldg(gb + (int64_t) t * md);
      p.dst[ns + f][b * D + d] = s;
    }
  }
  b2_pdl_trigger();
}

// ---------------------------------------------------------------------------------
// Key-tiled masked self-attention
// ---------------------------------------------------------------------------------
struct ta_dims {
  int L, md, H, dh, DP, nb;      // tokens, model_dim, heads, head width, smem pitch dh + 1, blocks of TA_TILE rows
};

__device__ __forceinline__ float ta_dot(const float* a, const float* b, int n) {
  float s = 0.f;
  for (int t = 0; t < n; ++t) s += a[t] * b[t];
  return s;
}

// The dropout keep of weight (b, h, i, j): element ((b H + h) L + i) L + j of the (B, H, L, L) weights.
__device__ __forceinline__ bool ta_keep(uint64_t seed, uint64_t off, int64_t b, int h, int i, int j, const ta_dims d,
                                        uint32_t thresh) {
  const uint64_t idx = (((uint64_t) b * d.H + h) * d.L + i) * d.L + j;
  return b2_drop_keep(seed, off, idx, thresh);
}

// Rows r0 .. r0 + TA_TILE - 1 (0 beyond L), columns c0 .. c0 + dh - 1 of M (row pitch ld) into S (TA_TILE x DP),
// times `scale`.
__device__ __forceinline__ void ta_stage(const float* __restrict__ M, int64_t ld, int r0, int c0, const ta_dims d,
                                         float* S, float scale) {
  for (int t = threadIdx.x; t < TA_TILE * d.dh; t += blockDim.x) {
    const int r = t / d.dh, c = t - r * d.dh;
    float v = 0.f;
    if (r0 + r < d.L) v = __ldg(M + (int64_t) (r0 + r) * ld + c0 + c) * scale;
    S[r * d.DP + c] = v;
  }
}

// Any live (valid) row among r0 .. r0 + TA_TILE - 1?  Every thread of the CTA calls this.
__device__ __forceinline__ bool ta_any_live(const uint8_t* __restrict__ vb, int r0, int L) {
  const int r = r0 + (int) threadIdx.x;
  return __syncthreads_or(threadIdx.x < TA_TILE && r < L && vb[r] != 0) != 0;
}

__device__ __forceinline__ void ta_block_of(int64_t blk, const ta_dims d, int64_t& b, int& h, int& r0) {
  const int64_t bh = blk / d.nb;
  r0 = (int) (blk - bh * d.nb) * TA_TILE;
  b = bh / d.H;
  h = (int) (bh - b * d.H);
}

// ctx[b L + i, h dh + c] = sum_j dropout(softmax_j((q_i scale) . k_j + mask)) v_j[c]; key j masked iff !valid[b, j].
template <int NV>
__global__ void __launch_bounds__(TA_THREADS, NV >= 8 ? 1 : 2)
ta_attn_fwd_kernel(const float* __restrict__ qkv, const uint8_t* __restrict__ valid, int64_t batch, ta_dims d,
                   float scale, const int64_t* __restrict__ drop_rng, int64_t drop_layer, uint32_t drop_thresh,
                   float drop_scale, float* __restrict__ ctx, void* aux, int aux_dtype, int64_t ld_aux,
                   float* __restrict__ stat_max, float* __restrict__ stat_sum) {
  extern __shared__ float smem[];
  float* Qs = smem;
  float* Ks = Qs + TA_TILE * d.DP;
  float* Vs = Ks + TA_TILE * d.DP;
  float* Ps = Vs + TA_TILE * d.DP;       // TA_TILE x TA_TP
  float* As = Ps + TA_TILE * TA_TP;      // per query: the rescale of this tile, then 1 / l
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int qr = tid >> 3, kg = tid & 7;
  b2_pdl_wait();
  uint64_t seed = 0, off = 0;
  if (drop_rng) {
    seed = (uint64_t) drop_rng[0];
    off = (uint64_t) drop_rng[1] + (uint64_t) drop_layer;
  }
  const int64_t ld = 3 * (int64_t) d.md;
  for (int64_t blk = blockIdx.x; blk < batch * d.H * d.nb; blk += gridDim.x) {
    int64_t b;
    int h, i0;
    ta_block_of(blk, d, b, h, i0);
    const int c0 = h * d.dh;
    const float* Xb = qkv + b * d.L * ld;
    const uint8_t* vb = valid + b * d.L;
    const int64_t bh = b * d.H + h;
    const int i = i0 + qr;
    const bool qlive = i < d.L && vb[i] != 0;
    float o[4][NV];
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
      for (int v = 0; v < NV; ++v) o[r][v] = 0.f;
    float m_run = -INFINITY, l_run = 0.f;
    if (ta_any_live(vb, i0, d.L)) {
      ta_stage(Xb, ld, i0, c0, d, Qs, scale);
      for (int j0 = 0; j0 < d.L; j0 += TA_TILE) {
        if (!ta_any_live(vb, j0, d.L)) continue;          // also orders the last tile's reads before the restage
        ta_stage(Xb, ld, j0, d.md + c0, d, Ks, 1.f);
        ta_stage(Xb, ld, j0, 2 * d.md + c0, d, Vs, 1.f);
        __syncthreads();
        float s[4], mt = -INFINITY;
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const int j = j0 + kg + 8 * u;
          s[u] = -INFINITY;
          if (qlive && j < d.L && vb[j]) s[u] = ta_dot(Qs + qr * d.DP, Ks + (kg + 8 * u) * d.DP, d.dh);
          mt = fmaxf(mt, s[u]);
        }
        for (int o_ = 1; o_ < 8; o_ <<= 1) mt = fmaxf(mt, __shfl_xor_sync(0xffffffffu, mt, o_));
        const float m_new = fmaxf(m_run, mt);
        const float alpha = m_new == -INFINITY ? 1.f : expf(m_run - m_new);
        float ls = 0.f;
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const int j = j0 + kg + 8 * u;
          float pv = s[u] == -INFINITY ? 0.f : expf(s[u] - m_new);
          ls += pv;
          if (drop_rng && pv != 0.f) pv = ta_keep(seed, off, b, h, i, j, d, drop_thresh) ? pv * drop_scale : 0.f;
          Ps[qr * TA_TP + kg + 8 * u] = pv;
        }
        for (int o_ = 1; o_ < 8; o_ <<= 1) ls += __shfl_xor_sync(0xffffffffu, ls, o_);
        l_run = l_run * alpha + ls;
        m_run = m_new;
        if (kg == 0) As[qr] = alpha;
        __syncthreads();
#pragma unroll
        for (int r = 0; r < 4; ++r) {
          const float a = As[4 * warp + r];
#pragma unroll
          for (int v = 0; v < NV; ++v) o[r][v] *= a;
        }
        const int jn = d.L - j0 < TA_TILE ? d.L - j0 : TA_TILE;
        for (int jj = 0; jj < jn; ++jj) {
          float vv[NV];
#pragma unroll
          for (int v = 0; v < NV; ++v) {
            const int c = lane + 32 * v;
            vv[v] = c < d.dh ? Vs[jj * d.DP + c] : 0.f;
          }
#pragma unroll
          for (int r = 0; r < 4; ++r) {
            const float pr = Ps[(4 * warp + r) * TA_TP + jj];
#pragma unroll
            for (int v = 0; v < NV; ++v) o[r][v] += pr * vv[v];
          }
        }
      }
    }
    __syncthreads();
    if (kg == 0) As[qr] = qlive ? 1.f / l_run : 0.f;
    if (kg == 0 && i < d.L) {
      stat_max[bh * d.L + i] = qlive ? m_run : 0.f;
      stat_sum[bh * d.L + i] = qlive ? l_run : 1.f;
    }
    __syncthreads();
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const int q = 4 * warp + r;
      if (i0 + q >= d.L) continue;
      const float inv = As[q];
      const int64_t row = b * d.L + i0 + q;
#pragma unroll
      for (int v = 0; v < NV; ++v) {
        const int c = lane + 32 * v;
        if (c < d.dh) {
          const float y = o[r][v] * inv;
          ctx[row * d.md + c0 + c] = y;
          if (aux) {
            const float w[1] = {y};
            rk_store_aux<1>(aux, aux_dtype, row * ld_aux + c0 + c, w);
          }
        }
      }
    }
  }
  b2_pdl_trigger();
}

// dQ pass, query-block outer.  With P the probabilities, P' = keep scale P, dP' = keep scale (dO . v_j):
//   D_i = dO_i . O_i ("=" into delta), dS = P (dP' - D), dq_i = scale sum_j dS_ij k_j ("=" into dqkv's Q columns)
template <int NV>
__global__ void __launch_bounds__(TA_THREADS, 1)
ta_attn_dq_kernel(const float* __restrict__ qkv, const uint8_t* __restrict__ valid, const float* __restrict__ ctx,
                  const float* __restrict__ dctx, const float* __restrict__ stat_max,
                  const float* __restrict__ stat_sum, int64_t batch, ta_dims d, float scale,
                  const int64_t* __restrict__ drop_rng, int64_t drop_layer, uint32_t drop_thresh, float drop_scale,
                  float* __restrict__ delta, float* __restrict__ dqkv, void* aux, int aux_dtype, int64_t ld_aux) {
  extern __shared__ float smem[];
  float* Qs = smem;                      // scaled q
  float* Gs = Qs + TA_TILE * d.DP;       // dO
  float* Ks = Gs + TA_TILE * d.DP;
  float* Vs = Ks + TA_TILE * d.DP;
  float* Ss = Vs + TA_TILE * d.DP;       // dS, TA_TILE x TA_TP
  float* Dd = Ss + TA_TILE * TA_TP;      // per query D_i
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int qr = tid >> 3, kg = tid & 7;
  b2_pdl_wait();
  uint64_t seed = 0, off = 0;
  if (drop_rng) {
    seed = (uint64_t) drop_rng[0];
    off = (uint64_t) drop_rng[1] + (uint64_t) drop_layer;
  }
  const int64_t ld = 3 * (int64_t) d.md;
  for (int64_t blk = blockIdx.x; blk < batch * d.H * d.nb; blk += gridDim.x) {
    int64_t b;
    int h, i0;
    ta_block_of(blk, d, b, h, i0);
    const int c0 = h * d.dh;
    const float* Xb = qkv + b * d.L * ld;
    const uint8_t* vb = valid + b * d.L;
    const int64_t bh = b * d.H + h;
    const int i = i0 + qr;
    const bool qlive = i < d.L && vb[i] != 0;
    float acc[4][NV];
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
      for (int v = 0; v < NV; ++v) acc[r][v] = 0.f;
    if (ta_any_live(vb, i0, d.L)) {
      ta_stage(Xb, ld, i0, c0, d, Qs, scale);
      ta_stage(dctx + b * d.L * d.md, d.md, i0, c0, d, Gs, 1.f);
      // D_i, warp per query
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        const int q = 4 * warp + r;
        float dd = 0.f;
        if (i0 + q < d.L) {
          const float* Ob = ctx + (b * d.L + i0 + q) * d.md + c0;
          for (int c = lane; c < d.dh; c += 32) dd += __ldg(dctx + (b * d.L + i0 + q) * d.md + c0 + c) * __ldg(Ob + c);
        }
        dd = b2_warp_sum(dd);
        if (lane == 0) {
          Dd[q] = dd;
          if (i0 + q < d.L) delta[bh * d.L + i0 + q] = dd;
        }
      }
      float m = 0.f, linv = 0.f;
      if (qlive) {
        m = __ldg(stat_max + bh * d.L + i);
        linv = 1.f / __ldg(stat_sum + bh * d.L + i);
      }
      for (int j0 = 0; j0 < d.L; j0 += TA_TILE) {
        if (!ta_any_live(vb, j0, d.L)) continue;
        ta_stage(Xb, ld, j0, d.md + c0, d, Ks, 1.f);
        ta_stage(Xb, ld, j0, 2 * d.md + c0, d, Vs, 1.f);
        __syncthreads();
        const float Di = Dd[qr];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const int j = j0 + kg + 8 * u;
          float ds = 0.f;
          if (qlive && j < d.L && vb[j]) {
            const float a = expf(ta_dot(Qs + qr * d.DP, Ks + (kg + 8 * u) * d.DP, d.dh) - m) * linv;
            float dp = ta_dot(Gs + qr * d.DP, Vs + (kg + 8 * u) * d.DP, d.dh);
            if (drop_rng) dp = ta_keep(seed, off, b, h, i, j, d, drop_thresh) ? dp * drop_scale : 0.f;
            ds = a * (dp - Di);
          }
          Ss[qr * TA_TP + kg + 8 * u] = ds;
        }
        __syncthreads();
        const int jn = d.L - j0 < TA_TILE ? d.L - j0 : TA_TILE;
        for (int jj = 0; jj < jn; ++jj) {
          float kv[NV];
#pragma unroll
          for (int v = 0; v < NV; ++v) {
            const int c = lane + 32 * v;
            kv[v] = c < d.dh ? Ks[jj * d.DP + c] : 0.f;
          }
#pragma unroll
          for (int r = 0; r < 4; ++r) {
            const float sr = Ss[(4 * warp + r) * TA_TP + jj];
#pragma unroll
            for (int v = 0; v < NV; ++v) acc[r][v] += sr * kv[v];
          }
        }
      }
    } else {
      for (int q = tid; q < TA_TILE && i0 + q < d.L; q += blockDim.x) delta[bh * d.L + i0 + q] = 0.f;
    }
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const int q = 4 * warp + r;
      if (i0 + q >= d.L) continue;
      const int64_t row = b * d.L + i0 + q;
#pragma unroll
      for (int v = 0; v < NV; ++v) {
        const int c = lane + 32 * v;
        if (c < d.dh) {
          const float y = acc[r][v] * scale;
          dqkv[row * ld + c0 + c] = y;
          if (aux) {
            const float w[1] = {y};
            rk_store_aux<1>(aux, aux_dtype, row * ld_aux + c0 + c, w);
          }
        }
      }
    }
    __syncthreads();
  }
  b2_pdl_trigger();
}

// dK, dV pass, key-block outer: dk_j = sum_i dS_ij (q_i scale), dv_j = sum_i P'_ij dO_i ("=" into dqkv's K, V columns)
template <int NV>
__global__ void __launch_bounds__(TA_THREADS, 1)
ta_attn_dkv_kernel(const float* __restrict__ qkv, const uint8_t* __restrict__ valid, const float* __restrict__ dctx,
                   const float* __restrict__ stat_max, const float* __restrict__ stat_sum,
                   const float* __restrict__ delta, int64_t batch, ta_dims d, float scale,
                   const int64_t* __restrict__ drop_rng, int64_t drop_layer, uint32_t drop_thresh, float drop_scale,
                   float* __restrict__ dqkv, void* aux, int aux_dtype, int64_t ld_aux) {
  extern __shared__ float smem[];
  float* Ks = smem;
  float* Vs = Ks + TA_TILE * d.DP;
  float* Qs = Vs + TA_TILE * d.DP;       // scaled q
  float* Gs = Qs + TA_TILE * d.DP;       // dO
  float* Ps = Gs + TA_TILE * d.DP;       // P', TA_TILE keys x TA_TP
  float* Ss = Ps + TA_TILE * TA_TP;      // dS
  float* Mq = Ss + TA_TILE * TA_TP;      // per query of the tile: max, 1 / sum, D
  float* Lq = Mq + TA_TILE;
  float* Dq = Lq + TA_TILE;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int kr = tid >> 3, qg = tid & 7;
  b2_pdl_wait();
  uint64_t seed = 0, off = 0;
  if (drop_rng) {
    seed = (uint64_t) drop_rng[0];
    off = (uint64_t) drop_rng[1] + (uint64_t) drop_layer;
  }
  const int64_t ld = 3 * (int64_t) d.md;
  for (int64_t blk = blockIdx.x; blk < batch * d.H * d.nb; blk += gridDim.x) {
    int64_t b;
    int h, j0;
    ta_block_of(blk, d, b, h, j0);
    const int c0 = h * d.dh;
    const float* Xb = qkv + b * d.L * ld;
    const float* Gb = dctx + b * d.L * d.md;
    const uint8_t* vb = valid + b * d.L;
    const int64_t bh = b * d.H + h;
    const int j = j0 + kr;
    const bool klive = j < d.L && vb[j] != 0;
    float dk[4][NV], dv[4][NV];
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
      for (int v = 0; v < NV; ++v) dk[r][v] = dv[r][v] = 0.f;
    if (ta_any_live(vb, j0, d.L)) {
      ta_stage(Xb, ld, j0, d.md + c0, d, Ks, 1.f);
      ta_stage(Xb, ld, j0, 2 * d.md + c0, d, Vs, 1.f);
      for (int i0 = 0; i0 < d.L; i0 += TA_TILE) {
        if (!ta_any_live(vb, i0, d.L)) continue;
        ta_stage(Xb, ld, i0, c0, d, Qs, scale);
        ta_stage(Gb, d.md, i0, c0, d, Gs, 1.f);
        if (tid < TA_TILE) {
          const int i = i0 + tid;
          const bool live = i < d.L && vb[i] != 0;
          Mq[tid] = live ? __ldg(stat_max + bh * d.L + i) : 0.f;
          Lq[tid] = live ? 1.f / __ldg(stat_sum + bh * d.L + i) : 0.f;
          Dq[tid] = live ? __ldg(delta + bh * d.L + i) : 0.f;
        }
        __syncthreads();
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const int qq = qg + 8 * u, i = i0 + qq;
          float ds = 0.f, pd = 0.f;
          if (klive && i < d.L && vb[i]) {
            const float a = expf(ta_dot(Qs + qq * d.DP, Ks + kr * d.DP, d.dh) - Mq[qq]) * Lq[qq];
            float dp = ta_dot(Gs + qq * d.DP, Vs + kr * d.DP, d.dh);
            pd = a;
            if (drop_rng) {
              const bool keep = ta_keep(seed, off, b, h, i, j, d, drop_thresh);
              dp = keep ? dp * drop_scale : 0.f;
              pd = keep ? a * drop_scale : 0.f;
            }
            ds = a * (dp - Dq[qq]);
          }
          Ps[kr * TA_TP + qq] = pd;
          Ss[kr * TA_TP + qq] = ds;
        }
        __syncthreads();
        const int in = d.L - i0 < TA_TILE ? d.L - i0 : TA_TILE;
        for (int ii = 0; ii < in; ++ii) {
          float qv[NV], gv[NV];
#pragma unroll
          for (int v = 0; v < NV; ++v) {
            const int c = lane + 32 * v;
            qv[v] = c < d.dh ? Qs[ii * d.DP + c] : 0.f;
            gv[v] = c < d.dh ? Gs[ii * d.DP + c] : 0.f;
          }
#pragma unroll
          for (int r = 0; r < 4; ++r) {
            const float sr = Ss[(4 * warp + r) * TA_TP + ii], pr = Ps[(4 * warp + r) * TA_TP + ii];
#pragma unroll
            for (int v = 0; v < NV; ++v) {
              dk[r][v] += sr * qv[v];
              dv[r][v] += pr * gv[v];
            }
          }
        }
      }
    }
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const int k = 4 * warp + r;
      if (j0 + k >= d.L) continue;
      const int64_t row = b * d.L + j0 + k;
#pragma unroll
      for (int v = 0; v < NV; ++v) {
        const int c = lane + 32 * v;
        if (c < d.dh) {
          dqkv[row * ld + d.md + c0 + c] = dk[r][v];
          dqkv[row * ld + 2 * d.md + c0 + c] = dv[r][v];
          if (aux) {
            const float wk[1] = {dk[r][v]}, wv[1] = {dv[r][v]};
            rk_store_aux<1>(aux, aux_dtype, row * ld_aux + d.md + c0 + c, wk);
            rk_store_aux<1>(aux, aux_dtype, row * ld_aux + 2 * d.md + c0 + c, wv);
          }
        }
      }
    }
    __syncthreads();
  }
  b2_pdl_trigger();
}

// ---------------------------------------------------------------------------------
// Output head: the last k slots (zeroed where padded) and the masked max over L, thread per (b, column)
// ---------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
ta_out_fwd_kernel(const float* __restrict__ y, const uint8_t* __restrict__ valid, int64_t batch, int L, int md, int k,
                  float* __restrict__ last, float* __restrict__ maxv, int32_t* __restrict__ argmax, void* aux,
                  int aux_dtype, int64_t ld_aux) {
  b2_pdl_wait();
  const int64_t nlast = batch * k * md, nmax = maxv ? batch * md : 0;
  for (int64_t e = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; e < nlast + nmax;
       e += (int64_t) gridDim.x * blockDim.x) {
    if (e < nlast) {
      const int64_t b = e / (k * md);
      const int r = (int) (e - b * k * md);
      const int t = L - k + r / md, c = r - (r / md) * md;
      last[e] = valid[b * L + t] ? __ldg(y + (b * L + t) * md + c) : 0.f;
    } else {
      const int64_t e2 = e - nlast;
      const int64_t b = e2 / md;
      const int c = (int) (e2 - b * md);
      // torch.max over the slots with the padded ones at -1e9: the first maximal slot wins
      float best = -INFINITY;
      int arg = 0;
      for (int t = 0; t < L; ++t) {
        const float v = valid[b * L + t] ? __ldg(y + (b * L + t) * md + c) : -1e9f;
        if (v > best) {
          best = v;
          arg = t;
        }
      }
      maxv[e2] = best;
      argmax[e2] = arg;
      if (aux) {
        const float w[1] = {best};
        rk_store_aux<1>(aux, aux_dtype, b * ld_aux + c, w);
      }
    }
  }
  b2_pdl_trigger();
}

// dy[b L + t, c] "=" dlast (t among the last k, not padded) + dmax (t the saved winner, not padded)
__global__ void __launch_bounds__(256)
ta_out_bwd_kernel(const float* __restrict__ dlast, const float* __restrict__ dmax, const int32_t* __restrict__ argmax,
                  const uint8_t* __restrict__ valid, int64_t batch, int L, int md, int k, float* __restrict__ dy) {
  b2_pdl_wait();
  const int64_t total = batch * L * md;
  for (int64_t e = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t) gridDim.x * blockDim.x) {
    const int64_t row = e / md;
    const int c = (int) (e - row * md);
    const int64_t b = row / L;
    const int t = (int) (row - b * L);
    float g = 0.f;
    if (valid[row]) {
      if (t >= L - k) g = __ldg(dlast + b * k * md + (int64_t) (t - (L - k)) * md + c);
      if (dmax && __ldg(argmax + b * md + c) == t) g += __ldg(dmax + b * md + c);
    }
    dy[e] = g;
  }
  b2_pdl_trigger();
}

// ---------------------------------------------------------------------------------
// Host side
// ---------------------------------------------------------------------------------
static int ta_check(int64_t batch, int L, int md) {
  B2_REQUIRE(L >= 1 && L <= B2_TRANSACT_MAX_LEN, "L = max_len %d outside [1, %d]", L, B2_TRANSACT_MAX_LEN);
  B2_REQUIRE(md >= 1 && md <= B2_TRANSACT_MAX_DIM, "model_dim %d outside [1, %d]", md, B2_TRANSACT_MAX_DIM);
  B2_REQUIRE(batch >= 0, "negative batch");
  B2_REQUIRE(batch <= (((int64_t) 1 << 31) - 1) / L, "batch * L >= 2^31");
  return B2_OK;
}

static int ta_grid(int64_t work, int per_block, int per_sm) {
  const int64_t blocks = b2_ceil_div(work, per_block), cap = (int64_t) B2_NUM_SMS * per_sm;
  return (int) (blocks < 1 ? 1 : (blocks > cap ? cap : blocks));
}

static int ta_parts_fill(ta_parts& p, int ns, int nt, const float* const* seq, const int64_t* seq_ld,
                         const float* const* tgt, const int64_t* tgt_ld, float* const* dseq, float* const* dtgt) {
  B2_REQUIRE(ns >= 1 && nt >= 1 && ns + nt <= B2_TRANSACT_MAX_PARTS, "fields per token %d + %d outside [2, %d]", ns,
             nt, B2_TRANSACT_MAX_PARTS);
  for (int f = 0; f < B2_TRANSACT_MAX_PARTS; ++f) {
    const bool is_seq = f < ns, in = f < ns + nt;
    const int g = is_seq ? f : f - ns;
    p.src[f] = in && seq ? (is_seq ? seq[g] : tgt[g]) : nullptr;
    p.ld[f] = in && seq ? (is_seq ? seq_ld[g] : tgt_ld[g]) : 0;
    p.dst[f] = in && dseq ? (is_seq ? dseq[g] : dtgt[g]) : nullptr;
    if (in && seq) B2_REQUIRE(p.src[f], "NULL embedding view %d", f);
    if (in && dseq) B2_REQUIRE(p.dst[f], "NULL embedding gradient %d", f);
  }
  return B2_OK;
}

template <typename K>
static int ta_smem_optin(K kernel, size_t smem) {
  cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) smem);
  if (e != cudaSuccess) return b2_fail(B2_E_CUDA, "transact: shared memory opt-in failed: %s", cudaGetErrorString(e));
  return B2_OK;
}

extern "C" B2_API int b2_transact_tokens_fwd(const float* const* seq, const int64_t* seq_ld, int ns,
                                             const float* const* tgt, const int64_t* tgt_ld, int nt, const void* ids,
                                             int ids_dtype, int64_t ld_ids, int64_t batch, int L, int D, float* tok,
                                             void* tok_aux, int aux_dtype, int64_t ld_aux, uint8_t* valid,
                                             void* stream) {
  B2_REQUIRE(seq && seq_ld && tgt && tgt_ld && ids && tok && valid, "NULL pointer");
  B2_REQUIRE(D >= 1, "embedding_dim %d < 1", D);
  B2_REQUIRE(ids_dtype == B2_F64 || ids_dtype == B2_I64 || ids_dtype == B2_I32 || ids_dtype == B2_F32,
             "ids dtype %d is not B2_F64, B2_I64, B2_I32 or B2_F32", ids_dtype);
  ta_parts p;
  if (int rc = ta_parts_fill(p, ns, nt, seq, seq_ld, tgt, tgt_ld, nullptr, nullptr)) return rc;
  const int md = D * (ns + nt);
  if (int rc = ta_check(batch, L, md)) return rc;
  B2_REQUIRE(ld_ids >= L, "ld_ids %lld < L %d", (long long) ld_ids, L);
  for (int f = 0; f < ns; ++f) B2_REQUIRE(seq_ld[f] >= (int64_t) L * D, "sequence view %d: row pitch too small", f);
  for (int f = 0; f < nt; ++f) B2_REQUIRE(tgt_ld[f] >= D, "target view %d: row pitch too small", f);
  if (int rc = rk_check_aux(tok_aux, aux_dtype, ld_aux, md)) return rc;
  if (batch == 0) return B2_OK;
  B2_LAUNCH(ta_tokens_fwd_kernel, ta_grid(batch * L * md, 256, 8), 256, 0, (cudaStream_t) stream, p, ns, nt, ids,
            ids_dtype, ld_ids, batch, L, D, tok, tok_aux, aux_dtype, ld_aux, valid);
  B2_CUDA_LAUNCH_CHECK("b2_transact_tokens_fwd");
  return B2_OK;
}

extern "C" B2_API int b2_transact_tokens_bwd(const float* g, int64_t batch, int L, int D, int ns, int nt,
                                             float* const* dseq, float* const* dtgt, void* stream) {
  B2_REQUIRE(g && dseq && dtgt, "NULL pointer");
  B2_REQUIRE(D >= 1, "embedding_dim %d < 1", D);
  ta_parts p;
  if (int rc = ta_parts_fill(p, ns, nt, nullptr, nullptr, nullptr, nullptr, dseq, dtgt)) return rc;
  if (int rc = ta_check(batch, L, D * (ns + nt))) return rc;
  if (batch == 0) return B2_OK;
  B2_LAUNCH(ta_tokens_bwd_kernel, ta_grid(batch * (L * ns + nt) * D, 256, 8), 256, 0, (cudaStream_t) stream, g,
            batch, L, D, ns, nt, p);
  B2_CUDA_LAUNCH_CHECK("b2_transact_tokens_bwd");
  return B2_OK;
}

static int ta_attn_check(int64_t batch, int L, int md, int heads, float scale) {
  if (int rc = ta_check(batch, L, md)) return rc;
  B2_REQUIRE(heads >= 1 && heads <= B2_TRANSACT_MAX_HEADS, "heads %d outside [1, %d]", heads, B2_TRANSACT_MAX_HEADS);
  B2_REQUIRE(md % heads == 0, "heads %d do not divide model_dim %d", heads, md);
  B2_REQUIRE(md / heads <= B2_TRANSACT_MAX_HEAD_DIM, "head width %d > %d", md / heads, B2_TRANSACT_MAX_HEAD_DIM);
  B2_REQUIRE(scale > 0.f, "scale must be positive");
  return B2_OK;
}

static ta_dims ta_make_dims(int L, int md, int heads) {
  ta_dims d;
  d.L = L;
  d.md = md;
  d.H = heads;
  d.dh = md / heads;
  d.DP = d.dh + 1;
  d.nb = (L + TA_TILE - 1) / TA_TILE;
  return d;
}

static int ta_per_sm(size_t smem) {
  const int64_t n = 220 * 1024 / (int64_t) (smem + 1024);
  return (int) (n < 1 ? 1 : (n > 8 ? 8 : n));
}

#define TA_NV_DISPATCH(dh, MACRO) \
  do {                            \
    if ((dh) <= 32) MACRO(1);     \
    else if ((dh) <= 64) MACRO(2);  \
    else if ((dh) <= 128) MACRO(4); \
    else MACRO(8);                \
  } while (0)

extern "C" B2_API int b2_transact_attn_fwd(const float* qkv, const uint8_t* valid, int64_t batch, int L, int md,
                                           int heads, float scale, const int64_t* drop_rng, int64_t drop_layer,
                                           uint32_t drop_thresh, float drop_scale, float* ctx, void* ctx_aux,
                                           int aux_dtype, int64_t ld_aux, float* stat_max, float* stat_sum,
                                           void* stream) {
  B2_REQUIRE(qkv && valid && ctx && stat_max && stat_sum, "NULL pointer");
  if (int rc = ta_attn_check(batch, L, md, heads, scale)) return rc;
  if (int rc = rk_check_aux(ctx_aux, aux_dtype, ld_aux, md)) return rc;
  if (batch == 0) return B2_OK;
  const ta_dims d = ta_make_dims(L, md, heads);
  const size_t smem = (size_t) (3 * TA_TILE * d.DP + TA_TILE * TA_TP + TA_TILE) * sizeof(float);
  const int grid = ta_grid(batch * heads * d.nb, 1, ta_per_sm(smem));
  const cudaStream_t st = (cudaStream_t) stream;
#define TA_ATTN_FWD(NV)                                                                                       \
  do {                                                                                                        \
    if (int rc = ta_smem_optin(ta_attn_fwd_kernel<NV>, smem)) return rc;                                      \
    B2_LAUNCH(ta_attn_fwd_kernel<NV>, grid, TA_THREADS, smem, st, qkv, valid, batch, d, scale, drop_rng,      \
              drop_layer, drop_thresh, drop_scale, ctx, ctx_aux, aux_dtype, ld_aux, stat_max, stat_sum);       \
  } while (0)
  TA_NV_DISPATCH(d.dh, TA_ATTN_FWD);
#undef TA_ATTN_FWD
  B2_CUDA_LAUNCH_CHECK("b2_transact_attn_fwd");
  return B2_OK;
}

extern "C" B2_API int b2_transact_attn_bwd(const float* qkv, const uint8_t* valid, const float* ctx,
                                           const float* dctx, const float* stat_max, const float* stat_sum,
                                           int64_t batch, int L, int md, int heads, float scale,
                                           const int64_t* drop_rng, int64_t drop_layer, uint32_t drop_thresh,
                                           float drop_scale, float* delta, float* dqkv, void* dqkv_aux,
                                           int aux_dtype, int64_t ld_aux, void* stream) {
  B2_REQUIRE(qkv && valid && ctx && dctx && stat_max && stat_sum && delta && dqkv, "NULL pointer");
  if (int rc = ta_attn_check(batch, L, md, heads, scale)) return rc;
  if (int rc = rk_check_aux(dqkv_aux, aux_dtype, ld_aux, 3 * md)) return rc;
  if (batch == 0) return B2_OK;
  const ta_dims d = ta_make_dims(L, md, heads);
  const cudaStream_t st = (cudaStream_t) stream;
  const size_t smem_q = (size_t) (4 * TA_TILE * d.DP + TA_TILE * TA_TP + TA_TILE) * sizeof(float);
  const size_t smem_kv = (size_t) (4 * TA_TILE * d.DP + 2 * TA_TILE * TA_TP + 3 * TA_TILE) * sizeof(float);
  const int grid_q = ta_grid(batch * heads * d.nb, 1, ta_per_sm(smem_q));
  const int grid_kv = ta_grid(batch * heads * d.nb, 1, ta_per_sm(smem_kv));
#define TA_ATTN_BWD(NV)                                                                                         \
  do {                                                                                                          \
    if (int rc = ta_smem_optin(ta_attn_dq_kernel<NV>, smem_q)) return rc;                                       \
    if (int rc = ta_smem_optin(ta_attn_dkv_kernel<NV>, smem_kv)) return rc;                                     \
    B2_LAUNCH(ta_attn_dq_kernel<NV>, grid_q, TA_THREADS, smem_q, st, qkv, valid, ctx, dctx, stat_max, stat_sum, \
              batch, d, scale, drop_rng, drop_layer, drop_thresh, drop_scale, delta, dqkv, dqkv_aux, aux_dtype, \
              ld_aux);                                                                                          \
    B2_LAUNCH(ta_attn_dkv_kernel<NV>, grid_kv, TA_THREADS, smem_kv, st, qkv, valid, dctx, stat_max, stat_sum,   \
              delta, batch, d, scale, drop_rng, drop_layer, drop_thresh, drop_scale, dqkv, dqkv_aux, aux_dtype, \
              ld_aux);                                                                                          \
  } while (0)
  TA_NV_DISPATCH(d.dh, TA_ATTN_BWD);
#undef TA_ATTN_BWD
  B2_CUDA_LAUNCH_CHECK("b2_transact_attn_bwd");
  return B2_OK;
}

extern "C" B2_API int b2_transact_out_fwd(const float* y, const uint8_t* valid, int64_t batch, int L, int md, int k,
                                          float* last, float* maxv, int32_t* argmax, void* max_aux, int aux_dtype,
                                          int64_t ld_aux, void* stream) {
  B2_REQUIRE(y && valid && last, "NULL pointer");
  B2_REQUIRE((maxv == nullptr) == (argmax == nullptr), "maxv and argmax: both or neither");
  if (int rc = ta_check(batch, L, md)) return rc;
  B2_REQUIRE(k >= 1 && k <= L, "first_k_cols %d outside [1, L = %d]", k, L);
  if (int rc = rk_check_aux(max_aux, aux_dtype, ld_aux, md)) return rc;
  B2_REQUIRE(max_aux == nullptr || maxv, "max_aux needs maxv");
  if (batch == 0) return B2_OK;
  B2_LAUNCH(ta_out_fwd_kernel, ta_grid(batch * (k + (maxv ? 1 : 0)) * md, 256, 8), 256, 0, (cudaStream_t) stream, y,
            valid, batch, L, md, k, last, maxv, argmax, max_aux, aux_dtype, ld_aux);
  B2_CUDA_LAUNCH_CHECK("b2_transact_out_fwd");
  return B2_OK;
}

extern "C" B2_API int b2_transact_out_bwd(const float* dlast, const float* dmax, const int32_t* argmax,
                                          const uint8_t* valid, int64_t batch, int L, int md, int k, float* dy,
                                          void* stream) {
  B2_REQUIRE(dlast && valid && dy, "NULL pointer");
  B2_REQUIRE(dmax == nullptr || argmax, "dmax needs argmax");
  if (int rc = ta_check(batch, L, md)) return rc;
  B2_REQUIRE(k >= 1 && k <= L, "first_k_cols %d outside [1, L = %d]", k, L);
  if (batch == 0) return B2_OK;
  B2_LAUNCH(ta_out_bwd_kernel, ta_grid(batch * L * md, 256, 8), 256, 0, (cudaStream_t) stream, dlast, dmax, argmax,
            valid, batch, L, md, k, dy);
  B2_CUDA_LAUNCH_CHECK("b2_transact_out_bwd");
  return B2_OK;
}

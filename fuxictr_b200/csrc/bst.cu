// bst.cu — the Behavior Sequence Transformer's row kernels (model_zoo/BST/src/BST.py), sm_90a.
//
// A TransformerBlock on the token matrix X (B L, md) is the in-projection GEMM, the masked self-attention row kernel,
// the out-projection GEMM, the residual + dropout + LayerNorm row kernel, the FFN as a two-layer MLP chain (LeakyReLU,
// B2_ACT_LEAKY_RELU, in its first GEMM's epilogue, dropout2 in its second's) and the residual + LayerNorm row kernel
// again; the GEMMs are the project's gemm_ex / gemm_f32.
// This file holds the row kernels, the token assembly (embeddings and position table -> X) and the sequence pooling.
// Layouts and range: include/fuxictr_b200.h "BST".
//
// Attention: one CTA of BST_THREADS threads per (sample, head).  Forward and backward stage two L x dh tiles in
// shared memory at a row pitch of dh + 1 (lane j reading row j meets no bank conflict); each warp takes query rows
// i = warp, warp + 8, ... and each lane keys j = lane, lane + 32, ..., so a softmax is two warp reductions.  No score
// or probability reaches HBM: the forward saves the softmax max and sum per (b, h, i) and the backward recomputes the
// probabilities from them (exactly: the same code on the same operands) and regenerates the dropout mask.  The
// backward runs in two phases: K, V staged, warp per query (dQ); then Q, dO staged, warp per key (dK, dV).
// The key-padding mask comes from a (B, L - 1) byte mask of real history slots; no (B H, L, L) mask exists.
// All arithmetic is fp32 on CUDA cores, expf (not __expf).
#include "row_common.cuh"
#include "philox.cuh"

#define BST_THREADS 256
#define BST_WARPS (BST_THREADS / 32)

struct bst_parts {
  const float* seq[B2_BST_MAX_PARTS];
  const float* tgt[B2_BST_MAX_PARTS];
  int64_t seq_ld[B2_BST_MAX_PARTS];
  int64_t tgt_ld[B2_BST_MAX_PARTS];
  float* dseq[B2_BST_MAX_PARTS];
  float* dtgt[B2_BST_MAX_PARTS];
};

// ---------------------------------------------------------------------------------
// Token assembly
// ---------------------------------------------------------------------------------
// X[b L + t, :] = [seq_0[b, t] .. seq_{nf-1}[b, t] | pos[t]] for t < L - 1, [tgt_0[b] .. tgt_{nf-1}[b] | pos[L-1]]
// for t = L - 1 ("=", with X's GEMM operand copy)
__global__ void __launch_bounds__(256)
bst_tokens_fwd_kernel(bst_parts p, const float* __restrict__ pos, int64_t batch, int L, int D, int nf, int md,
                      float* __restrict__ tok, void* aux, int aux_dtype, int64_t ld_aux) {
  b2_pdl_wait();
  const int64_t total = batch * L * md;
  for (int64_t e = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t) gridDim.x * blockDim.x) {
    const int64_t row = e / md;
    const int c = (int) (e - row * md);
    const int64_t b = row / L;
    const int t = (int) (row - b * L);
    float v;
    if (c < nf * D) {
      const int f = c / D, d = c - f * D;
      v = t < L - 1 ? __ldg(p.seq[f] + b * p.seq_ld[f] + (int64_t) t * D + d) : __ldg(p.tgt[f] + b * p.tgt_ld[f] + d);
    } else {
      v = __ldg(pos + (int64_t) t * D + (c - nf * D));
    }
    tok[e] = v;
    if (aux) {
      const float w[1] = {v};
      rk_store_aux<1>(aux, aux_dtype, row * ld_aux + c, w);
    }
  }
  b2_pdl_trigger();
}

// G = g (+ g2) (B L, md): the embedding parts "=" into dseq / dtgt, the position part summed over the batch "+="
// into dpos.  A CTA is 32 token columns (of the L md of a sample) x 8 warps striding over the batch.
__global__ void __launch_bounds__(256)
bst_tokens_bwd_kernel(const float* __restrict__ g, const float* __restrict__ g2, int64_t batch, int L, int D, int nf,
                      int md, bst_parts p, float* __restrict__ dpos) {
  __shared__ float red[BST_WARPS][32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  b2_pdl_wait();
  const int col = blockIdx.x * 32 + lane;         // t md + c
  const int t = col / md, c = col - t * md;
  const bool live = col < L * md;
  float acc = 0.f;
  for (int64_t b = (int64_t) blockIdx.y * BST_WARPS + warp; live && b < batch; b += (int64_t) gridDim.y * BST_WARPS) {
    const int64_t e = b * L * md + col;
    float v = __ldg(g + e);
    if (g2) v += __ldg(g2 + e);
    if (c < nf * D) {
      const int f = c / D, d = c - f * D;
      if (t < L - 1) p.dseq[f][(b * (L - 1) + t) * D + d] = v;
      else p.dtgt[f][b * D + d] = v;
    } else {
      acc += v;
    }
  }
  b2_pdl_trigger();
  if (dpos == nullptr) return;
  red[warp][lane] = acc;
  __syncthreads();
  if (warp == 0 && live && c >= nf * D) {
    float s = 0.f;
    for (int w = 0; w < BST_WARPS; ++w) s += red[w][lane];
    if (s != 0.f) b2_red_add(dpos + (int64_t) t * D + (c - nf * D), s);
  }
}

// ---------------------------------------------------------------------------------
// Masked multi-head self-attention
// ---------------------------------------------------------------------------------
struct bst_dims {
  int L, md, H, dh, DP, causal;      // tokens, model_dim, heads, head width, smem pitch dh + 1, causal mask
};

// Key j masked for query i: a padded history slot other than i itself, or (causal) a later token.
__device__ __forceinline__ bool bst_masked(const uint8_t* __restrict__ valid_b, const bst_dims d, int i, int j) {
  if (j == i) return false;
  if (d.causal && j > i) return true;
  return j < d.L - 1 && valid_b[j] == 0;
}

__device__ __forceinline__ float bst_dot(const float* a, const float* b, int n) {
  float s = 0.f;
  for (int t = 0; t < n; ++t) s += a[t] * b[t];
  return s;
}

// The dropout keep of probability (b, h, i, j): element ((b H + h) L + i) L + j of the (B, H, L, L) weights.
__device__ __forceinline__ bool bst_keep(uint64_t seed, uint64_t off, int64_t b, int h, int i, int j,
                                         const bst_dims d, uint32_t thresh) {
  const uint64_t idx = (((uint64_t) b * d.H + h) * d.L + i) * d.L + j;
  return b2_drop_keep(seed, off, idx, thresh);
}

// Stage columns c0 .. c0 + dh - 1 of the sample's L rows of M (row pitch ld) into S (L x DP); `scale` multiplies.
__device__ __forceinline__ void bst_stage(const float* __restrict__ M, int64_t ld, int c0, const bst_dims d, float* S,
                                          float scale) {
  for (int t = threadIdx.x; t < d.L * d.dh; t += blockDim.x) {
    const int r = t / d.dh, c = t - r * d.dh;
    const float v = __ldg(M + r * ld + c0 + c);
    S[r * d.DP + c] = scale != 1.f ? v * scale : v;
  }
}

// ctx[b L + i, h dh + c] = sum_j dropout(softmax_j((q_i scale) . k_j + mask)) v_j[c].  KPL keys per lane (L <= 32 KPL):
// the scores stay in registers, and a short sequence's instantiation holds few enough for four CTAs per SM.
template <int KPL>
__global__ void __launch_bounds__(BST_THREADS, KPL <= 2 ? 4 : 2)
bst_attn_fwd_kernel(const float* __restrict__ qkv, const uint8_t* __restrict__ valid, int64_t batch, bst_dims d,
                    float scale, const int64_t* __restrict__ drop_rng, int64_t drop_layer, uint32_t drop_thresh,
                    float drop_scale, float* __restrict__ ctx, void* aux, int aux_dtype, int64_t ld_aux,
                    float* __restrict__ stat_max, float* __restrict__ stat_sum) {
  extern __shared__ float smem[];
  float* Ks = smem;
  float* Vs = Ks + d.L * d.DP;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  float* qw = Vs + d.L * d.DP + warp * (d.dh + d.L);     // this warp's scaled query, then its probabilities
  float* pw = qw + d.dh;
  b2_pdl_wait();
  uint64_t seed = 0, off = 0;
  if (drop_rng) {
    seed = (uint64_t) drop_rng[0];
    off = (uint64_t) drop_rng[1] + (uint64_t) drop_layer;
  }
  const int64_t ld = 3 * (int64_t) d.md;
  for (int64_t bh = blockIdx.x; bh < batch * d.H; bh += gridDim.x) {
    const int64_t b = bh / d.H;
    const int h = (int) (bh - b * d.H), c0 = h * d.dh;
    const float* Xb = qkv + b * d.L * ld;
    const uint8_t* vb = valid + b * (d.L - 1);
    __syncthreads();
    bst_stage(Xb, ld, d.md + c0, d, Ks, 1.f);
    bst_stage(Xb, ld, 2 * d.md + c0, d, Vs, 1.f);
    __syncthreads();
    for (int i = warp; i < d.L; i += BST_WARPS) {
      for (int c = lane; c < d.dh; c += 32) qw[c] = __ldg(Xb + i * ld + c0 + c) * scale;
      __syncwarp();
      float s[KPL], m = -INFINITY;
#pragma unroll
      for (int u = 0; u < KPL; ++u) {
        const int j = lane + 32 * u;
        s[u] = -INFINITY;
        if (j < d.L && !bst_masked(vb, d, i, j)) s[u] = bst_dot(qw, Ks + j * d.DP, d.dh);
        m = fmaxf(m, s[u]);
      }
      for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
      float l = 0.f;
#pragma unroll
      for (int u = 0; u < KPL; ++u) {
        s[u] = lane + 32 * u < d.L ? expf(s[u] - m) : 0.f;
        l += s[u];
      }
      l = b2_warp_sum(l);
#pragma unroll
      for (int u = 0; u < KPL; ++u) {
        const int j = lane + 32 * u;
        if (j < d.L) {
          float a = s[u] / l;
          if (drop_rng) a = bst_keep(seed, off, b, h, i, j, d, drop_thresh) ? a * drop_scale : 0.f;
          pw[j] = a;
        }
      }
      __syncwarp();
      const int64_t row = b * d.L + i;
      for (int c = lane; c < d.dh; c += 32) {
        float o = 0.f;
        for (int j = 0; j < d.L; ++j) o += pw[j] * Vs[j * d.DP + c];
        ctx[row * d.md + c0 + c] = o;
        if (aux) {
          const float w[1] = {o};
          rk_store_aux<1>(aux, aux_dtype, row * ld_aux + c0 + c, w);
        }
      }
      if (lane == 0) {
        stat_max[bh * d.L + i] = m;
        stat_sum[bh * d.L + i] = l;
      }
      __syncwarp();
    }
  }
  b2_pdl_trigger();
}

// dQKV from dO = dctx: with P the probabilities, P' = keep scale P and dP' = dO . v_j,
//   dS = P (keep scale dP' - dO . O),  dq_i = scale sum_j dS_ij k_j,  dk_j = sum_i dS_ij (q_i scale),
//   dv_j = sum_i P'_ij dO_i   ("=" into dqkv, with its GEMM operand copy)
__global__ void __launch_bounds__(BST_THREADS, 4)
bst_attn_bwd_kernel(const float* __restrict__ qkv, const uint8_t* __restrict__ valid, const float* __restrict__ ctx,
                    const float* __restrict__ dctx, const float* __restrict__ stat_max,
                    const float* __restrict__ stat_sum, int64_t batch, bst_dims d, float scale,
                    const int64_t* __restrict__ drop_rng, int64_t drop_layer, uint32_t drop_thresh, float drop_scale,
                    float* __restrict__ dqkv, void* aux, int aux_dtype, int64_t ld_aux) {
  extern __shared__ float smem[];
  float* S0 = smem;                   // K, then the scaled Q
  float* S1 = S0 + d.L * d.DP;        // V, then dO
  float* Dm = S1 + d.L * d.DP;        // per query: dO . O, the softmax max and sum
  float* Mm = Dm + d.L;
  float* Lm = Mm + d.L;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  float* aw = Lm + d.L + warp * 2 * (d.dh + d.L);    // this warp's two row vectors and two key/query vectors
  float* bw = aw + d.dh;
  float* pw = bw + d.dh;
  float* sw = pw + d.L;
  b2_pdl_wait();
  uint64_t seed = 0, off = 0;
  if (drop_rng) {
    seed = (uint64_t) drop_rng[0];
    off = (uint64_t) drop_rng[1] + (uint64_t) drop_layer;
  }
  const int64_t ld = 3 * (int64_t) d.md;
  for (int64_t bh = blockIdx.x; bh < batch * d.H; bh += gridDim.x) {
    const int64_t b = bh / d.H;
    const int h = (int) (bh - b * d.H), c0 = h * d.dh;
    const float* Xb = qkv + b * d.L * ld;
    const float* Ob = ctx + b * d.L * d.md;
    const float* Gb = dctx + b * d.L * d.md;
    const uint8_t* vb = valid + b * (d.L - 1);
    __syncthreads();
    bst_stage(Xb, ld, d.md + c0, d, S0, 1.f);
    bst_stage(Xb, ld, 2 * d.md + c0, d, S1, 1.f);
    __syncthreads();
    // phase 1: warp per query i -> dq_i; D_i = dO_i . O_i, m_i, l_i to shared
    for (int i = warp; i < d.L; i += BST_WARPS) {
      const int64_t row = b * d.L + i;
      float dd = 0.f;
      for (int c = lane; c < d.dh; c += 32) {
        aw[c] = __ldg(Xb + i * ld + c0 + c) * scale;
        const float go = __ldg(Gb + i * d.md + c0 + c);
        bw[c] = go;
        dd += go * __ldg(Ob + i * d.md + c0 + c);
      }
      dd = b2_warp_sum(dd);
      __syncwarp();
      const float m = __ldg(stat_max + bh * d.L + i), l = __ldg(stat_sum + bh * d.L + i);
      for (int j = lane; j < d.L; j += 32) {
        float ds = 0.f;
        if (!bst_masked(vb, d, i, j)) {
          const float a = expf(bst_dot(aw, S0 + j * d.DP, d.dh) - m) / l;
          float dp = bst_dot(bw, S1 + j * d.DP, d.dh);
          if (drop_rng) dp = bst_keep(seed, off, b, h, i, j, d, drop_thresh) ? dp * drop_scale : 0.f;
          ds = a * (dp - dd);
        }
        sw[j] = ds;
      }
      __syncwarp();
      for (int c = lane; c < d.dh; c += 32) {
        float dq = 0.f;
        for (int j = 0; j < d.L; ++j) dq += sw[j] * S0[j * d.DP + c];
        dq *= scale;
        dqkv[row * ld + c0 + c] = dq;
        if (aux) {
          const float w[1] = {dq};
          rk_store_aux<1>(aux, aux_dtype, row * ld_aux + c0 + c, w);
        }
      }
      if (lane == 0) {
        Dm[i] = dd;
        Mm[i] = m;
        Lm[i] = l;
      }
      __syncwarp();
    }
    __syncthreads();
    bst_stage(Xb, ld, c0, d, S0, scale);
    bst_stage(Gb, d.md, c0, d, S1, 1.f);
    __syncthreads();
    // phase 2: warp per key j -> dk_j, dv_j
    for (int j = warp; j < d.L; j += BST_WARPS) {
      const int64_t row = b * d.L + j;
      for (int c = lane; c < d.dh; c += 32) {
        aw[c] = __ldg(Xb + j * ld + d.md + c0 + c);
        bw[c] = __ldg(Xb + j * ld + 2 * d.md + c0 + c);
      }
      __syncwarp();
      for (int i = lane; i < d.L; i += 32) {
        float ds = 0.f, ad = 0.f;
        if (!bst_masked(vb, d, i, j)) {
          const float a = expf(bst_dot(S0 + i * d.DP, aw, d.dh) - Mm[i]) / Lm[i];
          float dp = bst_dot(S1 + i * d.DP, bw, d.dh);
          ad = a;
          if (drop_rng) {
            const bool keep = bst_keep(seed, off, b, h, i, j, d, drop_thresh);
            dp = keep ? dp * drop_scale : 0.f;
            ad = keep ? a * drop_scale : 0.f;
          }
          ds = a * (dp - Dm[i]);
        }
        pw[i] = ad;
        sw[i] = ds;
      }
      __syncwarp();
      for (int c = lane; c < d.dh; c += 32) {
        float dk = 0.f, dv = 0.f;
        for (int i = 0; i < d.L; ++i) {
          dk += sw[i] * S0[i * d.DP + c];
          dv += pw[i] * S1[i * d.DP + c];
        }
        dqkv[row * ld + d.md + c0 + c] = dk;
        dqkv[row * ld + 2 * d.md + c0 + c] = dv;
        if (aux) {
          const float wk[1] = {dk}, wv[1] = {dv};
          rk_store_aux<1>(aux, aux_dtype, row * ld_aux + d.md + c0 + c, wk);
          rk_store_aux<1>(aux, aux_dtype, row * ld_aux + 2 * d.md + c0 + c, wv);
        }
      }
      __syncwarp();
    }
  }
  b2_pdl_trigger();
}

// ---------------------------------------------------------------------------------
// Residual + dropout + LayerNorm, warp per row, lane l owning columns l, l + 32, ... (NU of them)
// ---------------------------------------------------------------------------------
// out = LN(res + dropout(a)) (LN and res optional), with out's GEMM operand copy; mean, rstd per row "="
template <int NU>
__global__ void __launch_bounds__(256)
bst_addnorm_fwd_kernel(const float* __restrict__ a, const float* __restrict__ res, int64_t rows, int n,
                       const float* __restrict__ gamma, const float* __restrict__ beta, float eps,
                       const int64_t* __restrict__ drop_rng, int64_t drop_layer, uint32_t drop_thresh,
                       float drop_scale, float* __restrict__ out, void* aux, int aux_dtype, int64_t ld_aux,
                       float* __restrict__ ln_mean, float* __restrict__ ln_rstd) {
  const int lane = threadIdx.x & 31;
  b2_pdl_wait();
  uint64_t seed = 0, off = 0;
  if (drop_rng) {
    seed = (uint64_t) drop_rng[0];
    off = (uint64_t) drop_rng[1] + (uint64_t) drop_layer;
  }
  const int64_t nwarps = (int64_t) gridDim.x * (blockDim.x >> 5);
  for (int64_t row = (int64_t) blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); row < rows; row += nwarps) {
    float z[NU], sum = 0.f;
#pragma unroll
    for (int u = 0; u < NU; ++u) {
      const int c = lane + 32 * u;
      z[u] = 0.f;
      if (c < n) {
        float v = __ldg(a + row * n + c);
        if (drop_rng) v = b2_drop_keep(seed, off, (uint64_t) (row * n + c), drop_thresh) ? v * drop_scale : 0.f;
        if (res) v += __ldg(res + row * n + c);
        z[u] = v;
        sum += v;
      }
    }
    float mu = 0.f, rs = 1.f;
    if (gamma) {
      mu = b2_warp_sum(sum) / (float) n;
      float q = 0.f;
#pragma unroll
      for (int u = 0; u < NU; ++u) {
        const float dz = z[u] - mu;
        if (lane + 32 * u < n) q += dz * dz;
      }
      rs = 1.f / sqrtf(b2_warp_sum(q) / (float) n + eps);
      if (lane == 0) {
        ln_mean[row] = mu;
        ln_rstd[row] = rs;
      }
    }
#pragma unroll
    for (int u = 0; u < NU; ++u) {
      const int c = lane + 32 * u;
      if (c < n) {
        const float y = gamma ? (z[u] - mu) * rs * __ldg(gamma + c) + __ldg(beta + c) : z[u];
        out[row * n + c] = y;
        if (aux) {
          const float w[1] = {y};
          rk_store_aux<1>(aux, aux_dtype, row * ld_aux + c, w);
        }
      }
    }
  }
  b2_pdl_trigger();
}

// From G = g (+ g2): dz = LN'(G) (z recomputed from a, res and the mask), dres = dz "=", da = keep scale dz "="
// (with its GEMM operand copy); dgamma, dbeta "+=": per-CTA sums, one float atomic per column and CTA.
template <int NU>
__global__ void __launch_bounds__(256)
bst_addnorm_bwd_kernel(const float* __restrict__ a, const float* __restrict__ res, const float* __restrict__ g,
                       const float* __restrict__ g2, int64_t rows, int n, const float* __restrict__ gamma,
                       const float* __restrict__ ln_mean, const float* __restrict__ ln_rstd,
                       const int64_t* __restrict__ drop_rng, int64_t drop_layer, uint32_t drop_thresh,
                       float drop_scale, float* __restrict__ da, void* aux, int aux_dtype, int64_t ld_aux,
                       float* __restrict__ dres, float* __restrict__ dgamma, float* __restrict__ dbeta) {
  __shared__ float sg[B2_BST_MAX_DIM], sb[B2_BST_MAX_DIM];
  const int lane = threadIdx.x & 31;
  const bool affine = gamma != nullptr;
  if (affine) {
    for (int c = threadIdx.x; c < n; c += blockDim.x) sg[c] = sb[c] = 0.f;
  }
  __syncthreads();
  float acc_g[NU], acc_b[NU];
#pragma unroll
  for (int u = 0; u < NU; ++u) acc_g[u] = acc_b[u] = 0.f;
  b2_pdl_wait();
  uint64_t seed = 0, off = 0;
  if (drop_rng) {
    seed = (uint64_t) drop_rng[0];
    off = (uint64_t) drop_rng[1] + (uint64_t) drop_layer;
  }
  const int64_t nwarps = (int64_t) gridDim.x * (blockDim.x >> 5);
  for (int64_t row = (int64_t) blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); row < rows; row += nwarps) {
    float gy[NU], xh[NU], s1 = 0.f, s2 = 0.f, mu = 0.f, rs = 1.f;
    if (affine) {
      mu = __ldg(ln_mean + row);
      rs = __ldg(ln_rstd + row);
    }
#pragma unroll
    for (int u = 0; u < NU; ++u) {
      const int c = lane + 32 * u;
      gy[u] = xh[u] = 0.f;
      if (c < n) {
        gy[u] = __ldg(g + row * n + c);
        if (g2) gy[u] += __ldg(g2 + row * n + c);
        if (affine) {
          float z = __ldg(a + row * n + c);
          if (drop_rng) z = b2_drop_keep(seed, off, (uint64_t) (row * n + c), drop_thresh) ? z * drop_scale : 0.f;
          if (res) z += __ldg(res + row * n + c);
          xh[u] = (z - mu) * rs;
          const float t = __fmul_rn(gy[u], __ldg(gamma + c));
          s1 += t;
          s2 += t * xh[u];
          acc_g[u] += gy[u] * xh[u];
          acc_b[u] += gy[u];
        }
      }
    }
    if (affine) {
      s1 = b2_warp_sum(s1) / (float) n;
      s2 = b2_warp_sum(s2) / (float) n;
    }
#pragma unroll
    for (int u = 0; u < NU; ++u) {
      const int c = lane + 32 * u;
      if (c < n) {
        const float dz = affine ? rs * ((__fmul_rn(gy[u], __ldg(gamma + c)) - s1) - xh[u] * s2) : gy[u];
        if (dres) dres[row * n + c] = dz;
        float v = dz;
        if (drop_rng) v = b2_drop_keep(seed, off, (uint64_t) (row * n + c), drop_thresh) ? v * drop_scale : 0.f;
        da[row * n + c] = v;
        if (aux) {
          const float w[1] = {v};
          rk_store_aux<1>(aux, aux_dtype, row * ld_aux + c, w);
        }
      }
    }
  }
  b2_pdl_trigger();
  if (!affine) return;
#pragma unroll
  for (int u = 0; u < NU; ++u) {
    const int c = lane + 32 * u;
    if (c < n) {
      if (acc_g[u] != 0.f) atomicAdd(&sg[c], acc_g[u]);
      if (acc_b[u] != 0.f) atomicAdd(&sb[c], acc_b[u]);
    }
  }
  __syncthreads();
  for (int c = threadIdx.x; c < n; c += blockDim.x) {
    if (sg[c] != 0.f) b2_red_add(dgamma + c, sg[c]);
    if (sb[c] != 0.f) b2_red_add(dbeta + c, sb[c]);
  }
}

// ---------------------------------------------------------------------------------
// Pooling over the L tokens, warp per sample
// ---------------------------------------------------------------------------------
// weight of token t: mean / sum: 1 for real history slots and the target, 0 for padding; target: the last token only
__device__ __forceinline__ float bst_pool_w(const uint8_t* valid_b, int L, int mode, int t) {
  if (t == L - 1) return 1.f;
  return mode == B2_BST_POOL_TARGET ? 0.f : (valid_b[t] ? 1.f : 0.f);
}

__device__ __forceinline__ float bst_pool_den(const uint8_t* valid_b, int L, int mode) {
  if (mode != B2_BST_POOL_MEAN) return 1.f;
  float cnt = 1.f;
  for (int t = 0; t < L - 1; ++t) cnt += valid_b[t] ? 1.f : 0.f;
  return cnt + 1e-12f;
}

__global__ void __launch_bounds__(256)
bst_pool_fwd_kernel(const float* __restrict__ x, const uint8_t* __restrict__ valid, int64_t batch, int L, int md,
                    int mode, float* __restrict__ out, int64_t ld_out) {
  const int lane = threadIdx.x & 31;
  b2_pdl_wait();
  const int64_t nwarps = (int64_t) gridDim.x * (blockDim.x >> 5);
  for (int64_t b = (int64_t) blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); b < batch; b += nwarps) {
    const uint8_t* vb = valid + b * (L - 1);
    const float den = bst_pool_den(vb, L, mode);
    for (int c = lane; c < md; c += 32) {
      float s = 0.f;
      for (int t = 0; t < L; ++t) s += __ldg(x + (b * L + t) * md + c) * bst_pool_w(vb, L, mode, t);
      out[b * ld_out + c] = mode == B2_BST_POOL_MEAN ? s / den : s;
    }
  }
  b2_pdl_trigger();
}

__global__ void __launch_bounds__(256)
bst_pool_bwd_kernel(const float* __restrict__ g, int64_t ld_g, const uint8_t* __restrict__ valid, int64_t batch, int L,
                    int md, int mode, float* __restrict__ dx) {
  const int lane = threadIdx.x & 31;
  b2_pdl_wait();
  const int64_t nwarps = (int64_t) gridDim.x * (blockDim.x >> 5);
  for (int64_t b = (int64_t) blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); b < batch; b += nwarps) {
    const uint8_t* vb = valid + b * (L - 1);
    const float den = bst_pool_den(vb, L, mode);
    for (int c = lane; c < md; c += 32) {
      float gv = __ldg(g + b * ld_g + c);
      if (mode == B2_BST_POOL_MEAN) gv = gv / den;
      for (int t = 0; t < L; ++t) dx[(b * L + t) * md + c] = gv * bst_pool_w(vb, L, mode, t);
    }
  }
  b2_pdl_trigger();
}

// ---------------------------------------------------------------------------------
// Host side
// ---------------------------------------------------------------------------------
static int bst_check(int64_t batch, int L, int md) {
  B2_REQUIRE(L >= 2 && L <= B2_BST_MAX_LEN, "L = max_len + 1 = %d outside [2, %d]", L, B2_BST_MAX_LEN);
  B2_REQUIRE(md >= 1 && md <= B2_BST_MAX_DIM, "model_dim %d outside [1, %d]", md, B2_BST_MAX_DIM);
  B2_REQUIRE(batch >= 0, "negative batch");
  B2_REQUIRE(batch <= (((int64_t) 1 << 31) - 1) / L, "batch * L >= 2^31");
  return B2_OK;
}

static int bst_grid(int64_t work, int per_block, int per_sm) {
  const int64_t blocks = b2_ceil_div(work, per_block), cap = (int64_t) B2_NUM_SMS * per_sm;
  return (int) (blocks < 1 ? 1 : (blocks > cap ? cap : blocks));
}

static int bst_parts_fill(bst_parts& p, int nf, const float* const* seq, const int64_t* seq_ld, const float* const* tgt,
                          const int64_t* tgt_ld, float* const* dseq, float* const* dtgt) {
  B2_REQUIRE(nf >= 1 && nf <= B2_BST_MAX_PARTS, "fields per token %d outside [1, %d]", nf, B2_BST_MAX_PARTS);
  for (int f = 0; f < B2_BST_MAX_PARTS; ++f) {
    const bool in = f < nf;
    p.seq[f] = in && seq ? seq[f] : nullptr;
    p.tgt[f] = in && tgt ? tgt[f] : nullptr;
    p.seq_ld[f] = in && seq_ld ? seq_ld[f] : 0;
    p.tgt_ld[f] = in && tgt_ld ? tgt_ld[f] : 0;
    p.dseq[f] = in && dseq ? dseq[f] : nullptr;
    p.dtgt[f] = in && dtgt ? dtgt[f] : nullptr;
    if (in && seq) B2_REQUIRE(p.seq[f] && p.tgt[f], "NULL embedding view of field %d", f);
    if (in && dseq) B2_REQUIRE(p.dseq[f] && p.dtgt[f], "NULL embedding gradient of field %d", f);
  }
  return B2_OK;
}

template <typename K>
static int bst_smem_optin(K kernel, size_t smem) {
  cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) smem);
  if (e != cudaSuccess) return b2_fail(B2_E_CUDA, "bst: shared memory opt-in failed: %s", cudaGetErrorString(e));
  return B2_OK;
}

extern "C" B2_API int b2_bst_tokens_fwd(const float* const* seq, const int64_t* seq_ld, const float* const* tgt,
                                        const int64_t* tgt_ld, int nf, const float* pos, int64_t batch, int L, int D,
                                        float* tok, void* tok_aux, int aux_dtype, int64_t ld_aux, void* stream) {
  B2_REQUIRE(seq && seq_ld && tgt && tgt_ld && tok, "NULL pointer");
  B2_REQUIRE(D >= 1, "embedding_dim %d < 1", D);
  bst_parts p;
  if (int rc = bst_parts_fill(p, nf, seq, seq_ld, tgt, tgt_ld, nullptr, nullptr)) return rc;
  const int md = D * (nf + (pos ? 1 : 0));
  if (int rc = bst_check(batch, L, md)) return rc;
  for (int f = 0; f < nf; ++f)
    B2_REQUIRE(seq_ld[f] >= (int64_t) (L - 1) * D && tgt_ld[f] >= D, "embedding view %d: row pitch too small", f);
  if (int rc = rk_check_aux(tok_aux, aux_dtype, ld_aux, md)) return rc;
  if (batch == 0) return B2_OK;
  B2_LAUNCH(bst_tokens_fwd_kernel, bst_grid(batch * L * md, 256, 8), 256, 0, (cudaStream_t) stream, p, pos, batch, L,
            D, nf, md, tok, tok_aux, aux_dtype, ld_aux);
  B2_CUDA_LAUNCH_CHECK("b2_bst_tokens_fwd");
  return B2_OK;
}

extern "C" B2_API int b2_bst_tokens_bwd(const float* g, const float* g2, int64_t batch, int L, int D, int nf,
                                        int use_pos, float* const* dseq, float* const* dtgt, float* dpos,
                                        void* stream) {
  B2_REQUIRE(g && dseq && dtgt, "NULL pointer");
  B2_REQUIRE(D >= 1, "embedding_dim %d < 1", D);
  B2_REQUIRE(!use_pos || dpos, "use_pos needs dpos");
  bst_parts p;
  if (int rc = bst_parts_fill(p, nf, nullptr, nullptr, nullptr, nullptr, dseq, dtgt)) return rc;
  const int md = D * (nf + (use_pos ? 1 : 0));
  if (int rc = bst_check(batch, L, md)) return rc;
  if (batch == 0) return B2_OK;
  const int64_t gy = b2_ceil_div(batch, BST_WARPS * 16);
  const dim3 grid((unsigned) b2_ceil_div((int64_t) L * md, 32), (unsigned) (gy > 64 ? 64 : gy));
  B2_LAUNCH(bst_tokens_bwd_kernel, grid, 256, 0, (cudaStream_t) stream, g, g2, batch, L, D, nf, md, p,
            use_pos ? dpos : nullptr);
  B2_CUDA_LAUNCH_CHECK("b2_bst_tokens_bwd");
  return B2_OK;
}

static int bst_attn_check(int64_t batch, int L, int md, int heads) {
  if (int rc = bst_check(batch, L, md)) return rc;
  B2_REQUIRE(heads >= 1 && heads <= B2_BST_MAX_HEADS, "heads %d outside [1, %d]", heads, B2_BST_MAX_HEADS);
  B2_REQUIRE(md % heads == 0, "heads %d do not divide model_dim %d", heads, md);
  B2_REQUIRE(md / heads <= B2_BST_MAX_HEAD_DIM, "head width %d > %d", md / heads, B2_BST_MAX_HEAD_DIM);
  B2_REQUIRE(batch * heads <= (((int64_t) 1 << 31) - 1), "batch * heads >= 2^31");
  return B2_OK;
}

static bst_dims bst_make_dims(int L, int md, int heads, int causal) {
  bst_dims d;
  d.L = L;
  d.md = md;
  d.H = heads;
  d.dh = md / heads;
  d.DP = d.dh + 1;
  d.causal = causal ? 1 : 0;
  return d;
}

extern "C" B2_API int b2_bst_attn_fwd(const float* qkv, const uint8_t* valid, int64_t batch, int L, int md, int heads,
                                      int causal, float scale, const int64_t* drop_rng, int64_t drop_layer,
                                      uint32_t drop_thresh, float drop_scale, float* ctx, void* ctx_aux, int aux_dtype,
                                      int64_t ld_aux, float* stat_max, float* stat_sum, void* stream) {
  B2_REQUIRE(qkv && valid && ctx && stat_max && stat_sum, "NULL pointer");
  if (int rc = bst_attn_check(batch, L, md, heads)) return rc;
  B2_REQUIRE(scale > 0.f, "scale must be positive");
  if (int rc = rk_check_aux(ctx_aux, aux_dtype, ld_aux, md)) return rc;
  if (batch == 0) return B2_OK;
  const bst_dims d = bst_make_dims(L, md, heads, causal);
  const size_t smem = (size_t) (2 * L * d.DP + BST_WARPS * (d.dh + L)) * sizeof(float);
  const int64_t per_sm = 200 * 1024 / (int64_t) (smem + 1024);
  const int grid = bst_grid(batch * heads, 1, (int) (per_sm < 1 ? 1 : (per_sm > 8 ? 8 : per_sm)));
  const cudaStream_t st = (cudaStream_t) stream;
#define BST_ATTN_FWD(KPL)                                                                                      \
  do {                                                                                                         \
    if (int rc = bst_smem_optin(bst_attn_fwd_kernel<KPL>, smem)) return rc;                                    \
    B2_LAUNCH(bst_attn_fwd_kernel<KPL>, grid, BST_THREADS, smem, st, qkv, valid, batch, d, scale, drop_rng,   \
              drop_layer, drop_thresh, drop_scale, ctx, ctx_aux, aux_dtype, ld_aux, stat_max, stat_sum);        \
  } while (0)
  if (L <= 32) BST_ATTN_FWD(1);
  else if (L <= 64) BST_ATTN_FWD(2);
  else if (L <= 128) BST_ATTN_FWD(4);
  else BST_ATTN_FWD(8);
#undef BST_ATTN_FWD
  B2_CUDA_LAUNCH_CHECK("b2_bst_attn_fwd");
  return B2_OK;
}

extern "C" B2_API int b2_bst_attn_bwd(const float* qkv, const uint8_t* valid, const float* ctx, const float* dctx,
                                      const float* stat_max, const float* stat_sum, int64_t batch, int L, int md,
                                      int heads, int causal, float scale, const int64_t* drop_rng, int64_t drop_layer,
                                      uint32_t drop_thresh, float drop_scale, float* dqkv, void* dqkv_aux,
                                      int aux_dtype, int64_t ld_aux, void* stream) {
  B2_REQUIRE(qkv && valid && ctx && dctx && stat_max && stat_sum && dqkv, "NULL pointer");
  if (int rc = bst_attn_check(batch, L, md, heads)) return rc;
  B2_REQUIRE(scale > 0.f, "scale must be positive");
  if (int rc = rk_check_aux(dqkv_aux, aux_dtype, ld_aux, 3 * md)) return rc;
  if (batch == 0) return B2_OK;
  const bst_dims d = bst_make_dims(L, md, heads, causal);
  const size_t smem = (size_t) (2 * L * d.DP + 3 * L + BST_WARPS * 2 * (d.dh + L)) * sizeof(float);
  if (int rc = bst_smem_optin(bst_attn_bwd_kernel, smem)) return rc;
  const int64_t per_sm = 200 * 1024 / (int64_t) (smem + 1024);
  B2_LAUNCH(bst_attn_bwd_kernel, bst_grid(batch * heads, 1, (int) (per_sm < 1 ? 1 : (per_sm > 8 ? 8 : per_sm))),
            BST_THREADS, smem, (cudaStream_t) stream, qkv, valid, ctx, dctx, stat_max, stat_sum, batch, d, scale,
            drop_rng, drop_layer, drop_thresh, drop_scale, dqkv, dqkv_aux, aux_dtype, ld_aux);
  B2_CUDA_LAUNCH_CHECK("b2_bst_attn_bwd");
  return B2_OK;
}

#define BST_NU_DISPATCH(n, KERNEL, ...)                                      \
  do {                                                                       \
    if ((n) <= 32) B2_LAUNCH(KERNEL<1>, __VA_ARGS__);                        \
    else if ((n) <= 64) B2_LAUNCH(KERNEL<2>, __VA_ARGS__);                   \
    else if ((n) <= 128) B2_LAUNCH(KERNEL<4>, __VA_ARGS__);                  \
    else if ((n) <= 256) B2_LAUNCH(KERNEL<8>, __VA_ARGS__);                  \
    else B2_LAUNCH(KERNEL<16>, __VA_ARGS__);                                 \
  } while (0)

extern "C" B2_API int b2_bst_addnorm_fwd(const float* a, const float* res, int64_t rows, int n, const float* gamma,
                                         const float* beta, float eps, const int64_t* drop_rng, int64_t drop_layer,
                                         uint32_t drop_thresh, float drop_scale, float* out, void* out_aux,
                                         int aux_dtype, int64_t ld_aux, float* ln_mean, float* ln_rstd,
                                         void* stream) {
  B2_REQUIRE(a && out, "NULL pointer");
  B2_REQUIRE(n >= 1 && n <= B2_BST_MAX_DIM, "width %d outside [1, %d]", n, B2_BST_MAX_DIM);
  B2_REQUIRE(rows >= 0, "negative rows");
  B2_REQUIRE((gamma == nullptr) == (beta == nullptr), "gamma and beta: both or neither");
  B2_REQUIRE(gamma == nullptr || (ln_mean && ln_rstd), "LayerNorm needs ln_mean and ln_rstd");
  if (int rc = rk_check_aux(out_aux, aux_dtype, ld_aux, n)) return rc;
  if (rows == 0) return B2_OK;
  const int grid = bst_grid(rows, BST_WARPS, 8);
  BST_NU_DISPATCH(n, bst_addnorm_fwd_kernel, grid, 256, 0, (cudaStream_t) stream, a, res, rows, n, gamma, beta, eps,
                  drop_rng, drop_layer, drop_thresh, drop_scale, out, out_aux, aux_dtype, ld_aux, ln_mean, ln_rstd);
  B2_CUDA_LAUNCH_CHECK("b2_bst_addnorm_fwd");
  return B2_OK;
}

extern "C" B2_API int b2_bst_addnorm_bwd(const float* a, const float* res, const float* g, const float* g2,
                                         int64_t rows, int n, const float* gamma, const float* ln_mean,
                                         const float* ln_rstd, const int64_t* drop_rng, int64_t drop_layer,
                                         uint32_t drop_thresh, float drop_scale, float* da, void* da_aux,
                                         int aux_dtype, int64_t ld_aux, float* dres, float* dgamma, float* dbeta,
                                         void* stream) {
  B2_REQUIRE(g && da, "NULL pointer");
  B2_REQUIRE(n >= 1 && n <= B2_BST_MAX_DIM, "width %d outside [1, %d]", n, B2_BST_MAX_DIM);
  B2_REQUIRE(rows >= 0, "negative rows");
  B2_REQUIRE(gamma == nullptr || (a && ln_mean && ln_rstd && dgamma && dbeta),
             "LayerNorm needs a, ln_mean, ln_rstd, dgamma and dbeta");
  if (int rc = rk_check_aux(da_aux, aux_dtype, ld_aux, n)) return rc;
  if (rows == 0) return B2_OK;
  const int grid = bst_grid(rows, BST_WARPS, 4);
  BST_NU_DISPATCH(n, bst_addnorm_bwd_kernel, grid, 256, 0, (cudaStream_t) stream, a, res, g, g2, rows, n, gamma,
                  ln_mean, ln_rstd, drop_rng, drop_layer, drop_thresh, drop_scale, da, da_aux, aux_dtype, ld_aux,
                  dres, dgamma, dbeta);
  B2_CUDA_LAUNCH_CHECK("b2_bst_addnorm_bwd");
  return B2_OK;
}

extern "C" B2_API int b2_bst_pool_fwd(const float* x, const uint8_t* valid, int64_t batch, int L, int md, int mode,
                                      float* out, int64_t ld_out, void* stream) {
  B2_REQUIRE(x && valid && out, "NULL pointer");
  if (int rc = bst_check(batch, L, md)) return rc;
  B2_REQUIRE(mode == B2_BST_POOL_MEAN || mode == B2_BST_POOL_SUM || mode == B2_BST_POOL_TARGET,
             "pooling mode %d is not B2_BST_POOL_MEAN, _SUM or _TARGET", mode);
  B2_REQUIRE(ld_out >= md, "ld_out %lld < model_dim %d", (long long) ld_out, md);
  if (batch == 0) return B2_OK;
  B2_LAUNCH(bst_pool_fwd_kernel, bst_grid(batch, BST_WARPS, 8), 256, 0, (cudaStream_t) stream, x, valid, batch, L, md,
            mode, out, ld_out);
  B2_CUDA_LAUNCH_CHECK("b2_bst_pool_fwd");
  return B2_OK;
}

extern "C" B2_API int b2_bst_pool_bwd(const float* g, int64_t ld_g, const uint8_t* valid, int64_t batch, int L, int md,
                                      int mode, float* dx, void* stream) {
  B2_REQUIRE(g && valid && dx, "NULL pointer");
  if (int rc = bst_check(batch, L, md)) return rc;
  B2_REQUIRE(mode == B2_BST_POOL_MEAN || mode == B2_BST_POOL_SUM || mode == B2_BST_POOL_TARGET,
             "pooling mode %d is not B2_BST_POOL_MEAN, _SUM or _TARGET", mode);
  B2_REQUIRE(ld_g >= md, "ld_g %lld < model_dim %d", (long long) ld_g, md);
  if (batch == 0) return B2_OK;
  B2_LAUNCH(bst_pool_bwd_kernel, bst_grid(batch, BST_WARPS, 8), 256, 0, (cudaStream_t) stream, g, ld_g, valid, batch, L,
            md, mode, dx);
  B2_CUDA_LAUNCH_CHECK("b2_bst_pool_bwd");
  return B2_OK;
}

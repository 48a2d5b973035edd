// autoint.cu — AutoInt's multi-head field self-attention (model_zoo/AutoInt/src/AutoInt.py, MultiHeadSelfAttention),
// sm_90a.
//
// One layer on X (B, F, d_in) is one GEMM P = X Wp^T on the stacked Wp = [W_q; W_k; W_v (; W_res)] and one row
// kernel; this file holds the pack of Wp, the row kernels forward and backward, and the split of dWp.  Layouts and
// range: include/fuxictr_b200.h "AutoInt".
//
// Row kernels: one CTA of AI_THREADS threads per sample (grid stride over the batch).  The sample's Q, K and V
// (F x A each) are staged in shared memory at a row pitch of A + 1, so that lane j reading key row j for a score
// meets no bank conflict.  Per head: each warp takes query rows i = warp, warp + 8, ... and each lane keys
// j = lane, lane + 32, so the softmax over the keys is two warp reductions; the (dropped) probabilities go to a
// shared F x F tile, and all threads then form the head's output columns from it.  No score or probability ever
// reaches HBM: the forward saves the softmax max and sum per (b, h, i), the backward recomputes the probabilities
// from them (exactly: the same code on the same operands) and regenerates the dropout mask.
// The residual, the LayerNorm (nn.LayerNorm: mean first, then the biased variance from the centred values, eps
// inside the square root) and the ReLU run warp per row, lane l owning columns l and l + 32.
// All arithmetic is fp32 on CUDA cores; expf (not __expf), and the scores divided by scale as the reference does.
#include "row_common.cuh"
#include "philox.cuh"

#define AI_THREADS 256
#define AI_WARPS (AI_THREADS / 32)

struct ai_dims {
  int F, A, H, dh, NP, AP, FP;      // fields, attention_dim, heads, head width, P's row width, smem pitches
};

// Stage the sample's Q, K, V (columns 0 .. 3A - 1 of its F rows of P) into Qs, Ks, Vs (consecutive F x AP tiles).
template <int VW>
__device__ __forceinline__ void ai_stage(const float* __restrict__ Pb, const ai_dims& d, float* Qs) {
  const int per_row = 3 * d.A / VW;
  for (int t = threadIdx.x; t < d.F * per_row; t += blockDim.x) {
    const int i = t / per_row, cc = (t % per_row) * VW;
    const int part = cc / d.A, c = cc % d.A;
    float v[VW];
    rk_load<VW>(Pb + (int64_t) i * d.NP + cc, v);
    float* dst = Qs + part * d.F * d.AP + i * d.AP + c;
#pragma unroll
    for (int e = 0; e < VW; ++e) dst[e] = v[e];
  }
}

// Score of query row i with key row j in the head whose columns start at c0.
__device__ __forceinline__ float ai_score(const float* Qs, const float* Ks, const ai_dims& d, int i, int j, int c0,
                                          float scale) {
  const float* q = Qs + i * d.AP + c0;
  const float* k = Ks + j * d.AP + c0;
  float s = 0.f;
  for (int t = 0; t < d.dh; ++t) s += q[t] * k[t];
  return scale != 0.f ? s / scale : s;
}

// The dropout keep of probability (b, h, i, j): element ((b H + h) F + i) F + j of the layer's (B, H, F, F) weights.
__device__ __forceinline__ bool ai_keep(uint64_t seed, uint64_t off, int64_t b, int h, int i, int j, const ai_dims& d,
                                        uint32_t thresh) {
  const uint64_t idx = (((uint64_t) b * d.H + h) * d.F + i) * d.F + j;
  return b2_drop_keep(seed, off, idx, thresh);
}

// out = ReLU(LN(concat_h softmax(Q_h K_h^T [/ scale]) V_h + R))
template <int VW>
__global__ void __launch_bounds__(AI_THREADS)
ai_fwd_kernel(const float* __restrict__ P, const float* __restrict__ X, int64_t batch, ai_dims d, int res_mode,
              float scale, const float* __restrict__ gamma, const float* __restrict__ beta, float eps,
              const int64_t* __restrict__ drop_rng, int64_t drop_layer, uint32_t drop_thresh, float drop_scale,
              float* __restrict__ out, void* out_aux, int aux_dtype, int64_t ld_aux, float* __restrict__ stat_max,
              float* __restrict__ stat_sum, float* __restrict__ ln_mean, float* __restrict__ ln_rstd) {
  extern __shared__ float smem[];
  float* Qs = smem;
  float* Ks = Qs + d.F * d.AP;
  float* Vs = Ks + d.F * d.AP;
  float* Os = Vs + d.F * d.AP;
  float* Ps = Os + d.F * d.AP;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  b2_pdl_wait();
  uint64_t seed = 0, off = 0;
  if (drop_rng) {
    seed = (uint64_t) drop_rng[0];
    off = (uint64_t) drop_rng[1] + (uint64_t) drop_layer;
  }
  for (int64_t b = blockIdx.x; b < batch; b += gridDim.x) {
    const float* Pb = P + b * d.F * d.NP;
    ai_stage<VW>(Pb, d, Qs);
    __syncthreads();
    for (int h = 0; h < d.H; ++h) {
      const int c0 = h * d.dh;
      for (int i = warp; i < d.F; i += AI_WARPS) {
        float s[2], m = -INFINITY;
#pragma unroll
        for (int u = 0; u < 2; ++u) {
          const int j = lane + 32 * u;
          s[u] = j < d.F ? ai_score(Qs, Ks, d, i, j, c0, scale) : -INFINITY;
          m = fmaxf(m, s[u]);
        }
        for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
        float e[2];
#pragma unroll
        for (int u = 0; u < 2; ++u) e[u] = lane + 32 * u < d.F ? expf(s[u] - m) : 0.f;
        const float l = b2_warp_sum(e[0] + e[1]);
#pragma unroll
        for (int u = 0; u < 2; ++u) {
          const int j = lane + 32 * u;
          if (j < d.F) {
            float a = e[u] / l;
            if (drop_rng) a = ai_keep(seed, off, b, h, i, j, d, drop_thresh) ? a * drop_scale : 0.f;
            Ps[i * d.FP + j] = a;
          }
        }
        if (lane == 0) {
          const int64_t si = (b * d.H + h) * d.F + i;
          stat_max[si] = m;
          stat_sum[si] = l;
        }
      }
      __syncthreads();
      for (int t = threadIdx.x; t < d.F * d.dh; t += blockDim.x) {
        const int i = t / d.dh, c = c0 + t % d.dh;
        float o = 0.f;
        for (int j = 0; j < d.F; ++j) o += Ps[i * d.FP + j] * Vs[j * d.AP + c];
        Os[i * d.AP + c] = o;
      }
      __syncthreads();
    }
    for (int i = warp; i < d.F; i += AI_WARPS) {
      const int64_t row = b * d.F + i;
      float z[2], sum = 0.f;
#pragma unroll
      for (int u = 0; u < 2; ++u) {
        const int c = lane + 32 * u;
        z[u] = 0.f;
        if (c < d.A) {
          z[u] = Os[i * d.AP + c];
          if (res_mode == 1) z[u] += __ldg(X + row * d.A + c);
          else if (res_mode == 2) z[u] += __ldg(P + row * d.NP + 3 * d.A + c);
          sum += z[u];
        }
      }
      float mu = 0.f, rs = 1.f;
      if (gamma) {
        mu = b2_warp_sum(sum) / (float) d.A;
        float q = 0.f;
#pragma unroll
        for (int u = 0; u < 2; ++u) {
          const float dz = z[u] - mu;
          if (lane + 32 * u < d.A) q += dz * dz;
        }
        rs = 1.f / sqrtf(b2_warp_sum(q) / (float) d.A + eps);
        if (lane == 0) {
          ln_mean[row] = mu;
          ln_rstd[row] = rs;
        }
      }
#pragma unroll
      for (int u = 0; u < 2; ++u) {
        const int c = lane + 32 * u;
        if (c < d.A) {
          float y = gamma ? (z[u] - mu) * rs * __ldg(gamma + c) + __ldg(beta + c) : z[u];
          y = y > 0.f ? y : 0.f;
          out[row * d.A + c] = y;
          if (out_aux) {
            const float t[1] = {y};
            rk_store_aux<1>(out_aux, aux_dtype, row * ld_aux + c, t);
          }
        }
      }
    }
    __syncthreads();
  }
  b2_pdl_trigger();
}

// From the output gradient g and the saved out: dZ = LN'(ReLU'(out) g), the residual's gradient (P's W_res slot of
// dP, or gres for an identity residual), then per head dV = A'^T dO, dS = A (dA - rowsum(A dA)) [/ scale] with
// dA = keep scale (dO V^T), dQ = dS K, dK = dS^T Q into dP; dgamma, dbeta "+=".
template <int VW>
__global__ void __launch_bounds__(AI_THREADS)
ai_bwd_kernel(const float* __restrict__ P, const float* __restrict__ X, const float* __restrict__ out,
              const float* __restrict__ g, const float* __restrict__ stat_max, const float* __restrict__ stat_sum,
              const float* __restrict__ ln_mean, const float* __restrict__ ln_rstd, int64_t batch, ai_dims d,
              int res_mode, float scale, const float* __restrict__ gamma, const int64_t* __restrict__ drop_rng,
              int64_t drop_layer, uint32_t drop_thresh, float drop_scale, float* __restrict__ dP, void* dp_aux,
              int aux_dtype, int64_t ld_aux, float* __restrict__ gres, float* __restrict__ dgamma,
              float* __restrict__ dbeta) {
  extern __shared__ float smem[];
  __shared__ float sg[B2_AUTOINT_MAX_DIM], sb[B2_AUTOINT_MAX_DIM];
  float* Qs = smem;
  float* Ks = Qs + d.F * d.AP;
  float* Vs = Ks + d.F * d.AP;
  float* Os = Vs + d.F * d.AP;      // O, then dO
  float* Ps = Os + d.F * d.AP;      // the dropped probabilities A' of one head
  float* Ss = Ps + d.F * d.FP;      // dS of one head
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const bool affine = gamma != nullptr && dgamma != nullptr;
  if (affine) {
    for (int c = threadIdx.x; c < d.A; c += blockDim.x) sg[c] = sb[c] = 0.f;
  }
  float acc_g[2] = {0.f, 0.f}, acc_b[2] = {0.f, 0.f};
  b2_pdl_wait();
  uint64_t seed = 0, off = 0;
  if (drop_rng) {
    seed = (uint64_t) drop_rng[0];
    off = (uint64_t) drop_rng[1] + (uint64_t) drop_layer;
  }
  for (int64_t b = blockIdx.x; b < batch; b += gridDim.x) {
    const float* Pb = P + b * d.F * d.NP;
    ai_stage<VW>(Pb, d, Qs);
    __syncthreads();
    // the forward's attention output O, recomputed: only the LayerNorm backward reads Z = O + R
    for (int h = 0; gamma != nullptr && h < d.H; ++h) {
      const int c0 = h * d.dh;
      for (int i = warp; i < d.F; i += AI_WARPS) {
        const int64_t si = (b * d.H + h) * d.F + i;
        const float m = __ldg(stat_max + si), l = __ldg(stat_sum + si);
#pragma unroll
        for (int u = 0; u < 2; ++u) {
          const int j = lane + 32 * u;
          if (j < d.F) {
            float a = expf(ai_score(Qs, Ks, d, i, j, c0, scale) - m) / l;
            if (drop_rng) a = ai_keep(seed, off, b, h, i, j, d, drop_thresh) ? a * drop_scale : 0.f;
            Ps[i * d.FP + j] = a;
          }
        }
      }
      __syncthreads();
      for (int t = threadIdx.x; t < d.F * d.dh; t += blockDim.x) {
        const int i = t / d.dh, c = c0 + t % d.dh;
        float o = 0.f;
        for (int j = 0; j < d.F; ++j) o += Ps[i * d.FP + j] * Vs[j * d.AP + c];
        Os[i * d.AP + c] = o;
      }
      __syncthreads();
    }
    // dZ per row: ReLU' from the saved output, then the LayerNorm backward on Z = O + R recomputed
    for (int i = warp; i < d.F; i += AI_WARPS) {
      const int64_t row = b * d.F + i;
      float gy[2], xh[2], s1 = 0.f, s2 = 0.f;
      float mu = 0.f, rs = 1.f;
      if (gamma) {
        mu = __ldg(ln_mean + row);
        rs = __ldg(ln_rstd + row);
      }
#pragma unroll
      for (int u = 0; u < 2; ++u) {
        const int c = lane + 32 * u;
        gy[u] = xh[u] = 0.f;
        if (c < d.A) {
          gy[u] = __ldg(out + row * d.A + c) > 0.f ? __ldg(g + row * d.A + c) : 0.f;
          if (gamma) {
            float z = Os[i * d.AP + c];
            if (res_mode == 1) z += __ldg(X + row * d.A + c);
            else if (res_mode == 2) z += __ldg(P + row * d.NP + 3 * d.A + c);
            xh[u] = (z - mu) * rs;
            const float t = __fmul_rn(gy[u], __ldg(gamma + c));
            s1 += t;
            s2 += t * xh[u];
            acc_g[u] += gy[u] * xh[u];
            acc_b[u] += gy[u];
          }
        }
      }
      if (gamma) {
        s1 = b2_warp_sum(s1) / (float) d.A;
        s2 = b2_warp_sum(s2) / (float) d.A;
      }
#pragma unroll
      for (int u = 0; u < 2; ++u) {
        const int c = lane + 32 * u;
        if (c < d.A) {
          const float gz = gamma ? rs * ((__fmul_rn(gy[u], __ldg(gamma + c)) - s1) - xh[u] * s2) : gy[u];
          Os[i * d.AP + c] = gz;
          const float t[1] = {gz};
          if (res_mode == 2) {
            dP[row * d.NP + 3 * d.A + c] = gz;
            if (dp_aux) rk_store_aux<1>(dp_aux, aux_dtype, row * ld_aux + 3 * d.A + c, t);
          } else if (res_mode == 1) {
            gres[row * d.A + c] = gz;
          }
        }
      }
    }
    __syncthreads();
    // per head: A' and dS into shared, then dQ, dK, dV
    for (int h = 0; h < d.H; ++h) {
      const int c0 = h * d.dh;
      for (int i = warp; i < d.F; i += AI_WARPS) {
        const int64_t si = (b * d.H + h) * d.F + i;
        const float m = __ldg(stat_max + si), l = __ldg(stat_sum + si);
        float a[2], da[2], rsum = 0.f;
#pragma unroll
        for (int u = 0; u < 2; ++u) {
          const int j = lane + 32 * u;
          a[u] = da[u] = 0.f;
          if (j < d.F) {
            a[u] = expf(ai_score(Qs, Ks, d, i, j, c0, scale) - m) / l;
            const float* go = Os + i * d.AP + c0;
            const float* v = Vs + j * d.AP + c0;
            float t = 0.f;
            for (int k = 0; k < d.dh; ++k) t += go[k] * v[k];
            float ad = a[u];
            if (drop_rng) {
              const bool keep = ai_keep(seed, off, b, h, i, j, d, drop_thresh);
              ad = keep ? ad * drop_scale : 0.f;
              t = keep ? t * drop_scale : 0.f;
            }
            Ps[i * d.FP + j] = ad;
            da[u] = t;
            rsum += a[u] * t;
          }
        }
        rsum = b2_warp_sum(rsum);
#pragma unroll
        for (int u = 0; u < 2; ++u) {
          const int j = lane + 32 * u;
          if (j < d.F) {
            const float ds = a[u] * (da[u] - rsum);
            Ss[i * d.FP + j] = scale != 0.f ? ds / scale : ds;
          }
        }
      }
      __syncthreads();
      for (int t = threadIdx.x; t < d.F * d.dh; t += blockDim.x) {
        const int r = t / d.dh, c = c0 + t % d.dh;
        float dq = 0.f, dk = 0.f, dv = 0.f;
        for (int j = 0; j < d.F; ++j) {
          dq += Ss[r * d.FP + j] * Ks[j * d.AP + c];
          dk += Ss[j * d.FP + r] * Qs[j * d.AP + c];
          dv += Ps[j * d.FP + r] * Os[j * d.AP + c];
        }
        const int64_t row = b * d.F + r;
        float* dr = dP + row * d.NP;
        dr[c] = dq;
        dr[d.A + c] = dk;
        dr[2 * d.A + c] = dv;
        if (dp_aux) {
          const float vq[1] = {dq}, vk[1] = {dk}, vv[1] = {dv};
          rk_store_aux<1>(dp_aux, aux_dtype, row * ld_aux + c, vq);
          rk_store_aux<1>(dp_aux, aux_dtype, row * ld_aux + d.A + c, vk);
          rk_store_aux<1>(dp_aux, aux_dtype, row * ld_aux + 2 * d.A + c, vv);
        }
      }
      __syncthreads();
    }
  }
  b2_pdl_trigger();
  if (!affine) return;
#pragma unroll
  for (int u = 0; u < 2; ++u) {
    const int c = lane + 32 * u;
    if (c < d.A) {
      if (acc_g[u] != 0.f) atomicAdd(&sg[c], acc_g[u]);
      if (acc_b[u] != 0.f) atomicAdd(&sb[c], acc_b[u]);
    }
  }
  __syncthreads();
  for (int c = threadIdx.x; c < d.A; c += blockDim.x) {
    if (sg[c] != 0.f) b2_red_add(dgamma + c, sg[c]);
    if (sb[c] != 0.f) b2_red_add(dbeta + c, sb[c]);
  }
}

// Wp (parts A, d_in) = [W_q; W_k; W_v (; W_res)]  ("=")
__global__ void __launch_bounds__(256)
ai_pack_kernel(const float* __restrict__ Wq, const float* __restrict__ Wk, const float* __restrict__ Wv,
               const float* __restrict__ Wr, int64_t n, int parts, float* __restrict__ Wp) {
  b2_pdl_wait();
  for (int64_t t = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; t < parts * n;
       t += (int64_t) gridDim.x * blockDim.x) {
    const int p = (int) (t / n);
    const int64_t e = t - p * n;
    const float* src = p == 0 ? Wq : p == 1 ? Wk : p == 2 ? Wv : Wr;
    Wp[t] = __ldg(src + e);
  }
  b2_pdl_trigger();
}

// gW_q, gW_k, gW_v (, gW_res) = the parts of dWp  ("=")
__global__ void __launch_bounds__(256)
ai_unpack_kernel(const float* __restrict__ dWp, int64_t n, int parts, float* __restrict__ gq, float* __restrict__ gk,
                 float* __restrict__ gv, float* __restrict__ gr) {
  b2_pdl_wait();
  for (int64_t t = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; t < parts * n;
       t += (int64_t) gridDim.x * blockDim.x) {
    const int p = (int) (t / n);
    const int64_t e = t - p * n;
    float* dst = p == 0 ? gq : p == 1 ? gk : p == 2 ? gv : gr;
    dst[e] = __ldg(dWp + t);
  }
  b2_pdl_trigger();
}

// ---------------------------------------------------------------------------------
// Host side
// ---------------------------------------------------------------------------------
static int ai_check(int64_t batch, int fields, int din, int A, int heads, int res_mode) {
  B2_REQUIRE(fields >= 1 && fields <= B2_AUTOINT_MAX_FIELDS, "fields %d outside [1, %d]", fields,
             B2_AUTOINT_MAX_FIELDS);
  B2_REQUIRE(A >= 1 && A <= B2_AUTOINT_MAX_DIM, "attention_dim %d outside [1, %d]", A, B2_AUTOINT_MAX_DIM);
  B2_REQUIRE(heads >= 1 && A % heads == 0, "heads %d do not divide attention_dim %d", heads, A);
  B2_REQUIRE(din >= 1, "input_dim %d < 1", din);
  B2_REQUIRE(res_mode >= 0 && res_mode <= 2, "res_mode %d is not 0, 1 or 2", res_mode);
  B2_REQUIRE(res_mode != 1 || din == A, "an identity residual needs input_dim %d == attention_dim %d", din, A);
  B2_REQUIRE(batch >= 0, "negative batch");
  B2_REQUIRE(batch <= (((int64_t) 1 << 31) - 1) / ((int64_t) fields * 4 * A), "batch * fields * 4 attention_dim >= 2^31");
  return B2_OK;
}

static ai_dims ai_make_dims(int fields, int A, int heads, int res_mode) {
  ai_dims d;
  d.F = fields;
  d.A = A;
  d.H = heads;
  d.dh = A / heads;
  d.NP = (res_mode == 2 ? 4 : 3) * A;
  d.AP = A + 1;
  d.FP = fields + 1;
  return d;
}

static size_t ai_smem(const ai_dims& d, bool bwd) {
  return (size_t) (4 * d.F * d.AP + (bwd ? 2 : 1) * d.F * d.FP) * sizeof(float);
}

// One CTA per sample, as many per SM as the shared memory allows (at most 8), the batch in a grid stride.
static int ai_grid(int64_t batch, size_t smem) {
  int64_t per_sm = (int64_t) (200 * 1024 / (smem + 1024));
  per_sm = per_sm < 1 ? 1 : (per_sm > 8 ? 8 : per_sm);
  const int64_t cap = (int64_t) B2_NUM_SMS * per_sm;
  return (int) (batch < cap ? batch : cap);
}

// The dynamic shared memory a launch asks for is capped at 48 KiB minus the kernel's static shared memory unless the
// function opts in to more (the backward's static part makes that bite below a 48 KiB dynamic size): the attribute
// is set on every launch, a host call that enqueues nothing.
template <typename K>
static int ai_smem_optin(K kernel, size_t smem) {
  cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) smem);
  if (e != cudaSuccess) return b2_fail(B2_E_CUDA, "autoint: shared memory opt-in failed: %s", cudaGetErrorString(e));
  return B2_OK;
}

extern "C" B2_API int b2_autoint_pack(const float* Wq, const float* Wk, const float* Wv, const float* Wres, int din,
                                      int A, float* Wp, void* stream) {
  B2_REQUIRE(Wq && Wk && Wv && Wp, "NULL pointer");
  B2_REQUIRE(din >= 1 && A >= 1 && A <= B2_AUTOINT_MAX_DIM, "input_dim %d / attention_dim %d out of range", din, A);
  const int parts = Wres ? 4 : 3;
  const int64_t n = (int64_t) A * din;
  const int64_t blocks = b2_ceil_div(parts * n, 256), cap = (int64_t) B2_NUM_SMS * 8;
  B2_LAUNCH(ai_pack_kernel, (int) (blocks > cap ? cap : blocks), 256, 0, (cudaStream_t) stream, Wq, Wk, Wv, Wres, n,
            parts, Wp);
  B2_CUDA_LAUNCH_CHECK("b2_autoint_pack");
  return B2_OK;
}

extern "C" B2_API int b2_autoint_fwd(const float* P, const float* X, int64_t batch, int fields, int din, int A,
                                     int heads, int res_mode, float scale, const float* gamma, const float* beta,
                                     float eps, const int64_t* drop_rng, int64_t drop_layer, uint32_t drop_thresh,
                                     float drop_scale, float* out, void* out_aux, int aux_dtype, int64_t ld_aux,
                                     float* stat_max, float* stat_sum, float* ln_mean, float* ln_rstd, void* stream) {
  B2_REQUIRE(P && out && stat_max && stat_sum, "NULL pointer");
  if (int rc = ai_check(batch, fields, din, A, heads, res_mode)) return rc;
  B2_REQUIRE(res_mode != 1 || X, "an identity residual needs X");
  B2_REQUIRE((gamma == nullptr) == (beta == nullptr), "gamma and beta: both or neither");
  B2_REQUIRE(gamma == nullptr || (ln_mean && ln_rstd), "LayerNorm needs ln_mean and ln_rstd");
  B2_REQUIRE(scale >= 0.f, "negative scale");
  if (int rc = rk_check_aux(out_aux, aux_dtype, ld_aux, A)) return rc;
  if (batch == 0) return B2_OK;
  const ai_dims d = ai_make_dims(fields, A, heads, res_mode);
  const size_t smem = ai_smem(d, false);
  const int grid = ai_grid(batch, smem);
  if (A % 4 == 0 && rk_al16(P)) {
    if (int rc = ai_smem_optin(ai_fwd_kernel<4>, smem)) return rc;
    B2_LAUNCH(ai_fwd_kernel<4>, grid, AI_THREADS, smem, (cudaStream_t) stream, P, X, batch, d, res_mode, scale, gamma,
              beta, eps, drop_rng, drop_layer, drop_thresh, drop_scale, out, out_aux, aux_dtype, ld_aux, stat_max,
              stat_sum, ln_mean, ln_rstd);
  } else {
    if (int rc = ai_smem_optin(ai_fwd_kernel<1>, smem)) return rc;
    B2_LAUNCH(ai_fwd_kernel<1>, grid, AI_THREADS, smem, (cudaStream_t) stream, P, X, batch, d, res_mode, scale, gamma,
              beta, eps, drop_rng, drop_layer, drop_thresh, drop_scale, out, out_aux, aux_dtype, ld_aux, stat_max,
              stat_sum, ln_mean, ln_rstd);
  }
  B2_CUDA_LAUNCH_CHECK("b2_autoint_fwd");
  return B2_OK;
}

extern "C" B2_API int b2_autoint_bwd(const float* P, const float* X, const float* out, const float* g,
                                     const float* stat_max, const float* stat_sum, const float* ln_mean,
                                     const float* ln_rstd, int64_t batch, int fields, int din, int A, int heads,
                                     int res_mode, float scale, const float* gamma, const int64_t* drop_rng,
                                     int64_t drop_layer, uint32_t drop_thresh, float drop_scale, float* dP,
                                     void* dp_aux, int aux_dtype, int64_t ld_aux, float* gres, float* dgamma,
                                     float* dbeta, void* stream) {
  B2_REQUIRE(P && out && g && stat_max && stat_sum && dP, "NULL pointer");
  if (int rc = ai_check(batch, fields, din, A, heads, res_mode)) return rc;
  B2_REQUIRE(res_mode != 1 || (X && gres), "an identity residual needs X and gres");
  B2_REQUIRE(gamma == nullptr || (ln_mean && ln_rstd && dgamma && dbeta),
             "LayerNorm needs ln_mean, ln_rstd, dgamma and dbeta");
  B2_REQUIRE(scale >= 0.f, "negative scale");
  if (int rc = rk_check_aux(dp_aux, aux_dtype, ld_aux, (res_mode == 2 ? 4 : 3) * A)) return rc;
  if (batch == 0) return B2_OK;
  const ai_dims d = ai_make_dims(fields, A, heads, res_mode);
  const size_t smem = ai_smem(d, true);
  const int grid = ai_grid(batch, smem + 2 * B2_AUTOINT_MAX_DIM * sizeof(float));
  if (A % 4 == 0 && rk_al16(P)) {
    if (int rc = ai_smem_optin(ai_bwd_kernel<4>, smem)) return rc;
    B2_LAUNCH(ai_bwd_kernel<4>, grid, AI_THREADS, smem, (cudaStream_t) stream, P, X, out, g, stat_max, stat_sum,
              ln_mean, ln_rstd, batch, d, res_mode, scale, gamma, drop_rng, drop_layer, drop_thresh, drop_scale, dP,
              dp_aux, aux_dtype, ld_aux, gres, dgamma, dbeta);
  } else {
    if (int rc = ai_smem_optin(ai_bwd_kernel<1>, smem)) return rc;
    B2_LAUNCH(ai_bwd_kernel<1>, grid, AI_THREADS, smem, (cudaStream_t) stream, P, X, out, g, stat_max, stat_sum,
              ln_mean, ln_rstd, batch, d, res_mode, scale, gamma, drop_rng, drop_layer, drop_thresh, drop_scale, dP,
              dp_aux, aux_dtype, ld_aux, gres, dgamma, dbeta);
  }
  B2_CUDA_LAUNCH_CHECK("b2_autoint_bwd");
  return B2_OK;
}

extern "C" B2_API int b2_autoint_unpack(const float* dWp, int din, int A, float* gWq, float* gWk, float* gWv,
                                        float* gWres, void* stream) {
  B2_REQUIRE(dWp && gWq && gWk && gWv, "NULL pointer");
  B2_REQUIRE(din >= 1 && A >= 1 && A <= B2_AUTOINT_MAX_DIM, "input_dim %d / attention_dim %d out of range", din, A);
  const int parts = gWres ? 4 : 3;
  const int64_t n = (int64_t) A * din;
  const int64_t blocks = b2_ceil_div(parts * n, 256), cap = (int64_t) B2_NUM_SMS * 8;
  B2_LAUNCH(ai_unpack_kernel, (int) (blocks > cap ? cap : blocks), 256, 0, (cudaStream_t) stream, dWp, n, parts, gWq,
            gWk, gWv, gWres);
  B2_CUDA_LAUNCH_CHECK("b2_autoint_unpack");
  return B2_OK;
}

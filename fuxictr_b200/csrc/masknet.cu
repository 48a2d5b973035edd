// masknet.cu — MaskNet's row kernels (model_zoo/MaskNet/src/MaskNet.py), sm_90a.
//
// Two entry points share one LayerNorm row kernel, forward and backward:
//   - the per-field embedding LayerNorm: F separate nn.LayerNorm(D) over (B, F, D), one launch each way for all
//     F fields (field f is blockIdx.y; its gamma and beta sit at gamma + f * pstride, beta + f * pstride);
//   - one MaskBlock's tail, out = dropout(act(LN(z))) with z = (V_mask * v_in) W^T the hidden GEMM's output, written
//     at the caller's row pitch (a slice of ParallelMaskNet's concatenation) with its GEMM-operand copy.
// Layouts: include/fuxictr_b200.h "MaskNet".
//
// A row of n values belongs to a group of L lanes (a power of two, L <= 32, within one warp); lane l owns the chunks
// k L + l (k < NPL) of 4 columns, held in registers (one float4 access each on the float4 path, element accesses on
// the scalar one; the dropout mask takes one Philox call per chunk on both).  Tiers: NPL 2 (n <= 256) and 8
// (n <= B2_MASKNET_MAX_WIDTH).  The mean is
// reduced first, then the variance from the centred values in registers (not E[x^2] - E[x]^2), both with group
// shuffles.  A thread keeps one field and one column set for the whole launch, so the gamma / beta gradients are
// summed per thread (NPL <= MN_REG_NPL: in registers; wider tiers: shared atomics per row), then per CTA in shared
// memory, and added with one float atomic per column and CTA.
#include "row_common.cuh"
#include "philox.cuh"

#define MN_REG_NPL 2   // tiers up to this many chunks per lane sum the affine gradients in registers

__device__ __forceinline__ float mn_sigmoid(float z) { return 1.f / (1.f + expf(-z)); }

__device__ __forceinline__ float mn_group_sum(float v, int L, unsigned mask) {
  for (int o = L >> 1; o > 0; o >>= 1) v += __shfl_xor_sync(mask, v, o);
  return v;
}

__device__ __forceinline__ unsigned mn_group_mask(int L) {
  if (L == 32) return 0xffffffffu;
  const int base = (threadIdx.x & 31) / L * L;
  return ((1u << L) - 1u) << base;
}

// A chunk is 4 consecutive columns c .. c + 3 of a row of n.  VEC: n % 4 == 0 and 16-byte aligned rows, one float4
// access; else element by element, the columns past n read as 0 and never written.
template <bool VEC>
__device__ __forceinline__ void mn_load(const float* p, int c, int n, float (&v)[4]) {
  if constexpr (VEC) {
    rk_load<4>(p + c, v);
  } else {
#pragma unroll
    for (int e = 0; e < 4; ++e) v[e] = c + e < n ? __ldg(p + c + e) : 0.f;
  }
}

template <bool VEC>
__device__ __forceinline__ void mn_store(float* p, int c, int n, const float (&v)[4]) {
  if constexpr (VEC) {
    rk_store<4>(p + c, v);
  } else {
#pragma unroll
    for (int e = 0; e < 4; ++e)
      if (c + e < n) p[c + e] = v[e];
  }
}

// the GEMM-operand copy of the chunk at aux + row_off + c (rk_store_aux)
template <bool VEC>
__device__ __forceinline__ void mn_store_aux(void* aux, int aux_dtype, int64_t row_off, int c, int n,
                                             const float (&v)[4]) {
  if constexpr (VEC) {
    rk_store_aux<4>(aux, aux_dtype, row_off + c, v);
  } else {
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      if (c + e < n) {
        const float t[1] = {v[e]};
        rk_store_aux<1>(aux, aux_dtype, row_off + c + e, t);
      }
    }
  }
}

// out = dropout(act(LN(x) or x)), row (b, f) of x at x + b ld_x + f n, of out at out + b ld_out + f n
template <bool VEC, int NPL>
__global__ void __launch_bounds__(RK_THREADS, 1)
mn_ln_fwd_kernel(const float* __restrict__ x, int64_t ld_x, int64_t batch, int F, int n, int L,
                 const float* __restrict__ gamma, const float* __restrict__ beta, int64_t pstride, float eps, int act,
                 const int64_t* __restrict__ drop_rng, int64_t drop_layer, uint32_t drop_thresh, float drop_scale,
                 float* __restrict__ out, int64_t ld_out, void* out_aux, int aux_dtype, int64_t ld_aux,
                 float* __restrict__ mean_out, float* __restrict__ rstd_out) {
  const int lane = threadIdx.x % L, grp = threadIdx.x / L, G = blockDim.x / L;
  const int f = blockIdx.y;
  const unsigned gmask = mn_group_mask(L);
  const bool ln = gamma != nullptr;
  if (ln) {
    gamma += f * pstride;
    beta += f * pstride;
  }
  b2_pdl_wait();
  uint64_t seed = 0, off = 0;
  if (drop_rng) {
    seed = (uint64_t) drop_rng[0];
    off = (uint64_t) drop_rng[1] + (uint64_t) drop_layer;
  }
  for (int64_t b = (int64_t) blockIdx.x * G + grp; b < batch; b += (int64_t) gridDim.x * G) {
    const float* xr = x + b * ld_x + (int64_t) f * n;
    float v[NPL][4];
    float s = 0.f;
#pragma unroll
    for (int k = 0; k < NPL; ++k) {
      const int c = (k * L + lane) * 4;
      if (c < n) {
        mn_load<VEC>(xr, c, n, v[k]);
#pragma unroll
        for (int e = 0; e < 4; ++e) s += v[k][e];
      }
    }
    float mu = 0.f, rs = 1.f;
    if (ln) {
      mu = mn_group_sum(s, L, gmask) / (float) n;
      float q = 0.f;
#pragma unroll
      for (int k = 0; k < NPL; ++k) {
        const int c = (k * L + lane) * 4;
        if (c < n) {
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const float d = v[k][e] - mu;
            if (VEC || c + e < n) q += d * d;
          }
        }
      }
      rs = 1.f / sqrtf(mn_group_sum(q, L, gmask) / (float) n + eps);
    }
#pragma unroll
    for (int k = 0; k < NPL; ++k) {
      const int c = (k * L + lane) * 4;
      if (c < n) {
        float y[4];
        if (ln) {
          float ga[4], be[4];
          mn_load<VEC>(gamma, c, n, ga);
          mn_load<VEC>(beta, c, n, be);
#pragma unroll
          for (int e = 0; e < 4; ++e) y[e] = (v[k][e] - mu) * rs * ga[e] + be[e];
        } else {
#pragma unroll
          for (int e = 0; e < 4; ++e) y[e] = v[k][e];
        }
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          if (act == B2_ACT_RELU) y[e] = y[e] > 0.f ? y[e] : 0.f;
          else if (act == B2_ACT_SIGMOID) y[e] = mn_sigmoid(y[e]);
        }
        if (drop_rng) {
          const uint32_t keep = b2_drop_keep4(seed, off, (uint64_t) b * n + c, n - c < 4 ? n - c : 4, drop_thresh);
#pragma unroll
          for (int e = 0; e < 4; ++e) y[e] = (keep >> e) & 1u ? y[e] * drop_scale : 0.f;
        }
        mn_store<VEC>(out + b * ld_out + (int64_t) f * n, c, n, y);
        if (out_aux) mn_store_aux<VEC>(out_aux, aux_dtype, b * ld_aux + (int64_t) f * n, c, n, y);
      }
    }
    if (ln && mean_out && lane == 0) {
      mean_out[b * F + f] = mu;
      rstd_out[b * F + f] = rs;
    }
  }
  b2_pdl_trigger();
}

// From the output gradient g (row (b, f) at g + b ld_g + f n): gz = act'(y) * keep * scale * g with y the LN output the
// forward had before dropout (recomputed from x, mean, rstd), then the LN backward
//   dx = rstd (gz gamma - mean(gz gamma) - xh mean(gz gamma xh)),  xh = (x - mean) rstd
// dx "=" (or "+=" with accumulate) at dx + b ld_dx + f n, with its GEMM-operand copy; dgamma += sum_b gz xh,
// dbeta += sum_b gz (per field, at the parameters' stride).  Without LN (gamma NULL) dx = gz.
template <bool VEC, int NPL>
__global__ void __launch_bounds__(RK_THREADS, 1)
mn_ln_bwd_kernel(const float* __restrict__ x, int64_t ld_x, const float* __restrict__ mean,
                 const float* __restrict__ rstd, int64_t batch, int F, int n, int L, const float* __restrict__ gamma,
                 const float* __restrict__ beta, int64_t pstride, int act, const int64_t* __restrict__ drop_rng,
                 int64_t drop_layer, uint32_t drop_thresh, float drop_scale, const float* __restrict__ g,
                 int64_t ld_g, float* __restrict__ dx, int64_t ld_dx, int accumulate, void* dx_aux, int aux_dtype,
                 int64_t ld_aux, float* __restrict__ dgamma, float* __restrict__ dbeta) {
  __shared__ float sg[B2_MASKNET_MAX_WIDTH], sb[B2_MASKNET_MAX_WIDTH];
  constexpr bool REG = NPL <= MN_REG_NPL;
  const int lane = threadIdx.x % L, grp = threadIdx.x / L, G = blockDim.x / L;
  const int f = blockIdx.y;
  const unsigned gmask = mn_group_mask(L);
  const bool ln = gamma != nullptr, want_affine = ln && dgamma != nullptr;
  if (ln) {
    gamma += f * pstride;
    beta += f * pstride;
  }
  if (want_affine) {
    for (int c = threadIdx.x; c < n; c += blockDim.x) sg[c] = sb[c] = 0.f;
    __syncthreads();
  }
  float acc_g[REG ? NPL : 1][4], acc_b[REG ? NPL : 1][4];
#pragma unroll
  for (int k = 0; k < (REG ? NPL : 1); ++k)
#pragma unroll
    for (int e = 0; e < 4; ++e) acc_g[k][e] = acc_b[k][e] = 0.f;
  b2_pdl_wait();
  uint64_t seed = 0, off = 0;
  if (drop_rng) {
    seed = (uint64_t) drop_rng[0];
    off = (uint64_t) drop_rng[1] + (uint64_t) drop_layer;
  }
  for (int64_t b = (int64_t) blockIdx.x * G + grp; b < batch; b += (int64_t) gridDim.x * G) {
    const float* xr = x + b * ld_x + (int64_t) f * n;
    const float* gr = g + b * ld_g + (int64_t) f * n;
    float mu = 0.f, rs = 1.f;
    if (ln) {
      mu = __ldg(mean + b * F + f);
      rs = __ldg(rstd + b * F + f);
    }
    // the chunk's xh and gz (and gamma): kept in registers on the register tiers, recomputed in the second pass on
    // the wide ones (whose rows then come from L1 again) so that nothing spills
    auto chunk = [&](int c, float (&xh_)[4], float (&gz_)[4], float (&ga)[4]) {
      float gg[4], be[4];
      mn_load<VEC>(xr, c, n, xh_);
      mn_load<VEC>(gr, c, n, gg);
      if (ln) {
        mn_load<VEC>(gamma, c, n, ga);
        mn_load<VEC>(beta, c, n, be);
      }
      uint32_t keep = 0xfu;
      if (drop_rng) keep = b2_drop_keep4(seed, off, (uint64_t) b * n + c, n - c < 4 ? n - c : 4, drop_thresh);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        float y = xh_[e];
        if (ln) {
          xh_[e] = (xh_[e] - mu) * rs;
          y = xh_[e] * ga[e] + be[e];
        }
        float t = gg[e];
        if (drop_rng) t = (keep >> e) & 1u ? t * drop_scale : 0.f;
        if (act == B2_ACT_RELU) {
          t = y > 0.f ? t : 0.f;
        } else if (act == B2_ACT_SIGMOID) {
          const float sy = mn_sigmoid(y);
          t = t * (1.f - sy) * sy;
        }
        gz_[e] = t;
      }
    };
    float xh[REG ? NPL : 1][4], gz[REG ? NPL : 1][4];
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int k = 0; k < NPL; ++k) {
      const int c = (k * L + lane) * 4;
      if (c < n) {
        float ga[4], h[4], t[4];
        chunk(c, h, t, ga);
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          if (REG) {
            xh[REG ? k : 0][e] = h[e];
            gz[REG ? k : 0][e] = t[e];
          }
          if (ln) {
            const float d = __fmul_rn(t[e], ga[e]);    // rounded as in the second pass: a row of one gives dx = 0
            s1 += d;
            s2 += d * h[e];
            if (want_affine) {
              if constexpr (REG) {
                acc_g[k][e] += t[e] * h[e];
                acc_b[k][e] += t[e];
              } else if (VEC || c + e < n) {
                atomicAdd(&sg[c + e], t[e] * h[e]);
                atomicAdd(&sb[c + e], t[e]);
              }
            }
          }
        }
      }
    }
    if (ln) {
      s1 = mn_group_sum(s1, L, gmask) / (float) n;
      s2 = mn_group_sum(s2, L, gmask) / (float) n;
    }
#pragma unroll
    for (int k = 0; k < NPL; ++k) {
      const int c = (k * L + lane) * 4;
      if (c < n) {
        float o[4], ga[4], h[4], t[4];
        if constexpr (REG) {
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            h[e] = xh[REG ? k : 0][e];
            t[e] = gz[REG ? k : 0][e];
          }
          if (ln) mn_load<VEC>(gamma, c, n, ga);
        } else {
          chunk(c, h, t, ga);
        }
#pragma unroll
        for (int e = 0; e < 4; ++e) o[e] = ln ? rs * ((__fmul_rn(t[e], ga[e]) - s1) - h[e] * s2) : t[e];
        float* dr = dx + b * ld_dx + (int64_t) f * n;
        if (accumulate) {       // dx is not read through the read-only path: the caller may have just written it
          float prev[4];
          if constexpr (VEC) {
            const float4 q = *reinterpret_cast<const float4*>(dr + c);
            prev[0] = q.x; prev[1] = q.y; prev[2] = q.z; prev[3] = q.w;
          } else {
#pragma unroll
            for (int e = 0; e < 4; ++e) prev[e] = c + e < n ? dr[c + e] : 0.f;
          }
#pragma unroll
          for (int e = 0; e < 4; ++e) o[e] += prev[e];
        }
        mn_store<VEC>(dr, c, n, o);
        if (dx_aux) mn_store_aux<VEC>(dx_aux, aux_dtype, b * ld_aux + (int64_t) f * n, c, n, o);
      }
    }
  }
  b2_pdl_trigger();
  if (!want_affine) return;
  if constexpr (REG) {
#pragma unroll
    for (int k = 0; k < NPL; ++k) {
      const int c = (k * L + lane) * 4;
      if (c < n) {
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          if (acc_g[k][e] != 0.f) atomicAdd(&sg[c + e], acc_g[k][e]);
          if (acc_b[k][e] != 0.f) atomicAdd(&sb[c + e], acc_b[k][e]);
        }
      }
    }
  }
  __syncthreads();
  float* dg = dgamma + f * pstride;
  float* db = dbeta + f * pstride;
  for (int c = threadIdx.x; c < n; c += blockDim.x) {
    if (sg[c] != 0.f) b2_red_add(dg + c, sg[c]);
    if (sb[c] != 0.f) b2_red_add(db + c, sb[c]);
  }
}

// out = a * b ("=" or "+=")
template <int VW>
__global__ void __launch_bounds__(256)
mn_mul_kernel(const float* __restrict__ a, const float* __restrict__ b, int64_t nv, float* __restrict__ out,
              int accumulate) {
  b2_pdl_wait();
  for (int64_t t = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; t < nv; t += (int64_t) gridDim.x * blockDim.x) {
    float x[VW], y[VW], o[VW];
    rk_load<VW>(a + t * VW, x);
    rk_load<VW>(b + t * VW, y);
#pragma unroll
    for (int e = 0; e < VW; ++e) o[e] = x[e] * y[e];
    if (accumulate) {
      float p[VW];
      if constexpr (VW == 4) {
        const float4 q = *reinterpret_cast<const float4*>(out + t * VW);
        p[0] = q.x; p[1] = q.y; p[2] = q.z; p[3] = q.w;
      } else {
        p[0] = out[t];
      }
#pragma unroll
      for (int e = 0; e < VW; ++e) o[e] += p[e];
    }
    rk_store<VW>(out + t * VW, o);
  }
  b2_pdl_trigger();
}

// ---------------------------------------------------------------------------------
// Host side
// ---------------------------------------------------------------------------------
// Launch plan of a width-n row: the tier NPL (chunks per lane) and the group width L.
struct mn_plan {
  bool vec;
  int npl, L, groups;
};

static mn_plan mn_make_plan(int n, bool vec) {
  mn_plan p;
  p.vec = vec;
  const int chunks = (n + 3) / 4;
  p.npl = chunks <= 32 * MN_REG_NPL ? MN_REG_NPL : 8;
  int L = 1;
  while (L * p.npl < chunks) L <<= 1;
  p.L = L;
  p.groups = RK_THREADS / L;
  return p;
}

static dim3 mn_grid(int64_t batch, int F, int groups, int per_sm) {
  int64_t cap = (int64_t) B2_NUM_SMS * per_sm / F, gx = b2_ceil_div(batch, groups);
  cap = cap < 1 ? 1 : cap;
  gx = gx < 1 ? 1 : (gx > cap ? cap : gx);
  return dim3((unsigned) gx, (unsigned) F);
}

static int mn_check(int64_t batch, int F, int n) {
  B2_REQUIRE(n >= 1 && n <= B2_MASKNET_MAX_WIDTH, "row width %d outside [1, %d]", n, B2_MASKNET_MAX_WIDTH);
  B2_REQUIRE(F >= 1 && F <= 65535, "fields %d outside [1, 65535]", F);
  B2_REQUIRE(batch >= 0, "negative batch");
  return B2_OK;
}

#define MN_DISPATCH(KERNEL, plan, grid, stream, ...)                                                      \
  do {                                                                                                    \
    if ((plan).vec) {                                                                                     \
      if ((plan).npl == MN_REG_NPL) B2_LAUNCH((KERNEL<true, MN_REG_NPL>), grid, RK_THREADS, 0, stream, __VA_ARGS__); \
      else B2_LAUNCH((KERNEL<true, 8>), grid, RK_THREADS, 0, stream, __VA_ARGS__);                        \
    } else {                                                                                              \
      if ((plan).npl == MN_REG_NPL) B2_LAUNCH((KERNEL<false, MN_REG_NPL>), grid, RK_THREADS, 0, stream, __VA_ARGS__); \
      else B2_LAUNCH((KERNEL<false, 8>), grid, RK_THREADS, 0, stream, __VA_ARGS__);                       \
    }                                                                                                     \
  } while (0)

extern "C" B2_API int b2_field_ln_fwd(const float* x, int64_t batch, int fields, int dim, const float* gamma,
                                      const float* beta, int64_t pstride, float eps, float* out, float* mean,
                                      float* rstd, void* stream) {
  B2_REQUIRE(x && gamma && beta && out && mean && rstd, "NULL pointer");
  if (int rc = mn_check(batch, fields, dim)) return rc;
  B2_REQUIRE(pstride >= 0 && (fields == 1 || pstride >= dim), "parameter stride %lld < dim %d",
             (long long) pstride, dim);
  B2_REQUIRE(batch * fields * (int64_t) dim < ((int64_t) 1 << 31), "batch * fields * dim >= 2^31");
  if (batch == 0) return B2_OK;
  const bool vec = dim % 4 == 0 && pstride % 4 == 0 && rk_al16(x) && rk_al16(out) && rk_al16(gamma) &&
                   rk_al16(beta);
  const mn_plan p = mn_make_plan(dim, vec);
  const dim3 grid = mn_grid(batch, fields, p.groups, 8);
  const int64_t ld = (int64_t) fields * dim;
  MN_DISPATCH(mn_ln_fwd_kernel, p, grid, (cudaStream_t) stream, x, ld, batch, fields, dim, p.L, gamma, beta, pstride,
              eps, (int) B2_ACT_NONE, (const int64_t*) nullptr, (int64_t) 0, 0u, 0.f, out, ld, (void*) nullptr, 0,
              (int64_t) 0, mean, rstd);
  B2_CUDA_LAUNCH_CHECK("b2_field_ln_fwd");
  return B2_OK;
}

extern "C" B2_API int b2_field_ln_bwd(const float* x, const float* mean, const float* rstd, const float* g,
                                      int64_t batch, int fields, int dim, const float* gamma, int64_t pstride,
                                      float* dx, int accumulate, float* dgamma, float* dbeta, void* stream) {
  B2_REQUIRE(x && mean && rstd && g && gamma && dx && dgamma && dbeta, "NULL pointer");
  if (int rc = mn_check(batch, fields, dim)) return rc;
  B2_REQUIRE(pstride >= 0 && (fields == 1 || pstride >= dim), "parameter stride %lld < dim %d",
             (long long) pstride, dim);
  B2_REQUIRE(batch * fields * (int64_t) dim < ((int64_t) 1 << 31), "batch * fields * dim >= 2^31");
  if (batch == 0) return B2_OK;
  const bool vec = dim % 4 == 0 && pstride % 4 == 0 && rk_al16(x) && rk_al16(g) && rk_al16(dx) && rk_al16(gamma);
  const mn_plan p = mn_make_plan(dim, vec);
  const dim3 grid = mn_grid(batch, fields, p.groups, 4);
  const int64_t ld = (int64_t) fields * dim;
  // beta only enters the activation's backward, and the embedding LayerNorm has none: gamma stands in for it
  MN_DISPATCH(mn_ln_bwd_kernel, p, grid, (cudaStream_t) stream, x, ld, mean, rstd, batch, fields, dim, p.L, gamma,
              gamma, pstride, (int) B2_ACT_NONE, (const int64_t*) nullptr, (int64_t) 0, 0u, 0.f, g, ld, dx, ld,
              accumulate, (void*) nullptr, 0, (int64_t) 0, dgamma, dbeta);
  B2_CUDA_LAUNCH_CHECK("b2_field_ln_bwd");
  return B2_OK;
}

static int mn_check_act(int act) {
  B2_REQUIRE(act == B2_ACT_NONE || act == B2_ACT_RELU || act == B2_ACT_SIGMOID, "act %d is not a B2_ACT_* code",
             act);
  return B2_OK;
}

extern "C" B2_API int b2_mask_row_fwd(const float* z, int64_t batch, int n, const float* gamma, const float* beta,
                                      float eps, int act, const int64_t* drop_rng, int64_t drop_layer,
                                      uint32_t drop_thresh, float drop_scale, float* out, int64_t ld_out,
                                      void* out_aux, int aux_dtype, int64_t ld_aux, float* mean, float* rstd,
                                      void* stream) {
  B2_REQUIRE(z && out, "NULL pointer");
  B2_REQUIRE((gamma == nullptr) == (beta == nullptr), "gamma and beta: both or neither");
  B2_REQUIRE(gamma == nullptr || (mean && rstd), "LayerNorm needs mean and rstd");
  if (int rc = mn_check(batch, 1, n)) return rc;
  if (int rc = mn_check_act(act)) return rc;
  B2_REQUIRE(ld_out >= n, "ld_out %lld < width %d", (long long) ld_out, n);
  if (int rc = rk_check_aux(out_aux, aux_dtype, ld_aux, n)) return rc;
  B2_REQUIRE(batch * (ld_out > ld_aux ? ld_out : ld_aux) < ((int64_t) 1 << 31), "batch * row pitch >= 2^31");
  if (batch == 0) return B2_OK;
  const void* ptrs[] = {z, gamma, beta, out};
  const bool vec = rk_vec(n, ptrs, 4, out_aux, aux_dtype, ld_aux) && ld_out % 4 == 0;
  const mn_plan p = mn_make_plan(n, vec);
  const dim3 grid = mn_grid(batch, 1, p.groups, 8);
  MN_DISPATCH(mn_ln_fwd_kernel, p, grid, (cudaStream_t) stream, z, (int64_t) n, batch, 1, n, p.L, gamma, beta,
              (int64_t) 0, eps, act, drop_rng, drop_layer, drop_thresh, drop_scale, out, ld_out, out_aux, aux_dtype,
              ld_aux, mean, rstd);
  B2_CUDA_LAUNCH_CHECK("b2_mask_row_fwd");
  return B2_OK;
}

extern "C" B2_API int b2_mask_row_bwd(const float* z, const float* mean, const float* rstd, const float* gamma,
                                      const float* beta, int act, const int64_t* drop_rng, int64_t drop_layer,
                                      uint32_t drop_thresh, float drop_scale, const float* g, int64_t ld_g,
                                      int64_t batch, int n, float* dz, void* dz_aux, int aux_dtype, int64_t ld_aux,
                                      float* dgamma, float* dbeta, void* stream) {
  B2_REQUIRE(z && g && dz, "NULL pointer");
  B2_REQUIRE((gamma == nullptr) == (beta == nullptr), "gamma and beta: both or neither");
  B2_REQUIRE(gamma == nullptr || (mean && rstd && dgamma && dbeta), "LayerNorm needs mean, rstd, dgamma, dbeta");
  if (int rc = mn_check(batch, 1, n)) return rc;
  if (int rc = mn_check_act(act)) return rc;
  B2_REQUIRE(ld_g >= n, "ld_g %lld < width %d", (long long) ld_g, n);
  if (int rc = rk_check_aux(dz_aux, aux_dtype, ld_aux, n)) return rc;
  B2_REQUIRE(batch * (ld_g > ld_aux ? ld_g : ld_aux) < ((int64_t) 1 << 31), "batch * row pitch >= 2^31");
  if (batch == 0) return B2_OK;
  const void* ptrs[] = {z, gamma, beta, g, dz};
  const bool vec = rk_vec(n, ptrs, 5, dz_aux, aux_dtype, ld_aux) && ld_g % 4 == 0;
  const mn_plan p = mn_make_plan(n, vec);
  const dim3 grid = mn_grid(batch, 1, p.groups, 4);
  MN_DISPATCH(mn_ln_bwd_kernel, p, grid, (cudaStream_t) stream, z, (int64_t) n, mean, rstd, batch, 1, n, p.L, gamma,
              beta, (int64_t) 0, act, drop_rng, drop_layer, drop_thresh, drop_scale, g, ld_g, dz, (int64_t) n, 0,
              dz_aux, aux_dtype, ld_aux, dgamma, dbeta);
  B2_CUDA_LAUNCH_CHECK("b2_mask_row_bwd");
  return B2_OK;
}

extern "C" B2_API int b2_mask_mul(const float* a, const float* b, int64_t n, float* out, int accumulate,
                                  void* stream) {
  B2_REQUIRE(a && b && out, "NULL pointer");
  B2_REQUIRE(n >= 0, "negative size");
  if (n == 0) return B2_OK;
  const bool vec = n % 4 == 0 && rk_al16(a) && rk_al16(b) && rk_al16(out);
  const int64_t nv = vec ? n / 4 : n;
  const int64_t blocks = b2_ceil_div(nv, 256), cap = (int64_t) B2_NUM_SMS * 8;
  const int grid = (int) (blocks > cap ? cap : blocks);
  if (vec) B2_LAUNCH(mn_mul_kernel<4>, grid, 256, 0, (cudaStream_t) stream, a, b, nv, out, accumulate);
  else B2_LAUNCH(mn_mul_kernel<1>, grid, 256, 0, (cudaStream_t) stream, a, b, nv, out, accumulate);
  B2_CUDA_LAUNCH_CHECK("b2_mask_mul");
  return B2_OK;
}

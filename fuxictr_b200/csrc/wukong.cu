// wukong.cu — WuKong's layer (model_zoo/WuKong/src/WuKong.py, WuKongLayer), sm_90a.
//
// A layer keeps its input as X' (B D, fp): sample b's D rows, row d holding x[b, :, d] at a field pitch fp (F rounded
// up to 4, the pad columns zero), so that the linear-compression block, the residual projection and the factorization
// machine's projection are contractions over the row axis: one GEMM (the caller's) for the first two, the FM row
// kernel for the third.  This file holds that row kernel (FM product and its LayerNorm, forward and backward), the
// combine row kernel (concat + residual + LayerNorm(D), forward and backward) and the pack / unpack of the stacked
// field-axis weight.  Layouts and range: include/fuxictr_b200.h "WuKong".
//
// Both row kernels run one CTA of WK_THREADS threads per sample (grid stride over the batch) and stage the sample's
// tiles in shared memory, field-major at a pitch of D + 1 (fields) or k + 1 (rank), so that the field-axis and the
// rank-axis walks meet no bank conflict.  Every global access walks a sample's contiguous block in order.  LayerNorm
// is nn.LayerNorm's: the mean first, then the biased variance from the centred values, eps inside the square root.
// All arithmetic is fp32 on CUDA cores.
#include "row_common.cuh"

#define WK_THREADS 256
#define WK_WARPS (WK_THREADS / 32)

struct wk_fm_dims {
  int F, D, k, fp, DP, KP;      // fields, embedding dim, rank, X' field pitch, smem pitches
};

static inline int wk_pitch(int fields) { return (fields + 3) / 4 * 4; }

// Stage sample b's x into xs[f DP + d] from X (layout 0, (B, F, D)) or X' (layout 1, (B D, fp)).
template <int VW>
__device__ __forceinline__ void wk_stage_x(const float* __restrict__ x, int layout, int64_t b, const wk_fm_dims& d,
                                           float* xs) {
  if (layout == 0) {
    const float* xb = x + b * d.F * d.D;
    for (int t = threadIdx.x * VW; t < d.F * d.D; t += blockDim.x * VW) {
      float v[VW];
      rk_load<VW>(xb + t, v);
#pragma unroll
      for (int e = 0; e < VW; ++e) xs[((t + e) / d.D) * d.DP + (t + e) % d.D] = v[e];
    }
  } else {
    const float* xb = x + b * d.D * d.fp;
    for (int t = threadIdx.x * VW; t < d.D * d.fp; t += blockDim.x * VW) {
      float v[VW];
      rk_load<VW>(xb + t, v);
#pragma unroll
      for (int e = 0; e < VW; ++e) {
        const int f = (t + e) % d.fp;
        if (f < d.F) xs[f * d.DP + (t + e) / d.fp] = v[e];
      }
    }
  }
}

// Ps[d KP + c] = sum_f x[f][d] Y[f][c]  (P = x^T Y, D x k), then fms[f KP + c] = sum_d x[f][d] P[d][c]  (x P, F x k)
__device__ __forceinline__ void wk_fm_product(const float* xs, const float* Ys, const wk_fm_dims& d, float* Ps,
                                              float* fms) {
  for (int t = threadIdx.x; t < d.D * d.k; t += blockDim.x) {
    const int dd = t / d.k, c = t % d.k;
    float s = 0.f;
    for (int f = 0; f < d.F; ++f) s += xs[f * d.DP + dd] * Ys[f * d.KP + c];
    Ps[dd * d.KP + c] = s;
  }
  __syncthreads();
  for (int t = threadIdx.x; t < d.F * d.k; t += blockDim.x) {
    const int f = t / d.k, c = t % d.k;
    float s = 0.f;
    for (int dd = 0; dd < d.D; ++dd) s += xs[f * d.DP + dd] * Ps[dd * d.KP + c];
    fms[f * d.KP + c] = s;
  }
  __syncthreads();
}

// fm_out[b] = LN(flatten(x (x^T Y))) (+ its operand copy); layout 0 also writes X'_0 (+ its operand copy)
template <int VW>
__global__ void __launch_bounds__(WK_THREADS)
wk_fm_fwd_kernel(const float* __restrict__ x, int layout, int64_t batch, wk_fm_dims d, const float* __restrict__ Y,
                 const float* __restrict__ gamma, const float* __restrict__ beta, float eps, float* __restrict__ fm_out,
                 void* fm_aux, int aux_dtype, int64_t ld_aux, float* __restrict__ xp_out, void* xp_aux,
                 int64_t ld_xp_aux, float* __restrict__ ln_mean, float* __restrict__ ln_rstd) {
  extern __shared__ float smem[];
  __shared__ float red[32];
  float* Ys = smem;
  float* xs = Ys + d.F * d.KP;
  float* Ps = xs + d.F * d.DP;
  float* fms = Ps + d.D * d.KP;
  const int n = d.F * d.k;
  b2_pdl_wait();
  for (int t = threadIdx.x; t < n; t += blockDim.x) Ys[(t / d.k) * d.KP + t % d.k] = __ldg(Y + t);
  for (int64_t b = blockIdx.x; b < batch; b += gridDim.x) {
    wk_stage_x<VW>(x, layout, b, d, xs);
    __syncthreads();
    if (xp_out) {
      for (int t = threadIdx.x; t < d.D * d.fp; t += blockDim.x) {
        const int f = t % d.fp, dd = t / d.fp;
        const float v = f < d.F ? xs[f * d.DP + dd] : 0.f;
        xp_out[b * d.D * d.fp + t] = v;
        if (xp_aux) {
          const float w[1] = {v};
          rk_store_aux<1>(xp_aux, aux_dtype, (b * d.D + dd) * ld_xp_aux + f, w);
        }
      }
    }
    wk_fm_product(xs, Ys, d, Ps, fms);
    float s = 0.f;
    for (int t = threadIdx.x; t < n; t += blockDim.x) s += fms[(t / d.k) * d.KP + t % d.k];
    const float mu = b2_block_sum(s, red) / (float) n;
    float q = 0.f;
    for (int t = threadIdx.x; t < n; t += blockDim.x) {
      const float z = fms[(t / d.k) * d.KP + t % d.k] - mu;
      q += z * z;
    }
    const float rs = 1.f / sqrtf(b2_block_sum(q, red) / (float) n + eps);
    if (threadIdx.x == 0) {
      ln_mean[b] = mu;
      ln_rstd[b] = rs;
    }
    for (int t = threadIdx.x; t < n; t += blockDim.x) {
      const float y = (fms[(t / d.k) * d.KP + t % d.k] - mu) * rs * __ldg(gamma + t) + __ldg(beta + t);
      fm_out[b * n + t] = y;
      if (fm_aux) {
        const float w[1] = {y};
        rk_store_aux<1>(fm_aux, aux_dtype, b * ld_aux + t, w);
      }
    }
    __syncthreads();
  }
  b2_pdl_trigger();
}

// From g = d fm_out: the LayerNorm backward to dfm, dP = x^T dfm, dx = dfm P^T + Y dP^T ("=" or "+=", plus the
// transposed gxp in layout 0), dY += x dP, dgamma += g xhat, dbeta += g (per CTA, then one atomic per element and CTA)
template <int VW>
__global__ void __launch_bounds__(WK_THREADS)
wk_fm_bwd_kernel(const float* __restrict__ x, int layout, int64_t batch, wk_fm_dims d, const float* __restrict__ Y,
                 const float* __restrict__ gamma, const float* __restrict__ ln_mean, const float* __restrict__ ln_rstd,
                 const float* __restrict__ g, const float* __restrict__ gxp, float* __restrict__ gx, int accumulate,
                 float* __restrict__ gY, float* __restrict__ dgamma, float* __restrict__ dbeta) {
  extern __shared__ float smem[];
  __shared__ float red[32];
  const int n = d.F * d.k;
  float* Ys = smem;
  float* xs = Ys + d.F * d.KP;
  float* Ps = xs + d.F * d.DP;
  float* fms = Ps + d.D * d.KP;       // fm, then dfm
  float* dPs = fms + d.F * d.KP;
  float* accY = dPs + d.D * d.KP;
  float* accG = accY + n;
  float* accB = accG + n;
  b2_pdl_wait();
  for (int t = threadIdx.x; t < n; t += blockDim.x) {
    Ys[(t / d.k) * d.KP + t % d.k] = __ldg(Y + t);
    accY[t] = accG[t] = accB[t] = 0.f;
  }
  for (int64_t b = blockIdx.x; b < batch; b += gridDim.x) {
    wk_stage_x<VW>(x, layout, b, d, xs);
    __syncthreads();
    wk_fm_product(xs, Ys, d, Ps, fms);
    const float mu = __ldg(ln_mean + b), rs = __ldg(ln_rstd + b);
    const float* gb = g + b * n;
    float s1 = 0.f, s2 = 0.f;
    for (int t = threadIdx.x; t < n; t += blockDim.x) {
      const float xh = (fms[(t / d.k) * d.KP + t % d.k] - mu) * rs;
      const float gv = __ldg(gb + t);
      accG[t] += gv * xh;
      accB[t] += gv;
      const float gy = gv * __ldg(gamma + t);
      s1 += gy;
      s2 += gy * xh;
    }
    s1 = b2_block_sum(s1, red) / (float) n;
    s2 = b2_block_sum(s2, red) / (float) n;
    for (int t = threadIdx.x; t < n; t += blockDim.x) {
      float* p = fms + (t / d.k) * d.KP + t % d.k;
      const float xh = (*p - mu) * rs;
      *p = rs * ((__ldg(gb + t) * __ldg(gamma + t) - s1) - xh * s2);
    }
    __syncthreads();
    for (int t = threadIdx.x; t < d.D * d.k; t += blockDim.x) {
      const int dd = t / d.k, c = t % d.k;
      float s = 0.f;
      for (int f = 0; f < d.F; ++f) s += xs[f * d.DP + dd] * fms[f * d.KP + c];
      dPs[dd * d.KP + c] = s;
    }
    __syncthreads();
    if (layout == 0) {
      for (int t = threadIdx.x; t < d.F * d.D; t += blockDim.x) {
        const int f = t / d.D, dd = t % d.D;
        float v = 0.f;
        for (int c = 0; c < d.k; ++c) v += fms[f * d.KP + c] * Ps[dd * d.KP + c] + Ys[f * d.KP + c] * dPs[dd * d.KP + c];
        if (gxp) v += __ldg(gxp + (b * d.D + dd) * d.fp + f);
        float* o = gx + b * d.F * d.D + t;
        *o = accumulate ? *o + v : v;
      }
    } else {
      for (int t = threadIdx.x; t < d.D * d.fp; t += blockDim.x) {
        const int f = t % d.fp, dd = t / d.fp;
        float* o = gx + b * d.D * d.fp + t;
        if (f >= d.F) {
          if (!accumulate) *o = 0.f;
          continue;
        }
        float v = 0.f;
        for (int c = 0; c < d.k; ++c) v += fms[f * d.KP + c] * Ps[dd * d.KP + c] + Ys[f * d.KP + c] * dPs[dd * d.KP + c];
        *o = accumulate ? *o + v : v;
      }
    }
    for (int t = threadIdx.x; t < n; t += blockDim.x) {
      const int f = t / d.k, c = t % d.k;
      float s = 0.f;
      for (int dd = 0; dd < d.D; ++dd) s += xs[f * d.DP + dd] * dPs[dd * d.KP + c];
      accY[t] += s;
    }
    __syncthreads();
  }
  b2_pdl_trigger();
  for (int t = threadIdx.x; t < n; t += blockDim.x) {
    if (accY[t] != 0.f) b2_red_add(gY + t, accY[t]);
    if (accG[t] != 0.f) b2_red_add(dgamma + t, accG[t]);
    if (accB[t] != 0.f) b2_red_add(dbeta + t, accB[t]);
  }
}

struct wk_out_dims {
  int Fi, Fo, D, lcb, fmb, N, fpi, fpo, DP;   // fields in / out, dim, LCB and FMB fields, C's width, pitches
};

// Zs[j DP + d] = z[b, j, d] = cat(mlp_out, C's LCB columns)[j, d] + residual (X' or C's projection columns)
__device__ __forceinline__ void wk_stage_z(const float* __restrict__ mlp, const float* __restrict__ C,
                                           const float* __restrict__ xp, int res_mode, int64_t b,
                                           const wk_out_dims& d, float* Zs) {
  const float* mb = mlp + b * d.fmb * d.D;
  for (int t = threadIdx.x; t < d.fmb * d.D; t += blockDim.x) Zs[(t / d.D) * d.DP + t % d.D] = __ldg(mb + t);
  const float* cb = C + b * d.D * d.N;
  for (int t = threadIdx.x; t < d.D * d.N; t += blockDim.x) {
    const int c = t % d.N;
    if (c < d.lcb) Zs[(d.fmb + c) * d.DP + t / d.N] = __ldg(cb + t);
  }
  __syncthreads();
  if (res_mode == 2) {
    for (int t = threadIdx.x; t < d.D * d.N; t += blockDim.x) {
      const int c = t % d.N;
      if (c >= d.lcb) Zs[(c - d.lcb) * d.DP + t / d.N] += __ldg(cb + t);
    }
  } else {
    const float* xb = xp + b * d.D * d.fpi;
    for (int t = threadIdx.x; t < d.D * d.fpi; t += blockDim.x) {
      const int f = t % d.fpi;
      if (f < d.Fi) Zs[f * d.DP + t / d.fpi] += __ldg(xb + t);
    }
  }
  __syncthreads();
}

#define WK_DU 4     // columns per lane of a row of D <= 128

// out = [LN(D)](z): X'_next (out_layout 1, (B D, fpo)) or the flatten (out_layout 0, (B, Fo D)), + operand copy
__global__ void __launch_bounds__(WK_THREADS)
wk_out_fwd_kernel(const float* __restrict__ mlp, const float* __restrict__ C, const float* __restrict__ xp,
                  int64_t batch, wk_out_dims d, int res_mode, const float* __restrict__ gamma,
                  const float* __restrict__ beta, float eps, int out_layout, float* __restrict__ out, void* out_aux,
                  int aux_dtype, int64_t ld_aux, float* __restrict__ ln_mean, float* __restrict__ ln_rstd) {
  extern __shared__ float Zs[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  b2_pdl_wait();
  for (int64_t b = blockIdx.x; b < batch; b += gridDim.x) {
    wk_stage_z(mlp, C, xp, res_mode, b, d, Zs);
    for (int j = warp; j < d.Fo; j += WK_WARPS) {
      float z[WK_DU], s = 0.f;
#pragma unroll
      for (int u = 0; u < WK_DU; ++u) {
        const int c = lane + 32 * u;
        z[u] = c < d.D ? Zs[j * d.DP + c] : 0.f;
        s += z[u];
      }
      float mu = 0.f, rs = 1.f;
      if (gamma) {
        mu = b2_warp_sum(s) / (float) d.D;
        float q = 0.f;
#pragma unroll
        for (int u = 0; u < WK_DU; ++u) {
          const float dz = z[u] - mu;
          if (lane + 32 * u < d.D) q += dz * dz;
        }
        rs = 1.f / sqrtf(b2_warp_sum(q) / (float) d.D + eps);
        if (lane == 0) {
          ln_mean[b * d.Fo + j] = mu;
          ln_rstd[b * d.Fo + j] = rs;
        }
      }
#pragma unroll
      for (int u = 0; u < WK_DU; ++u) {
        const int c = lane + 32 * u;
        if (c < d.D) {
          const float y = gamma ? (z[u] - mu) * rs * __ldg(gamma + c) + __ldg(beta + c) : z[u];
          if (out_layout == 0) {
            const int64_t o = b * d.Fo * d.D + j * d.D + c;
            out[o] = y;
            if (out_aux) {
              const float w[1] = {y};
              rk_store_aux<1>(out_aux, aux_dtype, b * ld_aux + j * d.D + c, w);
            }
          } else {
            Zs[j * d.DP + c] = y;
          }
        }
      }
    }
    __syncthreads();
    if (out_layout == 1) {
      for (int t = threadIdx.x; t < d.D * d.fpo; t += blockDim.x) {
        const int j = t % d.fpo, dd = t / d.fpo;
        const float y = j < d.Fo ? Zs[j * d.DP + dd] : 0.f;
        out[b * d.D * d.fpo + t] = y;
        if (out_aux) {
          const float w[1] = {y};
          rk_store_aux<1>(out_aux, aux_dtype, (b * d.D + dd) * ld_aux + j, w);
        }
      }
      __syncthreads();
    }
  }
  b2_pdl_trigger();
}

// From the output gradient g (layout as the forward's out): dz = LN'(g), written as the FMB MLP's output gradient,
// as dC (LCB columns, and the projection columns), and for an identity residual into gxp ("=" or "+=");
// dbias (projection) += the column sums of dz; dgamma, dbeta += (one atomic per column and CTA)
__global__ void __launch_bounds__(WK_THREADS)
wk_out_bwd_kernel(const float* __restrict__ mlp, const float* __restrict__ C, const float* __restrict__ xp,
                  int64_t batch, wk_out_dims d, int res_mode, const float* __restrict__ gamma,
                  const float* __restrict__ ln_mean, const float* __restrict__ ln_rstd, int g_layout,
                  const float* __restrict__ g, float* __restrict__ g_mlp, float* __restrict__ dC, void* dc_aux,
                  int aux_dtype, int64_t ld_aux, float* __restrict__ gxp, int accumulate, float* __restrict__ dbias,
                  float* __restrict__ dgamma, float* __restrict__ dbeta) {
  extern __shared__ float smem[];
  __shared__ float sg[B2_WUKONG_MAX_DIM], sb[B2_WUKONG_MAX_DIM], sbias[B2_WUKONG_MAX_FIELDS];
  float* Gs = smem;
  float* Zs = Gs + d.Fo * d.DP;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int c = threadIdx.x; c < B2_WUKONG_MAX_DIM; c += blockDim.x) sg[c] = sb[c] = 0.f;
  for (int c = threadIdx.x; c < B2_WUKONG_MAX_FIELDS; c += blockDim.x) sbias[c] = 0.f;
  float acc_g[WK_DU], acc_b[WK_DU];
#pragma unroll
  for (int u = 0; u < WK_DU; ++u) acc_g[u] = acc_b[u] = 0.f;
  b2_pdl_wait();
  for (int64_t b = blockIdx.x; b < batch; b += gridDim.x) {
    if (g_layout == 0) {
      const float* gb = g + b * d.Fo * d.D;
      for (int t = threadIdx.x; t < d.Fo * d.D; t += blockDim.x) Gs[(t / d.D) * d.DP + t % d.D] = __ldg(gb + t);
    } else {
      const float* gb = g + b * d.D * d.fpo;
      for (int t = threadIdx.x; t < d.D * d.fpo; t += blockDim.x) {
        const int j = t % d.fpo;
        if (j < d.Fo) Gs[j * d.DP + t / d.fpo] = __ldg(gb + t);
      }
    }
    if (gamma) wk_stage_z(mlp, C, xp, res_mode, b, d, Zs);      // syncs
    else __syncthreads();
    for (int j = warp; j < d.Fo; j += WK_WARPS) {
      float gz[WK_DU], s = 0.f;
      if (gamma) {
        const float mu = __ldg(ln_mean + b * d.Fo + j), rs = __ldg(ln_rstd + b * d.Fo + j);
        float xh[WK_DU], gy[WK_DU], s1 = 0.f, s2 = 0.f;
#pragma unroll
        for (int u = 0; u < WK_DU; ++u) {
          const int c = lane + 32 * u;
          xh[u] = gy[u] = 0.f;
          if (c < d.D) {
            const float gv = Gs[j * d.DP + c];
            xh[u] = (Zs[j * d.DP + c] - mu) * rs;
            gy[u] = gv * __ldg(gamma + c);
            acc_g[u] += gv * xh[u];
            acc_b[u] += gv;
            s1 += gy[u];
            s2 += gy[u] * xh[u];
          }
        }
        s1 = b2_warp_sum(s1) / (float) d.D;
        s2 = b2_warp_sum(s2) / (float) d.D;
#pragma unroll
        for (int u = 0; u < WK_DU; ++u) gz[u] = rs * ((gy[u] - s1) - xh[u] * s2);
      } else {
#pragma unroll
        for (int u = 0; u < WK_DU; ++u) gz[u] = lane + 32 * u < d.D ? Gs[j * d.DP + lane + 32 * u] : 0.f;
      }
#pragma unroll
      for (int u = 0; u < WK_DU; ++u) {
        const int c = lane + 32 * u;
        if (c < d.D) {
          Gs[j * d.DP + c] = gz[u];
          s += gz[u];
          if (j < d.fmb) g_mlp[b * d.fmb * d.D + j * d.D + c] = gz[u];
        }
      }
      if (res_mode == 2) {
        s = b2_warp_sum(s);
        if (lane == 0) sbias[j] += s;       // row j is always this warp's
      }
    }
    __syncthreads();
    float* cb = dC + b * d.D * d.N;
    for (int t = threadIdx.x; t < d.D * d.N; t += blockDim.x) {
      const int c = t % d.N, dd = t / d.N;
      const float v = c < d.lcb ? Gs[(d.fmb + c) * d.DP + dd] : Gs[(c - d.lcb) * d.DP + dd];
      cb[t] = v;
      if (dc_aux) {
        const float w[1] = {v};
        rk_store_aux<1>(dc_aux, aux_dtype, (b * d.D + dd) * ld_aux + c, w);
      }
    }
    if (res_mode == 1) {
      float* xb = gxp + b * d.D * d.fpi;
      for (int t = threadIdx.x; t < d.D * d.fpi; t += blockDim.x) {
        const int f = t % d.fpi;
        const float v = f < d.Fi ? Gs[f * d.DP + t / d.fpi] : 0.f;
        xb[t] = accumulate ? xb[t] + v : v;
      }
    }
    __syncthreads();
  }
  b2_pdl_trigger();
  if (gamma) {
#pragma unroll
    for (int u = 0; u < WK_DU; ++u) {
      const int c = lane + 32 * u;
      if (c < d.D) {
        if (acc_g[u] != 0.f) atomicAdd(&sg[c], acc_g[u]);
        if (acc_b[u] != 0.f) atomicAdd(&sb[c], acc_b[u]);
      }
    }
  }
  __syncthreads();
  for (int c = threadIdx.x; gamma && c < d.D; c += blockDim.x) {
    if (sg[c] != 0.f) b2_red_add(dgamma + c, sg[c]);
    if (sb[c] != 0.f) b2_red_add(dbeta + c, sb[c]);
  }
  for (int j = threadIdx.x; res_mode == 2 && j < d.Fo; j += blockDim.x)
    if (sbias[j] != 0.f) b2_red_add(dbias + j, sbias[j]);
}

// Ws (N, fpi) = [W_lcb; W_res] zero-padded to fpi columns, bs (N) = [0; b_res]  ("=")
__global__ void __launch_bounds__(256)
wk_pack_kernel(const float* __restrict__ Wl, const float* __restrict__ Wr, const float* __restrict__ br, int Fi,
               int lcb, int N, int fpi, float* __restrict__ Ws, float* __restrict__ bs) {
  b2_pdl_wait();
  for (int64_t t = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; t < (int64_t) N * fpi;
       t += (int64_t) gridDim.x * blockDim.x) {
    const int r = (int) (t / fpi), f = (int) (t % fpi);
    float v = 0.f;
    if (f < Fi) v = r < lcb ? __ldg(Wl + (int64_t) r * Fi + f) : __ldg(Wr + (int64_t) (r - lcb) * Fi + f);
    Ws[t] = v;
    if (bs && f == 0) bs[r] = r < lcb ? 0.f : __ldg(br + r - lcb);
  }
  b2_pdl_trigger();
}

// gW_lcb (lcb, Fi), gW_res (N - lcb, Fi) = the parts of dWs (N, fpi)  ("=")
__global__ void __launch_bounds__(256)
wk_unpack_kernel(const float* __restrict__ dWs, int Fi, int lcb, int N, int fpi, float* __restrict__ gl,
                 float* __restrict__ gr) {
  b2_pdl_wait();
  for (int64_t t = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; t < (int64_t) N * Fi;
       t += (int64_t) gridDim.x * blockDim.x) {
    const int r = (int) (t / Fi), f = (int) (t % Fi);
    const float v = __ldg(dWs + (int64_t) r * fpi + f);
    if (r < lcb) gl[t] = v;
    else gr[t - (int64_t) lcb * Fi] = v;
  }
  b2_pdl_trigger();
}

// ---------------------------------------------------------------------------------
// Host side
// ---------------------------------------------------------------------------------
static int wk_check_fm(int64_t batch, int F, int D, int k) {
  B2_REQUIRE(F >= 1 && F <= B2_WUKONG_MAX_FIELDS, "fields %d outside [1, %d]", F, B2_WUKONG_MAX_FIELDS);
  B2_REQUIRE(D >= 1 && D <= B2_WUKONG_MAX_DIM, "embedding_dim %d outside [1, %d]", D, B2_WUKONG_MAX_DIM);
  B2_REQUIRE(k >= 1 && k <= B2_WUKONG_MAX_RANK, "rank %d outside [1, %d]", k, B2_WUKONG_MAX_RANK);
  B2_REQUIRE(F * k <= B2_WUKONG_MAX_FM_WIDTH, "fields * rank %d > %d", F * k, B2_WUKONG_MAX_FM_WIDTH);
  B2_REQUIRE(batch >= 0, "negative batch");
  const int64_t row = (int64_t) D * wk_pitch(F) > (int64_t) F * k ? (int64_t) D * wk_pitch(F) : (int64_t) F * k;
  B2_REQUIRE(batch <= (((int64_t) 1 << 31) - 1) / row, "batch * row width >= 2^31");
  return B2_OK;
}

static int wk_check_out(int64_t batch, int Fi, int D, int lcb, int fmb, int res_mode) {
  B2_REQUIRE(Fi >= 1 && Fi <= B2_WUKONG_MAX_FIELDS, "fields %d outside [1, %d]", Fi, B2_WUKONG_MAX_FIELDS);
  B2_REQUIRE(D >= 1 && D <= B2_WUKONG_MAX_DIM, "embedding_dim %d outside [1, %d]", D, B2_WUKONG_MAX_DIM);
  B2_REQUIRE(lcb >= 1 && fmb >= 1 && lcb + fmb <= B2_WUKONG_MAX_FIELDS, "lcb %d / fmb %d: need both >= 1 and a sum <= %d",
             lcb, fmb, B2_WUKONG_MAX_FIELDS);
  B2_REQUIRE(res_mode == 1 || res_mode == 2, "res_mode %d is not 1 or 2", res_mode);
  B2_REQUIRE(res_mode != 1 || Fi == lcb + fmb, "an identity residual needs fields %d == lcb + fmb %d", Fi, lcb + fmb);
  B2_REQUIRE(batch >= 0, "negative batch");
  B2_REQUIRE(batch <= (((int64_t) 1 << 31) - 1) / ((int64_t) D * 2 * B2_WUKONG_MAX_FIELDS), "batch * row width >= 2^31");
  return B2_OK;
}

static wk_fm_dims wk_make_fm(int F, int D, int k) {
  wk_fm_dims d;
  d.F = F;
  d.D = D;
  d.k = k;
  d.fp = wk_pitch(F);
  d.DP = D + 1;
  d.KP = k + 1;
  return d;
}

static wk_out_dims wk_make_out(int Fi, int D, int lcb, int fmb, int res_mode) {
  wk_out_dims d;
  d.Fi = Fi;
  d.Fo = lcb + fmb;
  d.D = D;
  d.lcb = lcb;
  d.fmb = fmb;
  d.N = lcb + (res_mode == 2 ? d.Fo : 0);
  d.fpi = wk_pitch(Fi);
  d.fpo = wk_pitch(d.Fo);
  d.DP = D + 1;
  return d;
}

static size_t wk_fm_smem(const wk_fm_dims& d, bool bwd) {
  const size_t n = (size_t) d.F * d.k;
  size_t s = (size_t) d.F * d.KP * 2 + (size_t) d.F * d.DP + (size_t) d.D * d.KP;
  if (bwd) s += (size_t) d.D * d.KP + 3 * n;
  return s * sizeof(float);
}

// One CTA per sample, as many per SM as the shared memory allows (at most 8), the batch in a grid stride.
static int wk_grid(int64_t batch, size_t smem) {
  int64_t per_sm = (int64_t) (200 * 1024 / (smem + 1024));
  per_sm = per_sm < 1 ? 1 : (per_sm > 8 ? 8 : per_sm);
  const int64_t cap = (int64_t) B2_NUM_SMS * per_sm;
  return (int) (batch < cap ? batch : cap);
}

// The dynamic shared memory of a launch may exceed 48 KiB only when the kernel opts in: set on every launch, a
// host call that enqueues nothing.
template <typename K>
static int wk_smem_optin(K kernel, size_t smem) {
  cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) smem);
  if (e != cudaSuccess) return b2_fail(B2_E_CUDA, "wukong: shared memory opt-in failed: %s", cudaGetErrorString(e));
  return B2_OK;
}

// float4 staging: X' rows are always a multiple of 4 wide; X (B, F, D) when D % 4 == 0; both 16-byte aligned
static bool wk_vec(const float* x, int layout, int D) { return rk_al16(x) && (layout == 1 || D % 4 == 0); }

extern "C" B2_API int b2_wukong_fm_fwd(const float* x, int layout, int64_t batch, int fields, int D, int k,
                                       const float* Y, const float* gamma, const float* beta, float eps,
                                       float* fm_out, void* fm_aux, int aux_dtype, int64_t ld_aux, float* xp_out,
                                       void* xp_aux, int64_t ld_xp_aux, float* ln_mean, float* ln_rstd,
                                       void* stream) {
  B2_REQUIRE(x && Y && gamma && beta && fm_out && ln_mean && ln_rstd, "NULL pointer");
  if (int rc = wk_check_fm(batch, fields, D, k)) return rc;
  B2_REQUIRE(layout == 0 || layout == 1, "layout %d is not 0 or 1", layout);
  B2_REQUIRE(xp_out == nullptr || layout == 0, "X'_0 is written from the (B, F, D) layout only");
  B2_REQUIRE(xp_aux == nullptr || xp_out, "xp_aux without xp_out");
  if (int rc = rk_check_aux(fm_aux, aux_dtype, ld_aux, fields * k)) return rc;
  if (int rc = rk_check_aux(xp_aux, aux_dtype, ld_xp_aux, wk_pitch(fields))) return rc;
  if (batch == 0) return B2_OK;
  const wk_fm_dims d = wk_make_fm(fields, D, k);
  const size_t smem = wk_fm_smem(d, false);
  const int grid = wk_grid(batch, smem);
  if (wk_vec(x, layout, D)) {
    if (int rc = wk_smem_optin(wk_fm_fwd_kernel<4>, smem)) return rc;
    B2_LAUNCH(wk_fm_fwd_kernel<4>, grid, WK_THREADS, smem, (cudaStream_t) stream, x, layout, batch, d, Y, gamma, beta,
              eps, fm_out, fm_aux, aux_dtype, ld_aux, xp_out, xp_aux, ld_xp_aux, ln_mean, ln_rstd);
  } else {
    if (int rc = wk_smem_optin(wk_fm_fwd_kernel<1>, smem)) return rc;
    B2_LAUNCH(wk_fm_fwd_kernel<1>, grid, WK_THREADS, smem, (cudaStream_t) stream, x, layout, batch, d, Y, gamma, beta,
              eps, fm_out, fm_aux, aux_dtype, ld_aux, xp_out, xp_aux, ld_xp_aux, ln_mean, ln_rstd);
  }
  B2_CUDA_LAUNCH_CHECK("b2_wukong_fm_fwd");
  return B2_OK;
}

extern "C" B2_API int b2_wukong_fm_bwd(const float* x, int layout, int64_t batch, int fields, int D, int k,
                                       const float* Y, const float* gamma, const float* ln_mean, const float* ln_rstd,
                                       const float* g, const float* gxp, float* gx, int accumulate, float* gY,
                                       float* dgamma, float* dbeta, void* stream) {
  B2_REQUIRE(x && Y && gamma && ln_mean && ln_rstd && g && gx && gY && dgamma && dbeta, "NULL pointer");
  if (int rc = wk_check_fm(batch, fields, D, k)) return rc;
  B2_REQUIRE(layout == 0 || layout == 1, "layout %d is not 0 or 1", layout);
  B2_REQUIRE(gxp == nullptr || layout == 0, "gxp is added in the (B, F, D) layout only");
  if (batch == 0) return B2_OK;
  const wk_fm_dims d = wk_make_fm(fields, D, k);
  const size_t smem = wk_fm_smem(d, true);
  const int grid = wk_grid(batch, smem);
  if (wk_vec(x, layout, D)) {
    if (int rc = wk_smem_optin(wk_fm_bwd_kernel<4>, smem)) return rc;
    B2_LAUNCH(wk_fm_bwd_kernel<4>, grid, WK_THREADS, smem, (cudaStream_t) stream, x, layout, batch, d, Y, gamma,
              ln_mean, ln_rstd, g, gxp, gx, accumulate, gY, dgamma, dbeta);
  } else {
    if (int rc = wk_smem_optin(wk_fm_bwd_kernel<1>, smem)) return rc;
    B2_LAUNCH(wk_fm_bwd_kernel<1>, grid, WK_THREADS, smem, (cudaStream_t) stream, x, layout, batch, d, Y, gamma,
              ln_mean, ln_rstd, g, gxp, gx, accumulate, gY, dgamma, dbeta);
  }
  B2_CUDA_LAUNCH_CHECK("b2_wukong_fm_bwd");
  return B2_OK;
}

extern "C" B2_API int b2_wukong_out_fwd(const float* mlp_out, const float* C, const float* xp, int64_t batch,
                                        int fields, int D, int lcb, int fmb, int res_mode, const float* gamma,
                                        const float* beta, float eps, int out_layout, float* out, void* out_aux,
                                        int aux_dtype, int64_t ld_aux, float* ln_mean, float* ln_rstd,
                                        void* stream) {
  B2_REQUIRE(mlp_out && C && out, "NULL pointer");
  if (int rc = wk_check_out(batch, fields, D, lcb, fmb, res_mode)) return rc;
  B2_REQUIRE(res_mode != 1 || xp, "an identity residual needs X'");
  B2_REQUIRE((gamma == nullptr) == (beta == nullptr), "gamma and beta: both or neither");
  B2_REQUIRE(gamma == nullptr || (ln_mean && ln_rstd), "LayerNorm needs ln_mean and ln_rstd");
  B2_REQUIRE(out_layout == 0 || out_layout == 1, "out_layout %d is not 0 or 1", out_layout);
  const int Fo = lcb + fmb;
  if (int rc = rk_check_aux(out_aux, aux_dtype, ld_aux, out_layout == 0 ? Fo * D : wk_pitch(Fo))) return rc;
  if (batch == 0) return B2_OK;
  const wk_out_dims d = wk_make_out(fields, D, lcb, fmb, res_mode);
  const size_t smem = (size_t) d.Fo * d.DP * sizeof(float);
  if (int rc = wk_smem_optin(wk_out_fwd_kernel, smem)) return rc;
  B2_LAUNCH(wk_out_fwd_kernel, wk_grid(batch, smem), WK_THREADS, smem, (cudaStream_t) stream, mlp_out, C, xp, batch,
            d, res_mode, gamma, beta, eps, out_layout, out, out_aux, aux_dtype, ld_aux, ln_mean, ln_rstd);
  B2_CUDA_LAUNCH_CHECK("b2_wukong_out_fwd");
  return B2_OK;
}

extern "C" B2_API int b2_wukong_out_bwd(const float* mlp_out, const float* C, const float* xp, int64_t batch,
                                        int fields, int D, int lcb, int fmb, int res_mode, const float* gamma,
                                        const float* ln_mean, const float* ln_rstd, int g_layout, const float* g,
                                        float* g_mlp, float* dC, void* dc_aux, int aux_dtype, int64_t ld_aux,
                                        float* gxp, int accumulate, float* dbias, float* dgamma, float* dbeta,
                                        void* stream) {
  B2_REQUIRE(g && g_mlp && dC, "NULL pointer");
  if (int rc = wk_check_out(batch, fields, D, lcb, fmb, res_mode)) return rc;
  B2_REQUIRE(res_mode != 1 || gxp, "an identity residual needs gxp");
  B2_REQUIRE(res_mode != 2 || dbias, "a projection residual needs dbias");
  B2_REQUIRE(gamma == nullptr || (mlp_out && C && (res_mode == 2 || xp) && ln_mean && ln_rstd && dgamma && dbeta),
             "LayerNorm needs mlp_out, C, X', ln_mean, ln_rstd, dgamma and dbeta");
  B2_REQUIRE(g_layout == 0 || g_layout == 1, "g_layout %d is not 0 or 1", g_layout);
  const int N = lcb + (res_mode == 2 ? lcb + fmb : 0);
  if (int rc = rk_check_aux(dc_aux, aux_dtype, ld_aux, N)) return rc;
  if (batch == 0) return B2_OK;
  const wk_out_dims d = wk_make_out(fields, D, lcb, fmb, res_mode);
  const size_t smem = (size_t) (gamma ? 2 : 1) * d.Fo * d.DP * sizeof(float);
  if (int rc = wk_smem_optin(wk_out_bwd_kernel, smem)) return rc;
  B2_LAUNCH(wk_out_bwd_kernel, wk_grid(batch, smem + 3 * 512), WK_THREADS, smem, (cudaStream_t) stream, mlp_out, C,
            xp, batch, d, res_mode, gamma, ln_mean, ln_rstd, g_layout, g, g_mlp, dC, dc_aux, aux_dtype, ld_aux, gxp,
            accumulate, dbias, dgamma, dbeta);
  B2_CUDA_LAUNCH_CHECK("b2_wukong_out_bwd");
  return B2_OK;
}

extern "C" B2_API int b2_wukong_pack(const float* W_lcb, const float* W_res, const float* b_res, int fields, int lcb,
                                     int out_fields, float* Ws, float* bs, void* stream) {
  B2_REQUIRE(W_lcb && Ws, "NULL pointer");
  B2_REQUIRE(fields >= 1 && fields <= B2_WUKONG_MAX_FIELDS && lcb >= 1 && lcb <= B2_WUKONG_MAX_FIELDS,
             "fields %d / lcb %d out of range", fields, lcb);
  B2_REQUIRE(W_res == nullptr || (b_res && bs && out_fields >= 1 && out_fields <= B2_WUKONG_MAX_FIELDS),
             "a projection needs b_res, bs and 1 <= out_fields <= %d", B2_WUKONG_MAX_FIELDS);
  const int N = lcb + (W_res ? out_fields : 0), fpi = wk_pitch(fields);
  const int64_t blocks = b2_ceil_div((int64_t) N * fpi, 256), cap = (int64_t) B2_NUM_SMS * 8;
  B2_LAUNCH(wk_pack_kernel, (int) (blocks > cap ? cap : blocks), 256, 0, (cudaStream_t) stream, W_lcb, W_res, b_res,
            fields, lcb, N, fpi, Ws, W_res ? bs : nullptr);
  B2_CUDA_LAUNCH_CHECK("b2_wukong_pack");
  return B2_OK;
}

extern "C" B2_API int b2_wukong_unpack(const float* dWs, int fields, int lcb, int out_fields, float* gW_lcb,
                                       float* gW_res, void* stream) {
  B2_REQUIRE(dWs && gW_lcb, "NULL pointer");
  B2_REQUIRE(fields >= 1 && fields <= B2_WUKONG_MAX_FIELDS && lcb >= 1 && lcb <= B2_WUKONG_MAX_FIELDS,
             "fields %d / lcb %d out of range", fields, lcb);
  B2_REQUIRE(gW_res == nullptr || (out_fields >= 1 && out_fields <= B2_WUKONG_MAX_FIELDS),
             "out_fields %d out of range", out_fields);
  const int N = lcb + (gW_res ? out_fields : 0);
  const int64_t blocks = b2_ceil_div((int64_t) N * fields, 256), cap = (int64_t) B2_NUM_SMS * 8;
  B2_LAUNCH(wk_unpack_kernel, (int) (blocks > cap ? cap : blocks), 256, 0, (cudaStream_t) stream, dWs, fields, lcb, N,
            wk_pitch(fields), gW_lcb, gW_res);
  B2_CUDA_LAUNCH_CHECK("b2_wukong_unpack");
  return B2_OK;
}

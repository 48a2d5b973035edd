// finalnet.cu — FinalNet's row kernels (model_zoo/FinalNet/src/FinalNet.py), sm_90a.
//
// One FactorizedInteraction layer of a FinalBlock is the caller's GEMM h = x W^T + b (B, 2m), then this file:
//   h2 = h[:, :m], h1 = h[:, m:]          (torch.chunk: the FIRST half is h2)
//   z  = [h2, h1 h2] (concat, n = 2m)  |  h2 + h1 h2 (sum, n = m)
//   out = dropout(act(BatchNorm1d(z)))   (each stage optional)
// z is never stored: every pass forms it again from h.  With batch norm in training mode the forward is a zero fill,
// a column-statistics pass (fp64 sums of z and z^2, one atomic per column and CTA, as Dice) and the apply pass, which
// finalizes mean and rstd per column itself (bn_common.cuh) and, in its blockIdx.x == 0 CTAs, writes them for the
// backward and updates the running statistics.  The backward is a statistics pass (fp64 sums of dy and dy zhat, which
// are dbeta and dgamma) and an apply pass that forms dz and then dh through the product, with dh's GEMM-operand copy
// and the bias gradient as a column sum.  The forward's zero fill also clears the backward's sums.
// Layout: row_common.cuh's; a slot owns VW half-columns j and reads h2 and h1 of them, so h is read once per pass.
//
// Feature gating (FeatureGating, gate_residual "concat") runs one CTA per sample with W (F, F) in shared memory:
//   g = W e + b over the field axis of e (F, D), out = [e, e * g] flattened to (2 F D).
// Its backward recomputes g and sums dW and db per CTA in shared memory (a thread owns fixed elements), then adds them
// with one float atomic per element and CTA.
//
// The 2B loss is one CTA: loss, y_pred and both logit gradients, with b2_logit_bce_fwd's clamp and gradient formula.
// sigmoid is 1 / (1 + expf(-z)) as torch evaluates it in fp32.
#include "row_common.cuh"
#include "bn_common.cuh"
#include "philox.cuh"

__device__ __forceinline__ float fn_sigmoid(float z) { return 1.f / (1.f + expf(-z)); }

__device__ __forceinline__ float fn_act(float y, int act) {
  if (act == B2_ACT_RELU) return y > 0.f ? y : 0.f;
  if (act == B2_ACT_SIGMOID) return fn_sigmoid(y);
  return y;
}

// t * act'(y), y the activation's input
__device__ __forceinline__ float fn_act_bwd(float t, float y, int act) {
  if (act == B2_ACT_RELU) return y > 0.f ? t : 0.f;
  if (act == B2_ACT_SIGMOID) {
    const float s = fn_sigmoid(y);
    return t * (1.f - s) * s;
  }
  return t;
}

// z of VW half-columns: lo (column j) and, with concat, hi (column m + j)
template <int VW>
__device__ __forceinline__ void fn_z(const float (&h2)[VW], const float (&h1)[VW], bool concat, float (&lo)[VW],
                                     float (&hi)[VW]) {
#pragma unroll
  for (int k = 0; k < VW; ++k) {
    const float p = h1[k] * h2[k];
    lo[k] = concat ? h2[k] : h2[k] + p;
    hi[k] = p;
  }
}

// The per-CTA sum over the ty_n rows of `v` (a thread's value of one column), valid in the ty == 0 threads.
__device__ __forceinline__ double fn_cta_sum(double* red, int tx, int tx_n, int ty_n, double v) {
  red[threadIdx.x] = v;
  __syncthreads();
  double s = 0.0;
  if (threadIdx.x < tx_n)
    for (int y = 0; y < ty_n; ++y) s += red[y * tx_n + tx];
  __syncthreads();
  return s;
}

// Adds the CTA's sums of the slot's columns: acc[q][s][k] is quantity q (0, 1) of set s (lo, hi) of column j + k;
// quantity q of column c goes to ws[q n + c].
template <int VW>
__device__ __forceinline__ void fn_flush_sums(double* red, int tx, int tx_n, int ty_n, int ty, int j, int m, int n,
                                              int sets, const double (&acc)[2][2][VW], double* ws) {
#pragma unroll
  for (int q = 0; q < 2; ++q)
#pragma unroll
    for (int s = 0; s < 2; ++s)
#pragma unroll
      for (int k = 0; k < VW; ++k) {
        if (s >= sets) continue;        // uniform over the CTA
        const double t = fn_cta_sum(red, tx, tx_n, ty_n, acc[q][s][k]);
        if (ty == 0 && j < m) atomicAdd(ws + (int64_t) q * n + s * m + j + k, t);
      }
}

// ---- factorized interaction, forward -----------------------------------------------------------------------
// ws[c] += sum_b z, ws[n + c] += sum_b z^2
template <int VW>
__global__ void __launch_bounds__(RK_THREADS)
fn_fi_stats_kernel(const float* __restrict__ h, int64_t batch, int m, int concat, int tx_n, double* __restrict__ ws) {
  __shared__ double red[RK_THREADS];
  const int tx = threadIdx.x % tx_n, ty = threadIdx.x / tx_n, ty_n = blockDim.x / tx_n;
  const int j = (blockIdx.y * tx_n + tx) * VW;
  const int n = concat ? 2 * m : m, sets = concat ? 2 : 1;
  double acc[2][2][VW];
#pragma unroll
  for (int q = 0; q < 2; ++q)
#pragma unroll
    for (int s = 0; s < 2; ++s)
#pragma unroll
      for (int k = 0; k < VW; ++k) acc[q][s][k] = 0.0;
  b2_pdl_wait();
  if (j < m) {
    for (int64_t row = (int64_t) blockIdx.x * ty_n + ty; row < batch; row += (int64_t) gridDim.x * ty_n) {
      float h2[VW], h1[VW], z[2][VW];
      rk_load<VW>(h + row * 2 * m + j, h2);
      rk_load<VW>(h + row * 2 * m + m + j, h1);
      fn_z<VW>(h2, h1, concat, z[0], z[1]);
#pragma unroll
      for (int s = 0; s < 2; ++s)
#pragma unroll
        for (int k = 0; k < VW; ++k) {
          acc[0][s][k] += (double) z[s][k];
          acc[1][s][k] += (double) z[s][k] * (double) z[s][k];
        }
    }
  }
  b2_pdl_trigger();
  fn_flush_sums<VW>(red, tx, tx_n, ty_n, ty, j, m, n, sets, acc, ws);
}

// out = dropout(act(BN(z))): mean / rstd from ws (training) or the running statistics (eval); the blockIdx.x == 0
// CTAs write them to mean_out / rstd_out and, in training, update the running statistics (and num_batches).
template <int VW>
__global__ void __launch_bounds__(RK_THREADS)
fn_fi_fwd_kernel(const float* __restrict__ h, int64_t batch, int m, int concat, int tx_n,
                 const float* __restrict__ gamma, const float* __restrict__ beta, float eps, float momentum,
                 int training, float* running_mean, float* running_var, int64_t* num_batches,
                 const double* __restrict__ ws, int act, const int64_t* __restrict__ drop_rng, int64_t drop_layer,
                 uint32_t drop_thresh, float drop_scale, float* __restrict__ out, void* out_aux, int aux_dtype,
                 int64_t ld_aux, float* __restrict__ mean_out, float* __restrict__ rstd_out) {
  const int tx = threadIdx.x % tx_n, ty = threadIdx.x / tx_n, ty_n = blockDim.x / tx_n;
  const int j = (blockIdx.y * tx_n + tx) * VW;
  const int n = concat ? 2 * m : m, sets = concat ? 2 : 1;
  const bool bn = gamma != nullptr;
  b2_pdl_wait();
  if (bn && training && blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0 && num_batches != nullptr)
    num_batches[0] += 1;
  if (j < m) {
    float mu[2][VW], rs[2][VW], ga[2][VW], be[2][VW];
    if (bn) {
      const bool writer = blockIdx.x == 0 && ty == 0;
#pragma unroll
      for (int s = 0; s < 2; ++s)
#pragma unroll
        for (int k = 0; k < VW; ++k) {
          if (s >= sets) continue;
          const int c = s * m + j + k;
          if (training) {
            b2_bn_finalize(ws[c], ws[n + c], batch, eps, momentum, &mu[s][k], &rs[s][k],
                           writer && running_mean ? running_mean + c : nullptr, writer ? running_var + c : nullptr);
          } else {
            mu[s][k] = running_mean[c];
            rs[s][k] = 1.f / sqrtf(running_var[c] + eps);
          }
          ga[s][k] = __ldg(gamma + c);
          be[s][k] = __ldg(beta + c);
          if (writer) {
            mean_out[c] = mu[s][k];
            rstd_out[c] = rs[s][k];
          }
        }
    }
    uint64_t seed = 0, off = 0;
    if (drop_rng) {
      seed = (uint64_t) drop_rng[0];
      off = (uint64_t) drop_rng[1] + (uint64_t) drop_layer;
    }
    for (int64_t row = (int64_t) blockIdx.x * ty_n + ty; row < batch; row += (int64_t) gridDim.x * ty_n) {
      float h2[VW], h1[VW], z[2][VW];
      rk_load<VW>(h + row * 2 * m + j, h2);
      rk_load<VW>(h + row * 2 * m + m + j, h1);
      fn_z<VW>(h2, h1, concat, z[0], z[1]);
#pragma unroll
      for (int s = 0; s < 2; ++s) {
        if (s >= sets) continue;
        const int c = s * m + j;
        float y[VW];
#pragma unroll
        for (int k = 0; k < VW; ++k) {
          const float t = bn ? (z[s][k] - mu[s][k]) * rs[s][k] * ga[s][k] + be[s][k] : z[s][k];
          y[k] = fn_act(t, act);
        }
        if (drop_rng) {
          const uint32_t keep = b2_drop_keep4(seed, off, (uint64_t) row * n + c, VW, drop_thresh);
#pragma unroll
          for (int k = 0; k < VW; ++k) y[k] = (keep >> k) & 1u ? y[k] * drop_scale : 0.f;
        }
        rk_store<VW>(out + row * n + c, y);
        if (out_aux) rk_store_aux<VW>(out_aux, aux_dtype, row * ld_aux + c, y);
      }
    }
  }
  b2_pdl_trigger();
}

// ---- factorized interaction, backward -----------------------------------------------------------------------
// dy of the VW columns of set s: g through the dropout mask and the activation, with zhat (BN) recomputed
template <int VW>
__device__ __forceinline__ void fn_dy(const float (&z)[VW], const float (&gg)[VW], bool bn, const float (&mu)[VW],
                                      const float (&rs)[VW], const float (&ga)[VW], const float (&be)[VW], int act,
                                      uint32_t keep, bool drop, float drop_scale, float (&xh)[VW], float (&dy)[VW]) {
#pragma unroll
  for (int k = 0; k < VW; ++k) {
    xh[k] = bn ? (z[k] - mu[k]) * rs[k] : z[k];
    const float y = bn ? xh[k] * ga[k] + be[k] : z[k];
    float t = gg[k];
    if (drop) t = (keep >> k) & 1u ? t * drop_scale : 0.f;
    dy[k] = fn_act_bwd(t, y, act);
  }
}

// MODE 0: ws[c] += sum_b dy, ws[n + c] += sum_b dy zhat.  MODE 1: dh (+ aux), dbias += colsum dh, and in the
// blockIdx.x == 0 CTAs dbeta = ws[:n], dgamma = ws[n:] ("=").
template <int VW, int MODE>
__global__ void __launch_bounds__(RK_THREADS)
fn_fi_bwd_kernel(const float* __restrict__ h, int64_t batch, int m, int concat, int tx_n,
                 const float* __restrict__ gamma, const float* __restrict__ beta, const float* __restrict__ mean,
                 const float* __restrict__ rstd, int training, double* __restrict__ ws, int act,
                 const int64_t* __restrict__ drop_rng, int64_t drop_layer, uint32_t drop_thresh, float drop_scale,
                 const float* __restrict__ g, float* __restrict__ dh, void* dh_aux, int aux_dtype, int64_t ld_aux,
                 float* __restrict__ dbias, float* __restrict__ dgamma, float* __restrict__ dbeta) {
  __shared__ double red[MODE == 0 ? RK_THREADS : 1];
  __shared__ float fred[MODE == 1 ? RK_THREADS * VW : 1];
  const int tx = threadIdx.x % tx_n, ty = threadIdx.x / tx_n, ty_n = blockDim.x / tx_n;
  const int j = (blockIdx.y * tx_n + tx) * VW;
  const int n = concat ? 2 * m : m, sets = concat ? 2 : 1;
  const bool bn = gamma != nullptr;
  double acc[2][2][VW];
  float cs[2][VW];
#pragma unroll
  for (int s = 0; s < 2; ++s)
#pragma unroll
    for (int k = 0; k < VW; ++k) {
      acc[0][s][k] = acc[1][s][k] = 0.0;
      cs[s][k] = 0.f;
    }
  b2_pdl_wait();
  if (j < m) {
    float mu[2][VW], rs[2][VW], ga[2][VW], be[2][VW], m0[2][VW], m1[2][VW];
#pragma unroll
    for (int s = 0; s < 2; ++s)
#pragma unroll
      for (int k = 0; k < VW; ++k) {
        mu[s][k] = be[s][k] = m0[s][k] = m1[s][k] = 0.f;
        rs[s][k] = ga[s][k] = 1.f;
        if (bn && s < sets) {
          const int c = s * m + j + k;
          mu[s][k] = __ldg(mean + c);
          rs[s][k] = __ldg(rstd + c);
          ga[s][k] = __ldg(gamma + c);
          be[s][k] = __ldg(beta + c);
          if (MODE == 1) {
            if (training) {
              m0[s][k] = (float) (ws[c] / (double) batch);
              m1[s][k] = (float) (ws[n + c] / (double) batch);
            }
            if (blockIdx.x == 0 && ty == 0) {
              dbeta[c] = (float) ws[c];
              dgamma[c] = (float) ws[n + c];
            }
          }
        }
      }
    uint64_t seed = 0, off = 0;
    if (drop_rng) {
      seed = (uint64_t) drop_rng[0];
      off = (uint64_t) drop_rng[1] + (uint64_t) drop_layer;
    }
    for (int64_t row = (int64_t) blockIdx.x * ty_n + ty; row < batch; row += (int64_t) gridDim.x * ty_n) {
      float h2[VW], h1[VW], z[2][VW], dz[2][VW];
      rk_load<VW>(h + row * 2 * m + j, h2);
      rk_load<VW>(h + row * 2 * m + m + j, h1);
      fn_z<VW>(h2, h1, concat, z[0], z[1]);
#pragma unroll
      for (int s = 0; s < 2; ++s) {
        if (s >= sets) continue;
        const int c = s * m + j;
        float gg[VW], xh[VW], dy[VW];
        rk_load<VW>(g + row * n + c, gg);
        const uint32_t keep = drop_rng ? b2_drop_keep4(seed, off, (uint64_t) row * n + c, VW, drop_thresh) : 0xfu;
        fn_dy<VW>(z[s], gg, bn, mu[s], rs[s], ga[s], be[s], act, keep, drop_rng != nullptr, drop_scale, xh, dy);
#pragma unroll
        for (int k = 0; k < VW; ++k) {
          if (MODE == 0) {
            acc[0][s][k] += (double) dy[k];
            acc[1][s][k] += (double) dy[k] * (double) xh[k];
          } else {
            dz[s][k] = bn ? (dy[k] - m0[s][k] - xh[k] * m1[s][k]) * rs[s][k] * ga[s][k] : dy[k];
          }
        }
      }
      if (MODE == 1) {
        float d2[VW], d1[VW];
#pragma unroll
        for (int k = 0; k < VW; ++k) {
          if (concat) {
            d2[k] = dz[0][k] + dz[1][k] * h1[k];
            d1[k] = dz[1][k] * h2[k];
          } else {
            d2[k] = dz[0][k] + dz[0][k] * h1[k];
            d1[k] = dz[0][k] * h2[k];
          }
          cs[0][k] += d2[k];
          cs[1][k] += d1[k];
        }
        rk_store<VW>(dh + row * 2 * m + j, d2);
        rk_store<VW>(dh + row * 2 * m + m + j, d1);
        if (dh_aux) {
          rk_store_aux<VW>(dh_aux, aux_dtype, row * ld_aux + j, d2);
          rk_store_aux<VW>(dh_aux, aux_dtype, row * ld_aux + m + j, d1);
        }
      }
    }
  }
  b2_pdl_trigger();
  if (MODE == 0) {
    fn_flush_sums<VW>(red, tx, tx_n, ty_n, ty, j, m, n, sets, acc, ws);
  } else if (dbias != nullptr) {
#pragma unroll
    for (int s = 0; s < 2; ++s) {
      rk_cta_colsum<VW>(fred, tx, tx_n, ty_n, cs[s]);
      if (ty == 0 && j < m) {
#pragma unroll
        for (int k = 0; k < VW; ++k)
          if (cs[s][k] != 0.f) b2_red_add(dbias + s * m + j + k, cs[s][k]);
      }
      __syncthreads();
    }
  }
}

// ---- feature gating ------------------------------------------------------------------------------------------
// out[b] = [e_b, e_b * (W e_b + bias)] over the field axis, one sample per CTA iteration
__global__ void __launch_bounds__(256)
fn_gate_fwd_kernel(const float* __restrict__ e, int64_t batch, int F, int D, const float* __restrict__ W,
                   const float* __restrict__ bias, float* __restrict__ out, void* out_aux, int aux_dtype,
                   int64_t ld_aux) {
  extern __shared__ float smem[];
  float* sW = smem;
  float* sb = sW + F * F;
  float* se = sb + F;
  const int FD = F * D;
  b2_pdl_wait();
  for (int t = threadIdx.x; t < F * F; t += blockDim.x) sW[t] = __ldg(W + t);
  for (int t = threadIdx.x; t < F; t += blockDim.x) sb[t] = __ldg(bias + t);
  for (int64_t b = blockIdx.x; b < batch; b += gridDim.x) {
    __syncthreads();
    for (int t = threadIdx.x; t < FD; t += blockDim.x) se[t] = __ldg(e + b * FD + t);
    __syncthreads();
    float* o = out + b * 2 * FD;
    for (int t = threadIdx.x; t < FD; t += blockDim.x) {
      const int i = t / D, d = t - i * D;
      float acc = 0.f;
      for (int jf = 0; jf < F; ++jf) acc = fmaf(sW[i * F + jf], se[jf * D + d], acc);
      const float ev = se[t], gv = ev * (acc + sb[i]);
      o[t] = ev;
      o[FD + t] = gv;
      if (out_aux) {
        const float a[1] = {ev}, c[1] = {gv};
        rk_store_aux<1>(out_aux, aux_dtype, b * ld_aux + t, a);
        rk_store_aux<1>(out_aux, aux_dtype, b * ld_aux + FD + t, c);
      }
    }
  }
  b2_pdl_trigger();
}

// From g = d out (B, 2 F D): de "=" or "+=" = g1 + g2 * gate + W^T (g2 * e) over the field axis; dW += (g2 * e) e^T,
// db += sum_d g2 * e (per CTA in shared memory, then one atomic per element and CTA)
__global__ void __launch_bounds__(256)
fn_gate_bwd_kernel(const float* __restrict__ e, int64_t batch, int F, int D, const float* __restrict__ W,
                   const float* __restrict__ bias, const float* __restrict__ g, float* de, int accumulate,
                   float* __restrict__ dW, float* __restrict__ db) {
  extern __shared__ float smem[];
  const int FD = F * D;
  float* sW = smem;
  float* sdW = sW + F * F;
  float* sb = sdW + F * F;
  float* sdb = sb + F;
  float* se = sdb + F;
  float* sdg = se + FD;
  float* sdd = sdg + FD;
  b2_pdl_wait();
  for (int t = threadIdx.x; t < F * F; t += blockDim.x) {
    sW[t] = __ldg(W + t);
    sdW[t] = 0.f;
  }
  for (int t = threadIdx.x; t < F; t += blockDim.x) {
    sb[t] = __ldg(bias + t);
    sdb[t] = 0.f;
  }
  for (int64_t b = blockIdx.x; b < batch; b += gridDim.x) {
    __syncthreads();
    for (int t = threadIdx.x; t < FD; t += blockDim.x) se[t] = __ldg(e + b * FD + t);
    __syncthreads();
    const float* gb = g + b * 2 * FD;
    for (int t = threadIdx.x; t < FD; t += blockDim.x) {
      const int i = t / D, d = t - i * D;
      float acc = 0.f;
      for (int jf = 0; jf < F; ++jf) acc = fmaf(sW[i * F + jf], se[jf * D + d], acc);
      const float g1 = __ldg(gb + t), g2 = __ldg(gb + FD + t);
      sdg[t] = g2 * se[t];
      sdd[t] = g1 + g2 * (acc + sb[i]);
    }
    __syncthreads();
    float* dr = de + b * FD;
    for (int t = threadIdx.x; t < FD; t += blockDim.x) {
      const int jf = t / D, d = t - jf * D;
      float v = sdd[t];
      for (int i = 0; i < F; ++i) v = fmaf(sW[i * F + jf], sdg[i * D + d], v);
      dr[t] = accumulate ? dr[t] + v : v;      // dr is not read through the read-only path: the caller may have just written it
    }
    for (int t = threadIdx.x; t < F * F; t += blockDim.x) {
      const int i = t / F, jf = t - i * F;
      float v = 0.f;
      for (int d = 0; d < D; ++d) v = fmaf(sdg[i * D + d], se[jf * D + d], v);
      sdW[t] += v;
    }
    for (int i = threadIdx.x; i < F; i += blockDim.x) {
      float v = 0.f;
      for (int d = 0; d < D; ++d) v += sdg[i * D + d];
      sdb[i] += v;
    }
  }
  b2_pdl_trigger();
  __syncthreads();
  for (int t = threadIdx.x; t < F * F; t += blockDim.x)
    if (sdW[t] != 0.f) b2_red_add(dW + t, sdW[t]);
  for (int t = threadIdx.x; t < F; t += blockDim.x)
    if (sdb[t] != 0.f) b2_red_add(db + t, sdb[t]);
}

// ---- the 2B loss ---------------------------------------------------------------------------------------------
__device__ __forceinline__ float fn_bce(float p, float y) {
  const float lp = fmaxf(logf(p), -100.f), lq = fmaxf(log1pf(-p), -100.f);
  return -(y * lp + (1.f - y) * lq);
}

// d BCE(sigmoid(z), y) / dz over the batch mean, as logit_bce_kernel forms it
__device__ __forceinline__ float fn_bce_grad(float p, float y, float inv_b) {
  const float pq = (1.f - p) * p;
  return ((p - y) / fmaxf(pq, 1e-12f)) * inv_b * pq;
}

__global__ void __launch_bounds__(1024)
fn_loss_kernel(const float* __restrict__ y1, const float* __restrict__ y2, const float* __restrict__ label,
               int64_t batch, float* __restrict__ loss, float* __restrict__ y_pred, float* __restrict__ g1,
               float* __restrict__ g2) {
  __shared__ float red[32];
  const float inv_b = 1.f / (float) batch;
  b2_pdl_wait();
  float part = 0.f;
  for (int64_t i = threadIdx.x; i < batch; i += blockDim.x) {
    const float a = __ldg(y1 + i), c = __ldg(y2 + i), y = __ldg(label + i);
    const float p = fn_sigmoid(0.5f * (a + c)), p1 = fn_sigmoid(a), p2 = fn_sigmoid(c);
    part += fn_bce(p, y) + fn_bce(p1, p) + fn_bce(p2, p);
    const float gm = 0.5f * fn_bce_grad(p, y, inv_b);
    y_pred[i] = p;
    g1[i] = gm + fn_bce_grad(p1, p, inv_b);
    g2[i] = gm + fn_bce_grad(p2, p, inv_b);
  }
  const float t = b2_block_sum(part, red);
  b2_pdl_trigger();
  if (threadIdx.x == 0) loss[0] = t * inv_b;
}

// ---------------------------------------------------------------------------------
// Host side
// ---------------------------------------------------------------------------------
static int fn_check_fi(int64_t batch, int half, int residual, int act, int training, const float* gamma,
                       const float* beta) {
  B2_REQUIRE(residual == B2_FINALNET_CONCAT || residual == B2_FINALNET_SUM, "residual %d is not a B2_FINALNET_* code",
             residual);
  const int n = residual == B2_FINALNET_CONCAT ? 2 * half : half;
  B2_REQUIRE(half >= 1 && n <= B2_FINALNET_MAX_WIDTH, "layer width %d (half %d) outside [1, %d]", n, half,
             B2_FINALNET_MAX_WIDTH);
  B2_REQUIRE(act == B2_ACT_NONE || act == B2_ACT_RELU || act == B2_ACT_SIGMOID, "act %d is not a B2_ACT_* code", act);
  B2_REQUIRE((gamma == nullptr) == (beta == nullptr), "gamma and beta: both or neither");
  B2_REQUIRE(batch >= 0, "negative batch");
  B2_REQUIRE(!(training && gamma != nullptr) || batch != 1,
             "batch norm in training mode needs more than 1 value per channel, got batch %lld", (long long) batch);
  B2_REQUIRE(batch * 2 * (int64_t) half < ((int64_t) 1 << 31), "batch * 2 half >= 2^31");
  return B2_OK;
}

// Launches k4 (the float4 instantiation) on the float4 path, k1 (the scalar one) otherwise.
template <typename K4, typename K1, typename... Args>
static void fn_launch(bool vec, K4 k4, K1 k1, const rk_grid& g, cudaStream_t st, Args... args) {
  if (vec) B2_LAUNCH(k4, g.grid, g.threads, 0, st, args...);
  else B2_LAUNCH(k1, g.grid, g.threads, 0, st, args...);
}

extern "C" B2_API int b2_finalnet_fi_fwd(const float* h, int64_t batch, int half, int residual, const float* gamma,
                                         const float* beta, float eps, float momentum, int training,
                                         float* running_mean, float* running_var, int64_t* num_batches,
                                         double* stats_ws, int act, const int64_t* drop_rng, int64_t drop_layer,
                                         uint32_t drop_thresh, float drop_scale, float* out, void* out_aux,
                                         int aux_dtype, int64_t ld_aux, float* mean, float* rstd, void* stream) {
  B2_REQUIRE(h && out, "NULL pointer");
  if (int rc = fn_check_fi(batch, half, residual, act, training, gamma, beta)) return rc;
  const bool bn = gamma != nullptr;
  B2_REQUIRE(!bn || (mean && rstd && running_mean && running_var), "batch norm needs mean, rstd and running statistics");
  B2_REQUIRE(!(bn && training) || (stats_ws && num_batches), "batch norm in training needs stats_ws and num_batches");
  const bool concat = residual == B2_FINALNET_CONCAT;
  const int n = concat ? 2 * half : half;
  if (int rc = rk_check_aux(out_aux, aux_dtype, ld_aux, n)) return rc;
  B2_REQUIRE(batch * (ld_aux > n ? ld_aux : (int64_t) n) < ((int64_t) 1 << 31), "batch * row pitch >= 2^31");
  if (batch == 0) return B2_OK;
  cudaStream_t st = (cudaStream_t) stream;
  const void* ptrs[] = {h, out};
  const bool vec = rk_vec(half, ptrs, 2, out_aux, aux_dtype, ld_aux);
  const rk_grid gr = rk_plan(batch, half, vec ? 4 : 1, 8);
  if (bn && training) {
    // the backward's two sums (stats_ws + 2n) are cleared here too
    cudaError_t e = cudaMemsetAsync(stats_ws, 0, sizeof(double) * 4 * n, st);
    if (e != cudaSuccess) return b2_fail(B2_E_CUDA, "b2_finalnet_fi_fwd: memset: %s", cudaGetErrorString(e));
    const rk_grid gs = rk_plan(batch, half, vec ? 4 : 1, 4);
    fn_launch(vec, fn_fi_stats_kernel<4>, fn_fi_stats_kernel<1>, gs, st, h, batch, half, (int) concat, gs.tx_n,
              stats_ws);
  }
  fn_launch(vec, fn_fi_fwd_kernel<4>, fn_fi_fwd_kernel<1>, gr, st, h, batch, half, (int) concat, gr.tx_n, gamma, beta,
            eps, momentum, training, running_mean, running_var, num_batches, (const double*) stats_ws, act, drop_rng,
            drop_layer, drop_thresh, drop_scale, out, out_aux, aux_dtype, ld_aux, mean, rstd);
  B2_CUDA_LAUNCH_CHECK("b2_finalnet_fi_fwd");
  return B2_OK;
}

extern "C" B2_API int b2_finalnet_fi_bwd(const float* h, int64_t batch, int half, int residual, const float* gamma,
                                         const float* beta, const float* mean, const float* rstd, int training,
                                         double* stats_ws, int zero_ws, int act, const int64_t* drop_rng,
                                         int64_t drop_layer, uint32_t drop_thresh, float drop_scale, const float* g,
                                         float* dh, void* dh_aux, int aux_dtype, int64_t ld_aux, float* dbias,
                                         float* dgamma, float* dbeta, void* stream) {
  B2_REQUIRE(h && g && dh, "NULL pointer");
  if (int rc = fn_check_fi(batch, half, residual, act, training, gamma, beta)) return rc;
  const bool bn = gamma != nullptr;
  B2_REQUIRE(!bn || (mean && rstd && stats_ws && dgamma && dbeta), "batch norm needs mean, rstd, stats_ws, dgamma, dbeta");
  if (int rc = rk_check_aux(dh_aux, aux_dtype, ld_aux, 2 * half)) return rc;
  B2_REQUIRE(batch * (ld_aux > 2 * half ? ld_aux : (int64_t) 2 * half) < ((int64_t) 1 << 31),
             "batch * row pitch >= 2^31");
  if (batch == 0) return B2_OK;
  cudaStream_t st = (cudaStream_t) stream;
  const bool concat = residual == B2_FINALNET_CONCAT;
  const int n = concat ? 2 * half : half;
  const void* ptrs[] = {h, g, dh};
  const bool vec = rk_vec(half, ptrs, 3, dh_aux, aux_dtype, ld_aux);
  const rk_grid gr = rk_plan(batch, half, vec ? 4 : 1, 4);
  auto launch = [&](auto k4, auto k1) {
    fn_launch(vec, k4, k1, gr, st, h, batch, half, (int) concat, gr.tx_n, gamma, beta, mean, rstd, training, stats_ws,
              act, drop_rng, drop_layer, drop_thresh, drop_scale, g, dh, dh_aux, aux_dtype, ld_aux, dbias, dgamma, dbeta);
  };
  if (bn) {
    if (zero_ws) {
      cudaError_t e = cudaMemsetAsync(stats_ws, 0, sizeof(double) * 2 * n, st);
      if (e != cudaSuccess) return b2_fail(B2_E_CUDA, "b2_finalnet_fi_bwd: memset: %s", cudaGetErrorString(e));
    }
    launch(fn_fi_bwd_kernel<4, 0>, fn_fi_bwd_kernel<1, 0>);
  }
  launch(fn_fi_bwd_kernel<4, 1>, fn_fi_bwd_kernel<1, 1>);
  B2_CUDA_LAUNCH_CHECK("b2_finalnet_fi_bwd");
  return B2_OK;
}

static int fn_check_gate(int64_t batch, int F, int D) {
  B2_REQUIRE(F >= 1 && F <= B2_FINALNET_MAX_FIELDS, "fields %d outside [1, %d]", F, B2_FINALNET_MAX_FIELDS);
  B2_REQUIRE(D >= 1 && D <= B2_FINALNET_MAX_DIM, "embedding dim %d outside [1, %d]", D, B2_FINALNET_MAX_DIM);
  B2_REQUIRE(F * D <= B2_FINALNET_MAX_GATE_WIDTH, "fields * dim = %d > %d", F * D, B2_FINALNET_MAX_GATE_WIDTH);
  B2_REQUIRE(batch >= 0, "negative batch");
  B2_REQUIRE(batch * 2 * (int64_t) F * D < ((int64_t) 1 << 31), "batch * 2 fields * dim >= 2^31");
  return B2_OK;
}

static unsigned fn_gate_grid(int64_t batch, size_t smem) {
  int per_sm = (int) (200 * 1024 / (smem + 1024));
  per_sm = per_sm < 1 ? 1 : (per_sm > 8 ? 8 : per_sm);
  const int64_t cap = (int64_t) B2_NUM_SMS * per_sm;
  return (unsigned) (batch < cap ? batch : cap);
}

extern "C" B2_API int b2_finalnet_gate_fwd(const float* e, int64_t batch, int fields, int dim, const float* W,
                                           const float* bias, float* out, void* out_aux, int aux_dtype,
                                           int64_t ld_aux, void* stream) {
  B2_REQUIRE(e && W && bias && out, "NULL pointer");
  if (int rc = fn_check_gate(batch, fields, dim)) return rc;
  if (int rc = rk_check_aux(out_aux, aux_dtype, ld_aux, 2 * fields * dim)) return rc;
  B2_REQUIRE(batch * (ld_aux > 2 * fields * dim ? ld_aux : (int64_t) 2 * fields * dim) < ((int64_t) 1 << 31),
             "batch * row pitch >= 2^31");
  if (batch == 0) return B2_OK;
  const size_t smem = sizeof(float) * ((size_t) fields * fields + fields + (size_t) fields * dim);
  cudaError_t err = cudaFuncSetAttribute(fn_gate_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) smem);
  if (err != cudaSuccess) return b2_fail(B2_E_CUDA, "b2_finalnet_gate_fwd: smem opt-in: %s", cudaGetErrorString(err));
  B2_LAUNCH(fn_gate_fwd_kernel, fn_gate_grid(batch, smem), 256, smem, (cudaStream_t) stream, e, batch, fields, dim, W,
            bias, out, out_aux, aux_dtype, ld_aux);
  B2_CUDA_LAUNCH_CHECK("b2_finalnet_gate_fwd");
  return B2_OK;
}

extern "C" B2_API int b2_finalnet_gate_bwd(const float* e, int64_t batch, int fields, int dim, const float* W,
                                           const float* bias, const float* g, float* de, int accumulate, float* dW,
                                           float* db, void* stream) {
  B2_REQUIRE(e && W && bias && g && de && dW && db, "NULL pointer");
  if (int rc = fn_check_gate(batch, fields, dim)) return rc;
  if (batch == 0) return B2_OK;
  const size_t smem = sizeof(float) * (2 * (size_t) fields * fields + 2 * fields + 3 * (size_t) fields * dim);
  cudaError_t err = cudaFuncSetAttribute(fn_gate_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) smem);
  if (err != cudaSuccess) return b2_fail(B2_E_CUDA, "b2_finalnet_gate_bwd: smem opt-in: %s", cudaGetErrorString(err));
  B2_LAUNCH(fn_gate_bwd_kernel, fn_gate_grid(batch, smem), 256, smem, (cudaStream_t) stream, e, batch, fields, dim, W,
            bias, g, de, accumulate, dW, db);
  B2_CUDA_LAUNCH_CHECK("b2_finalnet_gate_bwd");
  return B2_OK;
}

extern "C" B2_API int b2_finalnet_loss(const float* y1, const float* y2, const float* label, int64_t batch,
                                       float* loss, float* y_pred, float* g1, float* g2, void* stream) {
  B2_REQUIRE(y1 && y2 && label && loss && y_pred && g1 && g2, "NULL pointer");
  B2_REQUIRE(batch >= 1, "batch must be >= 1");
  B2_LAUNCH(fn_loss_kernel, 1, 1024, 0, (cudaStream_t) stream, y1, y2, label, batch, loss, y_pred, g1, g2);
  B2_CUDA_LAUNCH_CHECK("b2_finalnet_loss");
  return B2_OK;
}

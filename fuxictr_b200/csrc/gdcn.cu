// gdcn.cu — the gated cross layer of GDCN (Gated Deep & Cross Network), sm_90a.
//
// Layer i (x_i, x_0 (B, d)):  x_{i+1} = x_0 * (x_i W_i^T + b_i) * sigmoid(x_i Wg_i^T) + x_i
// Both contractions are ONE GEMM on the stacked weight Wp = [W; Wg] (2d, d): P = x_i Wp^T = [u | z].  This file
// holds what lies around it: the pack of Wp, the row kernel that gates P into x_{i+1} (and back), and the split
// of the stacked weight gradient.  Layouts: include/fuxictr_b200.h "GDCN".
//
// Row kernels: row_common.cuh's layout.  The backward sums dlin per column (rk_cta_colsum) and adds that into db with
// one float atomic per column and CTA (at most 4 CTAs per SM, so few atomics meet on one column).
// sigmoid is 1 / (1 + expf(-z)) as torch evaluates it in fp32 (not __expf: its error shows at the 1e-5 bar).
#include "row_common.cuh"

__device__ __forceinline__ float gd_sigmoid(float z) { return 1.f / (1.f + expf(-z)); }

// out = x0 * (u + b) * sigmoid(z) + xi, u = P[:, :d], z = P[:, d:]
template <int VW>
__global__ void __launch_bounds__(RK_THREADS)
gdcn_fwd_kernel(const float* __restrict__ P, const float* __restrict__ b, const float* __restrict__ x0,
                const float* __restrict__ xi, int64_t batch, int d, int tx_n, float* __restrict__ out,
                void* out_aux, int aux_dtype, int64_t ld_aux) {
  const int tx = threadIdx.x % tx_n, ty = threadIdx.x / tx_n, ty_n = blockDim.x / tx_n;
  const int c = (blockIdx.y * tx_n + tx) * VW;
  b2_pdl_wait();
  if (c < d) {
    float bb[VW];
    rk_load<VW>(b + c, bb);
    for (int64_t row = (int64_t) blockIdx.x * ty_n + ty; row < batch; row += (int64_t) gridDim.x * ty_n) {
      float u[VW], z[VW], a[VW], x[VW], o[VW];
      rk_load<VW>(P + row * 2 * d + c, u);
      rk_load<VW>(P + row * 2 * d + d + c, z);
      rk_load<VW>(x0 + row * d + c, a);
      rk_load<VW>(xi + row * d + c, x);
#pragma unroll
      for (int k = 0; k < VW; ++k) o[k] = a[k] * (u[k] + bb[k]) * gd_sigmoid(z[k]) + x[k];
      rk_store<VW>(out + row * d + c, o);
      if (out_aux) rk_store_aux<VW>(out_aux, aux_dtype, row * ld_aux + c, o);
    }
  }
  b2_pdl_trigger();
}

// dP = [g x0 s | g x0 lin s (1 - s)], gx0 = g lin s, db += sum_rows g x0 s    (lin = u + b, s = sigmoid(z))
template <int VW>
__global__ void __launch_bounds__(RK_THREADS)
gdcn_bwd_kernel(const float* __restrict__ P, const float* __restrict__ b, const float* __restrict__ x0,
                const float* __restrict__ g, int64_t batch, int d, int tx_n, float* __restrict__ dP, void* dp_aux,
                int aux_dtype, int64_t ld_aux, float* __restrict__ gx0, float* __restrict__ db) {
  __shared__ float red[RK_THREADS * VW];
  const int tx = threadIdx.x % tx_n, ty = threadIdx.x / tx_n, ty_n = blockDim.x / tx_n;
  const int c = (blockIdx.y * tx_n + tx) * VW;
  float acc[VW];
#pragma unroll
  for (int k = 0; k < VW; ++k) acc[k] = 0.f;
  b2_pdl_wait();
  if (c < d) {
    float bb[VW];
    rk_load<VW>(b + c, bb);
    for (int64_t row = (int64_t) blockIdx.x * ty_n + ty; row < batch; row += (int64_t) gridDim.x * ty_n) {
      float u[VW], z[VW], a[VW], gg[VW], du[VW], dz[VW], ga[VW];
      rk_load<VW>(P + row * 2 * d + c, u);
      rk_load<VW>(P + row * 2 * d + d + c, z);
      rk_load<VW>(x0 + row * d + c, a);
      rk_load<VW>(g + row * d + c, gg);
#pragma unroll
      for (int k = 0; k < VW; ++k) {
        const float lin = u[k] + bb[k], s = gd_sigmoid(z[k]), ga_s = gg[k] * a[k] * s;
        du[k] = ga_s;
        dz[k] = ga_s * lin * (1.f - s);
        ga[k] = gg[k] * lin * s;
        acc[k] += ga_s;
      }
      rk_store<VW>(dP + row * 2 * d + c, du);
      rk_store<VW>(dP + row * 2 * d + d + c, dz);
      rk_store<VW>(gx0 + row * d + c, ga);
      if (dp_aux) {
        rk_store_aux<VW>(dp_aux, aux_dtype, row * ld_aux + c, du);
        rk_store_aux<VW>(dp_aux, aux_dtype, row * ld_aux + d + c, dz);
      }
    }
  }
  b2_pdl_trigger();
  rk_cta_colsum<VW>(red, tx, tx_n, ty_n, acc);
  if (ty == 0 && c < d) {
#pragma unroll
    for (int k = 0; k < VW; ++k)
      if (acc[k] != 0.f) b2_red_add(db + c + k, acc[k]);
  }
}

// Wp (2d, d) = [W; Wg]  ("=")
__global__ void __launch_bounds__(256)
gdcn_pack_kernel(const float* __restrict__ W, const float* __restrict__ Wg, int64_t n, float* __restrict__ Wp) {
  b2_pdl_wait();
  for (int64_t t = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; t < 2 * n; t += (int64_t) gridDim.x * blockDim.x)
    Wp[t] = t < n ? __ldg(W + t) : __ldg(Wg + (t - n));
  b2_pdl_trigger();
}

// gW = dWp[:d], gWg = dWp[d:]  ("=")
__global__ void __launch_bounds__(256)
gdcn_unpack_kernel(const float* __restrict__ dWp, int64_t n, float* __restrict__ gW, float* __restrict__ gWg) {
  b2_pdl_wait();
  for (int64_t t = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; t < 2 * n; t += (int64_t) gridDim.x * blockDim.x) {
    const float v = __ldg(dWp + t);
    if (t < n) gW[t] = v;
    else gWg[t - n] = v;
  }
  b2_pdl_trigger();
}

// ---------------------------------------------------------------------------------
// Host side
// ---------------------------------------------------------------------------------
static int gd_check(int64_t batch, int d) {
  B2_REQUIRE(d >= 1, "width d = %d < 1", d);
  B2_REQUIRE(batch >= 0, "negative batch");
  B2_REQUIRE(batch * 2 * (int64_t) d < ((int64_t) 1 << 31), "batch * 2d = %lld >= 2^31",
             (long long) (batch * 2 * (int64_t) d));
  return B2_OK;
}

extern "C" B2_API int b2_gdcn_pack(const float* W, const float* Wg, int d, float* Wp, void* stream) {
  B2_REQUIRE(W && Wg && Wp, "NULL pointer");
  if (int rc = gd_check(0, d)) return rc;
  const int64_t n = (int64_t) d * d;
  const int64_t blocks = b2_ceil_div(2 * n, 256), cap = (int64_t) B2_NUM_SMS * 8;
  B2_LAUNCH(gdcn_pack_kernel, (int) (blocks > cap ? cap : blocks), 256, 0, (cudaStream_t) stream, W, Wg, n, Wp);
  B2_CUDA_LAUNCH_CHECK("b2_gdcn_pack");
  return B2_OK;
}

extern "C" B2_API int b2_gdcn_fwd(const float* P, const float* b, const float* x0, const float* xi, int64_t batch,
                                  int d, float* out, void* out_aux, int aux_dtype, int64_t ld_aux, void* stream) {
  B2_REQUIRE(P && b && x0 && xi && out, "NULL pointer");
  if (int rc = gd_check(batch, d)) return rc;
  if (int rc = rk_check_aux(out_aux, aux_dtype, ld_aux, d)) return rc;
  if (batch == 0) return B2_OK;
  const void* ptrs[] = {P, b, x0, xi, out};
  if (rk_vec(d, ptrs, 5, out_aux, aux_dtype, ld_aux)) {
    const rk_grid g = rk_plan(batch, d, 4, 8);
    B2_LAUNCH(gdcn_fwd_kernel<4>, g.grid, g.threads, 0, (cudaStream_t) stream, P, b, x0, xi, batch, d, g.tx_n,
              out, out_aux, aux_dtype, ld_aux);
  } else {
    const rk_grid g = rk_plan(batch, d, 1, 8);
    B2_LAUNCH(gdcn_fwd_kernel<1>, g.grid, g.threads, 0, (cudaStream_t) stream, P, b, x0, xi, batch, d, g.tx_n,
              out, out_aux, aux_dtype, ld_aux);
  }
  B2_CUDA_LAUNCH_CHECK("b2_gdcn_fwd");
  return B2_OK;
}

extern "C" B2_API int b2_gdcn_bwd(const float* P, const float* b, const float* x0, const float* g, int64_t batch,
                                  int d, float* dP, void* dp_aux, int aux_dtype, int64_t ld_aux, float* gx0, float* db,
                                  void* stream) {
  B2_REQUIRE(P && b && x0 && g && dP && gx0 && db, "NULL pointer");
  if (int rc = gd_check(batch, d)) return rc;
  if (int rc = rk_check_aux(dp_aux, aux_dtype, ld_aux, 2 * d)) return rc;
  if (batch == 0) return B2_OK;
  const void* ptrs[] = {P, b, x0, g, dP, gx0, db};
  if (rk_vec(d, ptrs, 7, dp_aux, aux_dtype, ld_aux)) {
    const rk_grid p = rk_plan(batch, d, 4, 4);
    B2_LAUNCH(gdcn_bwd_kernel<4>, p.grid, p.threads, 0, (cudaStream_t) stream, P, b, x0, g, batch, d, p.tx_n, dP,
              dp_aux, aux_dtype, ld_aux, gx0, db);
  } else {
    const rk_grid p = rk_plan(batch, d, 1, 4);
    B2_LAUNCH(gdcn_bwd_kernel<1>, p.grid, p.threads, 0, (cudaStream_t) stream, P, b, x0, g, batch, d, p.tx_n, dP,
              dp_aux, aux_dtype, ld_aux, gx0, db);
  }
  B2_CUDA_LAUNCH_CHECK("b2_gdcn_bwd");
  return B2_OK;
}

extern "C" B2_API int b2_gdcn_unpack(const float* dWp, int d, float* gW, float* gWg, void* stream) {
  B2_REQUIRE(dWp && gW && gWg, "NULL pointer");
  if (int rc = gd_check(0, d)) return rc;
  const int64_t n = (int64_t) d * d;
  const int64_t blocks = b2_ceil_div(2 * n, 256), cap = (int64_t) B2_NUM_SMS * 8;
  B2_LAUNCH(gdcn_unpack_kernel, (int) (blocks > cap ? cap : blocks), 256, 0, (cudaStream_t) stream, dWp, n, gW, gWg);
  B2_CUDA_LAUNCH_CHECK("b2_gdcn_unpack");
  return B2_OK;
}

// crossmix.cu — CrossNetMix (DCN-Mix), the low-rank mixture of experts of DCNv2, sm_90a.
//
// Reference semantics (reczoo/FuxiCTR v2.3.10):
//   CrossNetMix.forward  fuxictr/pytorch/layers/interactions/cross_net.py:158-201
//
// Layer i (x_l (B, d), experts e = 1..E, rank r):
//   h_e = tanh(x_l V_e)   v_e = tanh(h_e C_e^T)   p = softmax_e(x_l g_e^T)
//   x_{l+1} = x_l + x0 * ([p_1 v_1 | ... | p_E v_E] @ [U_1 | ... | U_E]^T + b)        (sum_e p_e = 1)
// The two contractions with d are the wgmma GEMM (or the SIMT GEMM) on packed weights; this file holds
// what lies between them: the pack of W1 = [V_e^T ; g_e] and W2 = [U_e], the per-row expert kernel in both
// directions, and the scatter of the packed weight gradients back to U, V and the gating weights.
// Layouts: include/fuxictr_b200.h "CrossNetMix".
//
// Row kernels: one warp per row; lane t owns the rank columns c = t, t + 32, ... of the E*r row.  All
// experts' C sit in shared memory with row pitch r + 1, so the lanes of a warp, which read consecutive rows
// of C, hit distinct banks.  tanhf / expf (not the .approx forms: their ~2^-11 error would show at the
// layer's 1e-5 bar).
#include "b2_common.cuh"

#define CM_WARPS 8
#define CM_THREADS (CM_WARPS * 32)
#define CM_MAX_COLS (B2_CROSSMIX_MAX_COLS / 32)    // rank columns per lane
#define CM_TILE_ROWS (2 * CM_WARPS)                // backward: rows whose h, dz are staged for one dC pass

static __host__ __device__ __forceinline__ int cm_n1(int r, int E) { return (E * r + E + 3) / 4 * 4; }
static __host__ __device__ __forceinline__ int cm_k2(int r, int E) { return (E * r + 3) / 4 * 4; }

__device__ __forceinline__ void cm_store_aux(void* aux, int aux_dtype, int64_t off, float v) {
  if (aux_dtype == B2_BF16) reinterpret_cast<__nv_bfloat16*>(aux)[off] = __float2bfloat16_rn(v);
  else reinterpret_cast<float*>(aux)[off] = b2_tf32_small(v);
}

// C (E, r, r) -> shared memory, row pitch r + 1
__device__ __forceinline__ void cm_load_c(const float* __restrict__ C, float* sC, int r, int E) {
  const int n = E * r * r;
  for (int t = threadIdx.x; t < n; t += blockDim.x) sC[(t / r) * (r + 1) + t % r] = __ldg(C + t);
}

// One row's h (into sh), v (registers) and softmax weights (into sp).  Returns nothing; the warp is
// synchronised on exit.
__device__ __forceinline__ void cm_row_forward(const float* __restrict__ prow, const float* sC, float* sh,
                                               float* sp, int r, int E, float (&v)[CM_MAX_COLS]) {
  const int lane = threadIdx.x & 31, R = E * r;
#pragma unroll
  for (int i = 0; i < CM_MAX_COLS; ++i) {
    const int c = lane + 32 * i;
    if (c < R) sh[c] = tanhf(__ldg(prow + c));
  }
  // softmax over the E gate logits (columns R .. R+E-1 of P)
  float m = -INFINITY;
  for (int e = lane; e < E; e += 32) m = fmaxf(m, __ldg(prow + R + e));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  float s = 0.f;
  for (int e = lane; e < E; e += 32) {
    const float x = expf(__ldg(prow + R + e) - m);
    sp[e] = x;
    s += x;
  }
  s = b2_warp_sum(s);
  __syncwarp();
  const float inv = 1.f / s;
  for (int e = lane; e < E; e += 32) sp[e] *= inv;
#pragma unroll
  for (int i = 0; i < CM_MAX_COLS; ++i) {
    const int c = lane + 32 * i;
    float u = 0.f;
    if (c < R) {
      const int e = c / r;
      const float* crow = sC + c * (r + 1);
      const float* he = sh + e * r;
      for (int k = 0; k < r; ++k) u = fmaf(crow[k], he[k], u);
    }
    v[i] = tanhf(u);
  }
  __syncwarp();
}

__global__ void __launch_bounds__(CM_THREADS)
crossmix_fwd_kernel(const float* __restrict__ P, const float* __restrict__ C, int64_t batch, int r, int E,
                    float* __restrict__ A2, void* a2_aux, int aux_dtype, int64_t ld_aux) {
  extern __shared__ float sm[];
  const int R = E * r, n1 = cm_n1(r, E), k2 = cm_k2(r, E);
  float* sC = sm;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float* sh = sC + R * (r + 1) + warp * (R + E);
  float* sp = sh + R;
  b2_pdl_wait();
  cm_load_c(C, sC, r, E);
  __syncthreads();
  for (int64_t row = (int64_t) blockIdx.x * CM_WARPS + warp; row < batch; row += (int64_t) gridDim.x * CM_WARPS) {
    float v[CM_MAX_COLS];
    cm_row_forward(P + row * n1, sC, sh, sp, r, E, v);
#pragma unroll
    for (int i = 0; i < CM_MAX_COLS; ++i) {
      const int c = lane + 32 * i;
      if (c < k2) {
        const float a = (c < R) ? sp[c / r] * v[i] : 0.f;
        A2[row * k2 + c] = a;
        if (a2_aux) cm_store_aux(a2_aux, aux_dtype, row * ld_aux + c, a);
      }
    }
    __syncwarp();
  }
  b2_pdl_trigger();
}

// Backward of the row kernel.  Per row, from P (h, v, p recomputed) and dA2:
//   dv = p_e dA2_e,  dp_e = <dA2_e, v_e>,  dlogit_e = p_e (dp_e - sum_f p_f dp_f),
//   dz = dv (1 - v^2),  dh_e = dz_e C_e,  dP = dh (1 - h^2);   dA1 = [dP | dlogit | 0].
// dC_e = sum_rows dz_e (x) h_e: the warps stage h and dz of CM_TILE_ROWS rows in shared memory, then every
// thread adds its own dC elements over the tile into a CTA-private copy (no shared atomics); at the end one
// global float atomic per element and CTA (dC must be zero on entry).
__global__ void __launch_bounds__(CM_THREADS)
crossmix_bwd_kernel(const float* __restrict__ P, const float* __restrict__ C, const float* __restrict__ dA2,
                    int64_t batch, int r, int E, float* __restrict__ dA1, void* da1_aux, int aux_dtype,
                    int64_t ld_aux, float* __restrict__ dC) {
  extern __shared__ float sm[];
  const int R = E * r, n1 = cm_n1(r, E), k2 = cm_k2(r, E), RR = R * r;
  float* sC = sm;                                  // R * (r + 1)
  float* sdC = sC + R * (r + 1);                   // R * r
  float* sH = sdC + RR;                            // CM_TILE_ROWS * R
  float* sZ = sH + CM_TILE_ROWS * R;               // CM_TILE_ROWS * R
  float* sw = sZ + CM_TILE_ROWS * R;               // per warp: p (E), dp (E), scratch (R)
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float* sp = sw + warp * (2 * E + R);
  float* sdp = sp + E;
  float* st = sdp + E;
  for (int t = threadIdx.x; t < RR; t += blockDim.x) sdC[t] = 0.f;
  b2_pdl_wait();
  cm_load_c(C, sC, r, E);
  __syncthreads();
  const int64_t tiles = (batch + CM_TILE_ROWS - 1) / CM_TILE_ROWS;
  for (int64_t tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
    const int64_t row0 = tile * CM_TILE_ROWS;
    const int nrows = (int) min((int64_t) CM_TILE_ROWS, batch - row0);
    for (int t = warp; t < nrows; t += CM_WARPS) {
      float* sh = sH + t * R;
      float* sz = sZ + t * R;
      const int64_t row = row0 + t;
      float v[CM_MAX_COLS], g[CM_MAX_COLS];
      cm_row_forward(P + row * n1, sC, sh, sp, r, E, v);
#pragma unroll
      for (int i = 0; i < CM_MAX_COLS; ++i) {
        const int c = lane + 32 * i;
        g[i] = (c < R) ? __ldg(dA2 + row * k2 + c) : 0.f;
        if (c < R) st[c] = g[i] * v[i];
      }
      __syncwarp();
      float pd = 0.f;
      for (int e = lane; e < E; e += 32) {
        float dp = 0.f;
        for (int j = 0; j < r; ++j) dp += st[e * r + j];
        sdp[e] = dp;
        pd = fmaf(sp[e], dp, pd);
      }
      pd = b2_warp_sum(pd);
      __syncwarp();
      float* drow = dA1 + row * n1;
      for (int e = lane; e < n1 - R; e += 32) {
        const float dl = (e < E) ? sp[e] * (sdp[e] - pd) : 0.f;
        drow[R + e] = dl;
        if (da1_aux) cm_store_aux(da1_aux, aux_dtype, row * ld_aux + R + e, dl);
      }
#pragma unroll
      for (int i = 0; i < CM_MAX_COLS; ++i) {
        const int c = lane + 32 * i;
        if (c < R) sz[c] = sp[c / r] * g[i] * (1.f - v[i] * v[i]);
      }
      __syncwarp();
#pragma unroll
      for (int i = 0; i < CM_MAX_COLS; ++i) {
        const int c = lane + 32 * i;
        if (c < R) {
          const int e = c / r, k = c - e * r;
          const float* ccol = sC + e * r * (r + 1) + k;
          const float* ze = sz + e * r;
          float dh = 0.f;
          for (int j = 0; j < r; ++j) dh = fmaf(ze[j], ccol[j * (r + 1)], dh);
          const float h = sh[c];
          const float dp = dh * (1.f - h * h);
          drow[c] = dp;
          if (da1_aux) cm_store_aux(da1_aux, aux_dtype, row * ld_aux + c, dp);
        }
      }
      __syncwarp();
    }
    __syncthreads();
    // dC[e, j, k] += sum_t dz[t, e*r+j] * h[t, e*r+k]
    for (int idx = threadIdx.x; idx < RR; idx += blockDim.x) {
      const int ej = idx / r, e = ej / r, k = idx - ej * r;
      float s = 0.f;
      for (int t = 0; t < nrows; ++t) s = fmaf(sZ[t * R + ej], sH[t * R + e * r + k], s);
      sdC[idx] += s;
    }
    __syncthreads();
  }
  b2_pdl_trigger();
  for (int t = threadIdx.x; t < RR; t += blockDim.x)
    if (sdC[t] != 0.f) b2_red_add(dC + t, sdC[t]);
}

// W1 (N1, d): row e*r+j = V[e, :, j], row E*r+e = G[e, :], zero rows after;  W2 (d, K2): W2[n, e*r+j] = U[e, n, j].
__global__ void __launch_bounds__(256)
crossmix_pack_kernel(const float* __restrict__ U, const float* __restrict__ V, const float* __restrict__ G, int d,
                     int r, int E, float* __restrict__ W1, float* __restrict__ W2) {
  const int R = E * r, n1 = cm_n1(r, E), k2 = cm_k2(r, E);
  const int64_t n_w1 = (int64_t) n1 * d, total = n_w1 + (int64_t) d * k2;
  b2_pdl_wait();
  for (int64_t t = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (int64_t) gridDim.x * blockDim.x) {
    if (t < n_w1) {
      const int row = (int) (t / d), n = (int) (t - (int64_t) row * d);
      float w = 0.f;
      if (row < R) w = __ldg(V + ((int64_t) (row / r) * d + n) * r + row % r);
      else if (row < R + E) w = __ldg(G + (int64_t) (row - R) * d + n);
      W1[t] = w;
    } else {
      const int64_t u = t - n_w1;
      const int n = (int) (u / k2), c = (int) (u - (int64_t) n * k2);
      W2[u] = (c < R) ? __ldg(U + ((int64_t) (c / r) * d + n) * r + c % r) : 0.f;
    }
  }
  b2_pdl_trigger();
}

// gV[e, n, j] = dW1[e*r+j, n], gG[e, n] = dW1[E*r+e, n], gU[e, n, j] = dW2[n, e*r+j]   ("=")
__global__ void __launch_bounds__(256)
crossmix_unpack_kernel(const float* __restrict__ dW1, const float* __restrict__ dW2, int d, int r, int E,
                       float* __restrict__ gU, float* __restrict__ gV, float* __restrict__ gG) {
  const int R = E * r, k2 = cm_k2(r, E);
  const int64_t n_uv = (int64_t) R * d, total = 2 * n_uv + (int64_t) E * d;
  b2_pdl_wait();
  for (int64_t t = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (int64_t) gridDim.x * blockDim.x) {
    if (t < 2 * n_uv) {
      const int64_t u = t < n_uv ? t : t - n_uv;     // (e, n, j) of U / V
      const int j = (int) (u % r), n = (int) ((u / r) % d), e = (int) (u / ((int64_t) r * d));
      if (t < n_uv) gU[u] = __ldg(dW2 + (int64_t) n * k2 + e * r + j);
      else gV[u] = __ldg(dW1 + (int64_t) (e * r + j) * d + n);
    } else {
      const int64_t u = t - 2 * n_uv;
      gG[u] = __ldg(dW1 + (int64_t) R * d + u);
    }
  }
  b2_pdl_trigger();
}

// ---------------------------------------------------------------------------------
// Host side
// ---------------------------------------------------------------------------------
static int cm_check_shape(int r, int E) {
  B2_REQUIRE(r >= 1 && r <= B2_CROSSMIX_MAX_RANK, "low_rank %d outside [1, %d]", r, B2_CROSSMIX_MAX_RANK);
  B2_REQUIRE(E >= 1 && (int64_t) E * r <= B2_CROSSMIX_MAX_COLS,
             "num_experts * low_rank = %lld outside [1, %d]", (long long) E * r, B2_CROSSMIX_MAX_COLS);
  return B2_OK;
}

static int cm_check_aux(const void* aux, int aux_dtype, int64_t ld_aux, int width) {
  if (aux == nullptr) return B2_OK;
  B2_REQUIRE(aux_dtype == B2_F32 || aux_dtype == B2_BF16, "aux_dtype must be B2_F32 or B2_BF16");
  B2_REQUIRE(ld_aux >= width, "ld_aux %lld < row width %d", (long long) ld_aux, width);
  return B2_OK;
}

static int cm_grid(int64_t blocks, int per_sm) {
  const int64_t cap = (int64_t) B2_NUM_SMS * per_sm;
  return (int) (blocks < 1 ? 1 : (blocks > cap ? cap : blocks));
}

static size_t cm_fwd_smem(int r, int E) {
  const int R = E * r;
  return sizeof(float) * ((size_t) R * (r + 1) + (size_t) CM_WARPS * (R + E));
}

static size_t cm_bwd_smem(int r, int E) {
  const int R = E * r;
  return sizeof(float) * ((size_t) R * (r + 1) + (size_t) R * r + 2 * (size_t) CM_TILE_ROWS * R +
                          (size_t) CM_WARPS * (2 * E + R));
}

extern "C" B2_API int b2_crossmix_pack(const float* U, const float* V, const float* G, int d, int r, int E,
                                       float* W1, float* W2, void* stream) {
  B2_REQUIRE(U && V && G && W1 && W2, "NULL pointer");
  B2_REQUIRE(d >= 1, "in_features %d < 1", d);
  if (int rc = cm_check_shape(r, E)) return rc;
  const int64_t total = (int64_t) cm_n1(r, E) * d + (int64_t) d * cm_k2(r, E);
  B2_LAUNCH(crossmix_pack_kernel, cm_grid(b2_ceil_div(total, 256), 8), 256, 0, (cudaStream_t) stream,
            U, V, G, d, r, E, W1, W2);
  B2_CUDA_LAUNCH_CHECK("b2_crossmix_pack");
  return B2_OK;
}

extern "C" B2_API int b2_crossmix_fwd(const float* P, const float* C, int64_t batch, int r, int E, float* A2,
                                      void* a2_aux, int aux_dtype, int64_t ld_aux, void* stream) {
  B2_REQUIRE(P && C && A2, "NULL pointer");
  B2_REQUIRE(batch >= 0, "negative batch");
  if (int rc = cm_check_shape(r, E)) return rc;
  if (int rc = cm_check_aux(a2_aux, aux_dtype, ld_aux, cm_k2(r, E))) return rc;
  if (batch == 0) return B2_OK;
  const size_t smem = cm_fwd_smem(r, E);
  if (smem > 48 * 1024)
    cudaFuncSetAttribute(crossmix_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) smem);
  B2_LAUNCH(crossmix_fwd_kernel, cm_grid(b2_ceil_div(batch, CM_WARPS), 4), CM_THREADS, smem,
            (cudaStream_t) stream, P, C, batch, r, E, A2, a2_aux, aux_dtype, ld_aux);
  B2_CUDA_LAUNCH_CHECK("b2_crossmix_fwd");
  return B2_OK;
}

extern "C" B2_API int b2_crossmix_bwd(const float* P, const float* C, const float* dA2, int64_t batch, int r, int E,
                                      float* dA1, void* da1_aux, int aux_dtype, int64_t ld_aux, float* dC,
                                      void* stream) {
  B2_REQUIRE(P && C && dA2 && dA1 && dC, "NULL pointer");
  B2_REQUIRE(batch >= 0, "negative batch");
  if (int rc = cm_check_shape(r, E)) return rc;
  if (int rc = cm_check_aux(da1_aux, aux_dtype, ld_aux, cm_n1(r, E))) return rc;
  if (batch == 0) return B2_OK;
  const size_t smem = cm_bwd_smem(r, E);
  if (smem > 48 * 1024)
    cudaFuncSetAttribute(crossmix_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) smem);
  // at most two CTAs per SM: each one ends with E*r*r global atomics
  B2_LAUNCH(crossmix_bwd_kernel, cm_grid(b2_ceil_div(batch, CM_TILE_ROWS), 2), CM_THREADS, smem,
            (cudaStream_t) stream, P, C, dA2, batch, r, E, dA1, da1_aux, aux_dtype, ld_aux, dC);
  B2_CUDA_LAUNCH_CHECK("b2_crossmix_bwd");
  return B2_OK;
}

extern "C" B2_API int b2_crossmix_unpack(const float* dW1, const float* dW2, int d, int r, int E, float* gU,
                                         float* gV, float* gG, void* stream) {
  B2_REQUIRE(dW1 && dW2 && gU && gV && gG, "NULL pointer");
  B2_REQUIRE(d >= 1, "in_features %d < 1", d);
  if (int rc = cm_check_shape(r, E)) return rc;
  const int64_t total = 2 * (int64_t) E * r * d + (int64_t) E * d;
  B2_LAUNCH(crossmix_unpack_kernel, cm_grid(b2_ceil_div(total, 256), 8), 256, 0, (cudaStream_t) stream,
            dW1, dW2, d, r, E, gU, gV, gG);
  B2_CUDA_LAUNCH_CHECK("b2_crossmix_unpack");
  return B2_OK;
}

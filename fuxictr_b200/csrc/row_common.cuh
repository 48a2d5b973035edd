// row_common.cuh — the layout and the loads/stores the elementwise row kernels share (gdcn.cu, finalmlp.cu).
//
// A CTA is ty_n rows of tx_n column slots (rk_plan); a slot owns VW consecutive columns (4 on the float4 path, 1 on
// the scalar one) and walks the batch rows with a grid stride.  Column sums over the batch (bias and broadcast-gate
// gradients) are taken per slot in registers, then over the ty_n rows of the CTA in shared memory (rk_cta_colsum),
// and added with one float atomic per column and CTA.
#pragma once
#include "b2_common.cuh"

#define RK_THREADS 256

template <int VW>
__device__ __forceinline__ void rk_load(const float* p, float (&v)[VW]) {
  if constexpr (VW == 4) {
    const float4 t = __ldg(reinterpret_cast<const float4*>(p));
    v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
  } else {
    v[0] = __ldg(p);
  }
}

template <int VW>
__device__ __forceinline__ void rk_store(float* p, const float (&v)[VW]) {
  if constexpr (VW == 4) *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]);
  else p[0] = v[0];
}

// The GEMM-operand copy of VW values at aux + off: bf16 rounding or 3xTF32 small part (as b2_crossmix_fwd).
template <int VW>
__device__ __forceinline__ void rk_store_aux(void* aux, int aux_dtype, int64_t off, const float (&v)[VW]) {
  if (aux_dtype == B2_BF16) {
    __nv_bfloat16* a = reinterpret_cast<__nv_bfloat16*>(aux) + off;
    if constexpr (VW == 4) {
      __nv_bfloat162 lo = __floats2bfloat162_rn(v[0], v[1]), hi = __floats2bfloat162_rn(v[2], v[3]);
      uint2 w;
      w.x = *reinterpret_cast<uint32_t*>(&lo);
      w.y = *reinterpret_cast<uint32_t*>(&hi);
      *reinterpret_cast<uint2*>(a) = w;
    } else {
      a[0] = __float2bfloat16_rn(v[0]);
    }
  } else {
    float s[VW];
#pragma unroll
    for (int k = 0; k < VW; ++k) s[k] = b2_tf32_small(v[k]);
    rk_store<VW>(reinterpret_cast<float*>(aux) + off, s);
  }
}

// Sum of acc over the ty_n rows of the CTA for each of the slot's VW columns, valid in the ty == 0 threads.  `red` is
// __shared__ float[RK_THREADS * VW]; every thread of the CTA calls this.
template <int VW>
__device__ __forceinline__ void rk_cta_colsum(float* red, int tx, int tx_n, int ty_n, float (&acc)[VW]) {
#pragma unroll
  for (int k = 0; k < VW; ++k) red[threadIdx.x * VW + k] = acc[k];
  __syncthreads();
#pragma unroll
  for (int k = 0; k < VW; ++k) {
    float s = 0.f;
    for (int y = 0; y < ty_n; ++y) s += red[(y * tx_n + tx) * VW + k];
    acc[k] = s;
  }
}

static inline int rk_check_aux(const void* aux, int aux_dtype, int64_t ld_aux, int width) {
  if (aux == nullptr) return B2_OK;
  B2_REQUIRE(aux_dtype == B2_F32 || aux_dtype == B2_BF16, "aux_dtype must be B2_F32 or B2_BF16");
  B2_REQUIRE(ld_aux >= width, "ld_aux %lld < row width %d", (long long) ld_aux, width);
  return B2_OK;
}

static inline bool rk_al16(const void* p) { return p == nullptr || ((uintptr_t) p & 15) == 0; }

// float4 path: d % 4 == 0, every row 16-byte aligned, the auxiliary rows 16 (fp32) / 8 (bf16) bytes
static inline bool rk_vec(int d, const void* const* ptrs, int n, const void* aux, int aux_dtype, int64_t ld_aux) {
  if (d % 4 != 0) return false;
  for (int i = 0; i < n; ++i)
    if (!rk_al16(ptrs[i])) return false;
  if (aux == nullptr) return true;
  const uintptr_t align = aux_dtype == B2_BF16 ? 8 : 16;
  return ld_aux % 4 == 0 && ((uintptr_t) aux & (align - 1)) == 0;
}

// The columns split into gy chunks of at most RK_THREADS slots; a CTA is ty_n rows of tx_n slots (tx_n: a chunk
// rounded up to a warp), at most per_sm CTAs per SM over the batch.
struct rk_grid {
  dim3 grid;
  int threads, tx_n;
};

static inline rk_grid rk_plan(int64_t batch, int d, int vw, int per_sm) {
  const int cols = (d + vw - 1) / vw;
  const int gy = (cols + RK_THREADS - 1) / RK_THREADS;
  const int tx_n = ((cols + gy - 1) / gy + 31) / 32 * 32;
  const int ty_n = RK_THREADS / tx_n;
  int64_t cap = (int64_t) B2_NUM_SMS * per_sm / gy, gx = b2_ceil_div(batch, ty_n);
  cap = cap < 1 ? 1 : cap;
  gx = gx < 1 ? 1 : (gx > cap ? cap : gx);
  return {dim3((unsigned) gx, (unsigned) gy), tx_n * ty_n, tx_n};
}

// b2_common.cuh — shared device/host helpers for the sm_90a kernels.
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <stdio.h>
#include <stdarg.h>

#include "../../include/fuxictr_b200.h"

#define B2_NUM_SMS 132  // H100 SXM: 132 SMs; grids are sized in multiples of this

// ---- per-thread last-error string (no C++ exceptions cross the ABI) --------
extern thread_local char b2_tls_error[512];
int b2_fail(int code, const char* fmt, ...);

#define B2_REQUIRE(cond, ...)                                 \
  do {                                                        \
    if (!(cond)) return b2_fail(B2_E_INVALID, __VA_ARGS__);   \
  } while (0)

#define B2_CUDA_LAUNCH_CHECK(name)                                                     \
  do {                                                                                 \
    cudaError_t e__ = cudaGetLastError();                                              \
    if (e__ != cudaSuccess)                                                            \
      return b2_fail(B2_E_CUDA, "%s: launch failed: %s", name, cudaGetErrorString(e__)); \
  } while (0)

static inline int64_t b2_ceil_div(int64_t a, int64_t b) { return (a + b - 1) / b; }

// ---- programmatic dependent launch (on by default; B2_PDL=0 launches plainly) --------------------
// The step is a chain of ~45 short kernels; with PDL a kernel's CTAs are scheduled while its predecessor
// drains and sit at griddepcontrol.wait (which returns only when the predecessor has COMPLETED and its
// writes are visible), so the launch latency — and, for the GEMM, the barrier/tensormap prologue —
// overlaps the predecessor's tail.  Captured into CUDA graphs as programmatic dependency edges.
#include <stdlib.h>
static inline bool b2_pdl_on() {
  static const bool on = [] { const char* e = getenv("B2_PDL"); return e == nullptr || atoi(e) != 0; }();
  return on;
}
#define B2_LAUNCH(kernel, grid, block, smem, st, ...)                                             \
  do {                                                                                              \
    if (b2_pdl_on()) {                                                                              \
      cudaLaunchConfig_t cfg__ = {};                                                                \
      cfg__.gridDim = dim3(grid); cfg__.blockDim = dim3(block);                                     \
      cfg__.dynamicSmemBytes = (size_t) (smem); cfg__.stream = (st);                                \
      cudaLaunchAttribute at__[1];                                                                  \
      at__[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;                              \
      at__[0].val.programmaticStreamSerializationAllowed = 1;                                       \
      cfg__.attrs = at__; cfg__.numAttrs = 1;                                                       \
      cudaLaunchKernelEx(&cfg__, kernel, __VA_ARGS__);                                              \
    } else {                                                                                        \
      kernel<<<grid, block, smem, st>>>(__VA_ARGS__);                                               \
    }                                                                                               \
  } while (0)

// ---- device helpers ----------------------------------------------------------
// No-ops for a kernel launched without the PDL attribute.
__device__ __forceinline__ void b2_pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void b2_pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ float b2_warp_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 16);
  v += __shfl_xor_sync(0xffffffffu, v, 8);
  v += __shfl_xor_sync(0xffffffffu, v, 4);
  v += __shfl_xor_sync(0xffffffffu, v, 2);
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  return v;
}

// Block-wide sum; `red` is __shared__ float[32]. Result valid in all threads.
__device__ __forceinline__ float b2_block_sum(float v, float* red) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  v = b2_warp_sum(v);
  __syncthreads();
  if (lane == 0) red[warp] = v;
  __syncthreads();
  const int nwarps = (blockDim.x + 31) >> 5;
  float t = (threadIdx.x < nwarps) ? red[threadIdx.x] : 0.f;
  if (warp == 0) {
    t = b2_warp_sum(t);
    if (lane == 0) red[0] = t;
  }
  __syncthreads();
  return red[0];
}

// Streaming 128-bit loads/stores that do not pollute L1 (one-touch data).
__device__ __forceinline__ float4 b2_ldg_stream(const float4* p) {
  float4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w)
               : "l"(p));
  return r;
}
__device__ __forceinline__ void b2_stg_stream(float4* p, const float4& v) {
  asm volatile("st.global.L1::no_allocate.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(v.x),
               "f"(v.y), "f"(v.z), "f"(v.w)
               : "memory");
}

// Vector reductions to global memory (sm_90+): one 16-byte / 8-byte atomic per lane.
__device__ __forceinline__ void b2_red_add_v4(float* p, const float4& v) {
  asm volatile("red.global.add.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(v.x), "f"(v.y),
               "f"(v.z), "f"(v.w)
               : "memory");
}
__device__ __forceinline__ void b2_red_add_v2(float* p, float x, float y) {
  asm volatile("red.global.add.v2.f32 [%0], {%1,%2};" ::"l"(p), "f"(x), "f"(y) : "memory");
}
__device__ __forceinline__ void b2_red_add(float* p, float x) {
  asm volatile("red.global.add.f32 [%0], %1;" ::"l"(p), "f"(x) : "memory");
}

// 3xTF32 split: small(x) = rna_tf32(x - big(x)), big(x) = x with the 13 low mantissa bits cleared (what
// the GEMM feeds the tensor core as the tf32 operand).  x - big(x) is exact; rounding it to a tf32-representable
// value HERE (round-to-nearest) makes the hardware truncation of the small operand a no-op, so the
// residual of the split is unbiased instead of always toward zero.
__device__ __forceinline__ float b2_tf32_small(float v) {
  const float big = __uint_as_float(__float_as_uint(v) & 0xffffe000u);
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(v - big));
  return __uint_as_float(r);
}

// Index fetch with the reference's `.long()` semantics (feature_embedding.py:284):
// float64 ids are truncated toward zero.
template <typename IdxT>
__device__ __forceinline__ int64_t b2_load_index(const void* base, int64_t off) {
  return (int64_t) reinterpret_cast<const IdxT*>(base)[off];
}
template <>
__device__ __forceinline__ int64_t b2_load_index<double>(const void* base, int64_t off) {
  return __double2ll_rz(reinterpret_cast<const double*>(base)[off]);
}

// lsh_common.cuh — the SimHash code word shared by ETA / SDIM (lsh.cu) and MIRRN (mirrn.cu).
// Bit j of a row v is v . R[:, j] > 0, an fp32 FMA over the d columns in ascending order.
#pragma once
#include "b2_common.cuh"

// Code word w (bits [32 w, min(32 w + 32, nbits))) of row v under R (d rows of pitch ldr; column c0 + j is bit j).
// kShared: v lies in shared memory (read with plain loads) instead of read-only global memory.
template <bool kShared = false>
__device__ __forceinline__ uint32_t lsh_word(const float* __restrict__ v, const float* sR, int d, int ldr, int c0,
                                             int nbits) {
  float acc[32];
#pragma unroll
  for (int j = 0; j < 32; ++j) acc[j] = 0.f;
  for (int i = 0; i < d; ++i) {
    const float vi = kShared ? v[i] : __ldg(v + i);
    const float* r = sR + i * ldr + c0;
#pragma unroll
    for (int j = 0; j < 32; ++j)
      if (j < nbits) acc[j] = fmaf(vi, r[j], acc[j]);
  }
  uint32_t code = 0;
#pragma unroll
  for (int j = 0; j < 32; ++j)
    if (j < nbits && acc[j] > 0.f) code |= 1u << j;
  return code;
}

__device__ __forceinline__ void lsh_stage(const float* __restrict__ R, int n, float* sR) {
  for (int e = threadIdx.x; e < n; e += blockDim.x) sR[e] = __ldg(R + e);
}

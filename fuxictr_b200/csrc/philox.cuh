// philox.cuh — Philox4x32-10 (Salmon et al., "Parallel random numbers: as easy as 1, 2, 3", SC 2011) and the
// dropout mask built on it, shared by every kernel that applies or regenerates a dropout mask.
//
// keep(seed, offset, m, n) for an element (m, n) of an (M, N) layer output, probability p of dropping:
//   i = m * N + n                       (64-bit element index of the row-major, unpadded matrix)
//   r = Philox4x32-10(counter = {lo(i >> 2), hi(i >> 2), lo(offset), hi(offset)}, key = {lo(seed), hi(seed)})
//   keep  <=>  r[i & 3] < thresh,   thresh = min(round((1 - p) * 2^32), 2^32 - 1) (computed once on the host)
// so one Philox call serves a group of 4 consecutive elements, and a 16-byte row segment that starts on a group
// needs one call.  `offset` is the forward's snapshot offset plus the ordinal of the dropout layer in its chain
// (b2_dropout_rng_take advances the state by the chain's dropout layers), so no two (forward, layer, element)
// triples share a counter.  The CPU tests restate this in numpy.
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define B2_HD __host__ __device__ __forceinline__
#else
#define B2_HD inline
#endif

struct b2_u32x4 { uint32_t v[4]; };

B2_HD uint32_t b2_mulhilo(uint32_t a, uint32_t b, uint32_t* hi) {
#if defined(__CUDA_ARCH__)
  *hi = __umulhi(a, b);
  return a * b;
#else
  const uint64_t p = (uint64_t) a * b;
  *hi = (uint32_t) (p >> 32);
  return (uint32_t) p;
#endif
}

B2_HD b2_u32x4 b2_philox4x32_10(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3, uint32_t k0, uint32_t k1) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    uint32_t hi0, hi1;
    const uint32_t lo0 = b2_mulhilo(0xD2511F53u, c0, &hi0);
    const uint32_t lo1 = b2_mulhilo(0xCD9E8D57u, c2, &hi1);
    const uint32_t n0 = hi1 ^ c1 ^ k0, n2 = hi0 ^ c3 ^ k1;
    c0 = n0; c1 = lo1; c2 = n2; c3 = lo0;
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
  b2_u32x4 r;
  r.v[0] = c0; r.v[1] = c1; r.v[2] = c2; r.v[3] = c3;
  return r;
}

// Word j of r by selects, not by a dynamic index (which would put r in local memory).
B2_HD uint32_t b2_word(const b2_u32x4& r, uint32_t j) {
  return j == 0 ? r.v[0] : j == 1 ? r.v[1] : j == 2 ? r.v[2] : r.v[3];
}

// The four draws of element group g (elements 4g .. 4g + 3) under `seed` and counter offset `off`.
B2_HD b2_u32x4 b2_drop_group(uint64_t seed, uint64_t off, uint64_t g) {
  return b2_philox4x32_10((uint32_t) g, (uint32_t) (g >> 32), (uint32_t) off, (uint32_t) (off >> 32),
                          (uint32_t) seed, (uint32_t) (seed >> 32));
}

// keep(element i): one Philox call; the elementwise kernels use it, the GEMM epilogue shares calls per group.
B2_HD bool b2_drop_keep(uint64_t seed, uint64_t off, uint64_t i, uint32_t thresh) {
  return b2_word(b2_drop_group(seed, off, i >> 2), (uint32_t) (i & 3)) < thresh;
}

// Keep bits (bit e for element i0 + e, e < nv <= 4) of nv consecutive elements: one Philox call when they lie in
// one group, two when they straddle a group boundary.
B2_HD uint32_t b2_drop_keep4(uint64_t seed, uint64_t off, uint64_t i0, int nv, uint32_t thresh) {
  const uint64_t g0 = i0 >> 2, g1 = (i0 + (uint64_t) (nv > 0 ? nv - 1 : 0)) >> 2;
  const b2_u32x4 r0 = b2_drop_group(seed, off, g0);
  uint32_t bits = 0;
  if (g1 == g0 && (i0 & 3) == 0) {      // the aligned case of every 16-byte segment of a width % 4 == 0 output
#pragma unroll
    for (int e = 0; e < 4; ++e)
      if (e < nv && r0.v[e] < thresh) bits |= 1u << e;
    return bits;
  }
  b2_u32x4 r1 = r0;
  if (g1 != g0) r1 = b2_drop_group(seed, off, g1);
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    const uint64_t i = i0 + e;
    const uint32_t j = (uint32_t) (i & 3), u0 = b2_word(r0, j), u1 = b2_word(r1, j);
    const uint32_t u = (i >> 2) == g0 ? u0 : u1;
    if (e < nv && u < thresh) bits |= 1u << e;
  }
  return bits;
}

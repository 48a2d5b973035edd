// topk_select.cuh — one CTA selects the k largest of n fp32 keys held in shared memory (SIM and TWIN, topk_retrieval.cu).
//
// The project's order: descending by value, ties to the lower position, output sorted by (value desc, position asc).
// -0.0 and +0.0 are the same key (SIM's masked negative scores come out as -0.0 and must tie with +0.0).  torch.topk
// leaves tie order unspecified, so this rule is the project's own.
// Method: the keys are mapped to orderable uint32 (b2_topk_key); a radix select over four 8-bit digits finds the k-th
// largest key T and how many of the chosen keys equal it; the warps then compact, in ascending position, every key
// above T and the lowest-positioned keys equal to T; the k chosen are finally ranked by (key desc, position asc).
// Every step is deterministic: the histogram counts are order-free and the compaction and ranking are exact.
#pragma once
#include "b2_common.cuh"

#define B2_TOPK_SELECT_MAX_K 256

struct B2TopkSmem {
  uint32_t hist[256];
  uint32_t tkey[B2_TOPK_SELECT_MAX_K];
  int32_t tpos[B2_TOPK_SELECT_MAX_K];
  int32_t wcnt[32][2];
  int32_t digit, above;
};

// A larger float gives a larger key; -0.0 maps to +0.0's key.
__device__ __forceinline__ uint32_t b2_topk_key(float v) {
  uint32_t u = __float_as_uint(v);
  if ((u & 0x7fffffffu) == 0) u = 0;
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

// The float of a key (+0.0 for either zero).
__device__ __forceinline__ float b2_topk_value(uint32_t key) {
  return __uint_as_float((key & 0x80000000u) ? (key & 0x7fffffffu) : ~key);
}

// All threads of the CTA call it; blockDim.x a multiple of 32.  key (n) in shared memory, 1 <= k <= min(n,
// B2_TOPK_SELECT_MAX_K).  sel (k, shared) receives the chosen positions in the project's order.  Ends synchronised.
__device__ void b2_topk_select(const uint32_t* key, int n, int k, int32_t* sel, B2TopkSmem& s) {
  const int t = threadIdx.x, lane = t & 31, w = t >> 5, nw = blockDim.x >> 5;
  uint32_t prefix = 0, pmask = 0;
  int need = k;                                          // how many of the keys matching prefix are still wanted
  for (int shift = 24; shift >= 0; shift -= 8) {
    for (int e = t; e < 256; e += blockDim.x) s.hist[e] = 0;
    __syncthreads();
    for (int i = t; i < n; i += blockDim.x) {
      const uint32_t u = key[i];
      if ((u & pmask) == prefix) atomicAdd(&s.hist[(u >> shift) & 255u], 1u);
    }
    __syncthreads();
    if (w == 0) {                                        // lane j holds bins 255 - 8 j down to 248 - 8 j
      int c = 0;
#pragma unroll
      for (int j = 0; j < 8; ++j) c += (int) s.hist[255 - 8 * lane - j];
      int incl = c;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int v = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += v;
      }
      const int excl = incl - c;
      if (excl < need && need <= incl) {
        int run = excl;
        for (int j = 0; j < 8; ++j) {
          const int b = 255 - 8 * lane - j, h = (int) s.hist[b];
          if (run + h >= need) {
            s.digit = b;
            s.above = run;
            break;
          }
          run += h;
        }
      }
    }
    __syncthreads();
    prefix |= (uint32_t) s.digit << shift;
    pmask |= 255u << shift;
    need -= s.above;
  }
  const uint32_t T = prefix;                              // the k-th largest key; `need` of the chosen equal it
  const int seg = (((n + nw - 1) / nw) + 31) & ~31;
  const int lo = min(n, w * seg), hi = min(n, lo + seg);
  const uint32_t lt = (1u << lane) - 1u;
  int gt = 0, eq = 0;
  for (int base = lo; base < hi; base += 32) {
    const int i = base + lane;
    const uint32_t u = i < hi ? key[i] : 0u;
    gt += __popc(__ballot_sync(0xffffffffu, i < hi && u > T));
    eq += __popc(__ballot_sync(0xffffffffu, i < hi && u == T));
  }
  if (lane == 0) {
    s.wcnt[w][0] = gt;
    s.wcnt[w][1] = eq;
  }
  __syncthreads();
  gt = eq = 0;
  for (int v = 0; v < w; ++v) {
    gt += s.wcnt[v][0];
    eq += s.wcnt[v][1];
  }
  for (int base = lo; base < hi; base += 32) {
    const int i = base + lane;
    const uint32_t u = i < hi ? key[i] : 0u;
    const bool isgt = i < hi && u > T, iseq = i < hi && u == T;
    const uint32_t bg = __ballot_sync(0xffffffffu, isgt), be = __ballot_sync(0xffffffffu, iseq);
    const int eq_before = eq + __popc(be & lt);
    if (isgt || (iseq && eq_before < need)) {
      const int slot = gt + __popc(bg & lt) + min(eq_before, need);
      s.tkey[slot] = u;
      s.tpos[slot] = i;
    }
    gt += __popc(bg);
    eq += __popc(be);
  }
  __syncthreads();
  for (int a = t; a < k; a += blockDim.x) {              // slots are in ascending position
    const uint32_t u = s.tkey[a];
    int r = 0;
    for (int j = 0; j < k; ++j) {
      const uint32_t v = s.tkey[j];
      r += (v > u) || (v == u && j < a);
    }
    sel[r] = s.tpos[a];
  }
  __syncthreads();
}

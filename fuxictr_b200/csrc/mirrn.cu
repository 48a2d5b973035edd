// mirrn.cu — MIRRN (model_zoo/LongCTR/MIRRN/MIRRN.py): three SimHash retrievals over a long behaviour sequence and
// the FilterLayer2 blocks on what they retrieve, sm_90a.
//
// x is item_feat_emb (B, L + 1, d): positions [0, L) are the history h, position L the target t.  Three queries hash
// against the history: t, the masked mean of h[:, -16:] and the masked mean of all of h.  A mean's code is taken from
// the masked sum: dividing by count + 1e-9 > 0 does not change a projection's sign, and an empty history gives a zero
// vector (all bits 0) either way.  Bit j is x . R[:, j] > 0 in fp32 FMA (lsh_common.cuh), in every matmul mode.  The
// distance to position l is popc(code_l ^ code_q), bits + 1 where mask is 0; each query keeps the k = min(topk, L)
// smallest, ties to the lower position, written in ascending position order (the reference's topk_index.sort(-1)).
// With one rotation set the history is hashed once for all three queries.
//
// FilterLayer2 is LN(dropout(irfft(rfft(u) W)) + u) over the k retrieved rows u.  Its einsum "blnd,ndd->blnd" keeps
// the diagonal of each block, so W is one complex weight a_c + i b_c per channel c = n (d / 4) + j, read from
// complex_weight[n, j, j, :].  A frequency-independent weight makes the filter a_c u + b_c (H u) along the slot axis,
// H the antisymmetric k x k circulant (H u)_t = sum_s h[(t - s) mod k] u_s whose first column h the host builds.  The
// add + dropout + LayerNorm run on b2_bst_addnorm_fwd / _bwd; these kernels do the gather, the filter, the mean over
// the k slots and the backward assembly.  Each kernel waits for its predecessor (programmatic dependent launch)
// before its first read and never triggers its successor early.
#include "b2_common.cuh"
#include "lsh_common.cuh"

#define MIRRN_THREADS 256
#define MIRRN_SHORT 16          // the reference's sequence_emb[:, -16:]

static int mirrn_check(int64_t batch, int L, int d, int k) {
  B2_REQUIRE(d >= 4 && d <= B2_LSH_MAX_DIM && d % 4 == 0,
             "MIRRN: the item width d must be a multiple of 4 in [4, %d], got %d", B2_LSH_MAX_DIM, d);
  B2_REQUIRE(L >= 1 && L <= B2_LSH_MAX_LEN, "MIRRN: the history length L must lie in [1, %d], got %d",
             B2_LSH_MAX_LEN, L);
  B2_REQUIRE(k >= 1 && k <= L && k <= B2_LSH_MAX_TOPK, "MIRRN: k must lie in [1, min(L, %d)], got %d (L = %d)",
             B2_LSH_MAX_TOPK, k, L);
  B2_REQUIRE(batch >= 0, "MIRRN: negative batch %lld", (long long) batch);
  B2_REQUIRE(batch * (L + 1) < ((int64_t) 1 << 31), "MIRRN: batch (L + 1) must stay below 2^31");
  return B2_OK;
}

// ---------------------------------------------------------------------------------------------------------------
// Retrieval
// shared: R (nsets d bits) f32 | part (G 2 d) f32 | qsum (2 d) f32 | hist (3 (bits + 2)) i32 | qcode (3 2) u32 |
//         dist (3 L) u8
__global__ void __launch_bounds__(MIRRN_THREADS)
mirrn_retrieve_kernel(const float* __restrict__ x, const uint8_t* __restrict__ mask, const float* __restrict__ R,
                      int64_t r_stride, int L, int d, int bits, int k, int32_t* __restrict__ topk_pos) {
  extern __shared__ float smem[];
  b2_pdl_wait();
  const int nsets = r_stride ? 3 : 1;
  const int G = blockDim.x / d;
  float* sR = smem;
  float* part = sR + nsets * d * bits;
  float* qsum = part + G * 2 * d;
  int32_t* hist = (int32_t*) (qsum + 2 * d);
  uint32_t* qcode = (uint32_t*) (hist + 3 * (bits + 2));
  uint8_t* dist = (uint8_t*) (qcode + 6);
  const int64_t b = blockIdx.x;
  const int t = threadIdx.x;
  const float* xb = x + b * (int64_t) (L + 1) * d;
  const uint8_t* mb = mask + b * (int64_t) L;
  const int words = (bits + 31) >> 5;
  for (int q = 0; q < nsets; ++q) lsh_stage(R + q * r_stride, d * bits, sR + q * d * bits);
  for (int e = t; e < 3 * (bits + 2); e += blockDim.x) hist[e] = 0;
  // masked sums of the last min(16, L) rows and of all L rows: column t % d, rows t / d mod G, then the G partial
  // sums in a fixed order
  const int g = t / d, c = t - g * d;
  if (g < G) {
    float s16 = 0.f, sall = 0.f;
    for (int l = g; l < L; l += G) {
      if (mb[l]) {
        const float v = xb[(int64_t) l * d + c];
        sall += v;
        if (l >= L - MIRRN_SHORT) s16 += v;
      }
    }
    part[g * 2 * d + c] = s16;
    part[g * 2 * d + d + c] = sall;
  }
  __syncthreads();
  for (int e = t; e < 2 * d; e += blockDim.x) {
    float s = 0.f;
    for (int q = 0; q < G; ++q) s += part[q * 2 * d + e];
    qsum[e] = s;
  }
  __syncthreads();
  if (t < 3 * words) {
    const int q = t / words, w = t - q * words;
    const float* Rq = sR + (nsets > 1 ? q : 0) * d * bits;
    const int nb = min(32, bits - 32 * w);
    qcode[2 * q + w] = q == 0 ? lsh_word(xb + (int64_t) L * d, Rq, d, bits, 32 * w, nb)
                              : lsh_word<true>(qsum + (q - 1) * d, Rq, d, bits, 32 * w, nb);
  }
  __syncthreads();
  uint32_t qc[3][2];
#pragma unroll
  for (int q = 0; q < 3; ++q) {
    qc[q][0] = qcode[2 * q];
    qc[q][1] = words > 1 ? qcode[2 * q + 1] : 0u;
  }
  for (int l = t; l < L; l += blockDim.x) {
    int dl[3] = {bits + 1, bits + 1, bits + 1};
    if (mb[l]) {
      const float* v = xb + (int64_t) l * d;
      uint32_t c0 = 0, c1 = 0;
#pragma unroll
      for (int q = 0; q < 3; ++q) {
        if (q == 0 || nsets > 1) {
          const float* Rq = sR + q * d * bits;
          c0 = lsh_word(v, Rq, d, bits, 0, min(32, bits));
          c1 = words > 1 ? lsh_word(v, Rq, d, bits, 32, bits - 32) : 0u;
        }
        dl[q] = __popc(c0 ^ qc[q][0]) + __popc(c1 ^ qc[q][1]);
      }
    }
#pragma unroll
    for (int q = 0; q < 3; ++q) {
      dist[q * L + l] = (uint8_t) dl[q];
      atomicAdd(hist + q * (bits + 2) + dl[q], 1);
    }
  }
  __syncthreads();
  // warp q selects for query q: every position below the threshold distance D, then the first `need` positions at D
  const int warp = t >> 5, lane = t & 31;
  if (warp < 3) {
    const int32_t* hq = hist + warp * (bits + 2);
    int D = bits + 1, need = k, cum = 0;
    for (int e = 0; e < bits + 2; ++e) {
      const int n = hq[e];
      if (cum + n >= k) {
        D = e;
        need = k - cum;
        break;
      }
      cum += n;
    }
    const uint8_t* dq = dist + warp * L;
    int32_t* out = topk_pos + (b * 3 + warp) * (int64_t) k;
    const uint32_t lt = (1u << lane) - 1u;
    int base = 0;
    for (int c0 = 0; c0 < L && base < k; c0 += 32) {
      const int l = c0 + lane;
      const int dl = l < L ? dq[l] : 255;
      const uint32_t eq = __ballot_sync(0xffffffffu, dl == D);
      const bool keep = dl < D || (dl == D && __popc(eq & lt) < need);
      const uint32_t kb = __ballot_sync(0xffffffffu, keep);
      if (keep) out[base + __popc(kb & lt)] = l;
      base += __popc(kb);
      need -= min(__popc(eq), need);
    }
  }
}

static size_t mirrn_retrieve_smem(int L, int d, int bits, int nsets) {
  const int G = MIRRN_THREADS / d;
  return (size_t) nsets * d * bits * 4 + (size_t) G * 2 * d * 4 + (size_t) 2 * d * 4 + (size_t) 3 * (bits + 2) * 4 +
         24 + (size_t) 3 * L;
}

extern "C" B2_API int b2_mirrn_retrieve_fwd(const float* x, const uint8_t* mask, const float* R, int64_t r_stride,
                                            int64_t batch, int L, int d, int bits, int k, int32_t* topk_pos,
                                            void* stream) {
  if (int rc = mirrn_check(batch, L, d, k)) return rc;
  B2_REQUIRE(x && mask && R && topk_pos, "NULL pointer");
  B2_REQUIRE(bits >= 1 && bits <= B2_MIRRN_MAX_BITS, "MIRRN: hash_bits must lie in [1, %d], got %d",
             B2_MIRRN_MAX_BITS, bits);
  B2_REQUIRE(r_stride == 0 || r_stride >= (int64_t) d * bits, "MIRRN: r_stride must be 0 or >= d bits");
  if (batch == 0) return B2_OK;
  const size_t smem = mirrn_retrieve_smem(L, d, bits, r_stride ? 3 : 1);
  B2_REQUIRE(smem <= B2_LSH_MAX_SMEM, "MIRRN: d hash_bits = %d needs more shared memory than a CTA has", d * bits);
  B2_REQUIRE(cudaFuncSetAttribute(mirrn_retrieve_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) smem) ==
                 cudaSuccess, "MIRRN: cannot reserve %zu bytes of shared memory", smem);
  B2_LAUNCH(mirrn_retrieve_kernel, (unsigned) batch, MIRRN_THREADS, smem, (cudaStream_t) stream, x, mask, R, r_stride,
            L, d, bits, k, topk_pos);
  B2_CUDA_LAUNCH_CHECK("b2_mirrn_retrieve_fwd");
  return B2_OK;
}

// ---------------------------------------------------------------------------------------------------------------
// Filter.  One CTA per (sample, retrieval); u, y, du are (3, B, k, d), so each retrieval's rows are one contiguous
// (B k, d) block for the add-norm.  Thread t works on column t % d and slots t / d mod G.
struct MirrnWeights {
  const float* cw[3];
  // a constant-index select keeps the parameter struct out of local memory
  __device__ __forceinline__ const float* of(int q) const { return q == 0 ? cw[0] : q == 1 ? cw[1] : cw[2]; }
};
struct MirrnGrads {
  float* cw[3];
  __device__ __forceinline__ float* of(int q) const { return q == 0 ? cw[0] : q == 1 ? cw[1] : cw[2]; }
};

__device__ __forceinline__ int mirrn_diag(int c, int d) {       // complex_weight[n, j, j, 0] of channel c
  const int w = d / 4, n = c / w, j = c - n * w;
  return ((n * w + j) * w + j) * 2;
}

// (H v)_s = sum_t h[(s - t) mod k] v_t over column c of the (k, d) tile v
__device__ __forceinline__ float mirrn_circ(const float* sh, const float* v, int s, int c, int d, int k) {
  float acc = 0.f;
  int m = s;
  for (int t = 0; t < k; ++t) {
    acc = fmaf(sh[m], v[t * d + c], acc);
    m = m == 0 ? k - 1 : m - 1;
  }
  return acc;
}

// shared: u (k d) f32 | h (k) f32 | pos (k) i32
__global__ void __launch_bounds__(MIRRN_THREADS)
mirrn_filter_fwd_kernel(const float* __restrict__ x, const int32_t* __restrict__ topk_pos,
                        const float* __restrict__ pos_table, MirrnWeights W, const float* __restrict__ htab,
                        int64_t batch, int L, int d, int k, float* __restrict__ u, float* __restrict__ y) {
  extern __shared__ float smem[];
  b2_pdl_wait();
  float* su = smem;
  float* sh = su + k * d;
  int32_t* sp = (int32_t*) (sh + k);
  const int64_t b = blockIdx.x;
  const int q = blockIdx.y, t = threadIdx.x;
  const float* xb = x + b * (int64_t) (L + 1) * d;
  for (int s = t; s < k; s += blockDim.x) {
    sp[s] = topk_pos[(b * 3 + q) * k + s];
    sh[s] = htab[s];
  }
  __syncthreads();
  const int64_t o = ((int64_t) q * batch + b) * k * d;
  for (int e = t; e < k * d; e += blockDim.x) {
    const int s = e / d, c = e - s * d;
    const int p = sp[s];
    const float v = __fadd_rn(xb[(int64_t) p * d + c], __fmul_rn(pos_table[(int64_t) (L - p) * d + c], 0.02f));
    su[e] = v;
    u[o + e] = v;
  }
  __syncthreads();
  const float* cw = W.of(q);
  const int G = blockDim.x / d, g = t / d, c = t - g * d;
  if (g < G) {
    const int di = mirrn_diag(c, d);
    const float a = cw[di], bb = cw[di + 1];
    for (int s = g; s < k; s += G)
      y[o + s * d + c] = fmaf(a, su[s * d + c], bb * mirrn_circ(sh, su, s, c, d, k));
  }
}

// shared: dy (k d) f32 | u (k d) f32 | h (k) f32 | pos (k) i32 | part (G 2 d) f32
__global__ void __launch_bounds__(MIRRN_THREADS)
mirrn_filter_bwd_kernel(const float* __restrict__ dy, const float* __restrict__ dres, const float* __restrict__ u,
                        const int32_t* __restrict__ topk_pos, MirrnWeights W, const float* __restrict__ htab,
                        int64_t batch, int L, int d, int k, float* __restrict__ du, MirrnGrads dW,
                        float* __restrict__ dpos) {
  extern __shared__ float smem[];
  b2_pdl_wait();
  const int G = blockDim.x / d;
  float* sdy = smem;
  float* su = sdy + k * d;
  float* sh = su + k * d;
  int32_t* sp = (int32_t*) (sh + k);
  float* part = (float*) (sp + k);
  const int64_t b = blockIdx.x;
  const int q = blockIdx.y, t = threadIdx.x;
  for (int s = t; s < k; s += blockDim.x) {
    sp[s] = topk_pos[(b * 3 + q) * k + s];
    sh[s] = htab[s];
  }
  const int64_t o = ((int64_t) q * batch + b) * k * d;
  for (int e = t; e < k * d; e += blockDim.x) {
    sdy[e] = dy[o + e];
    su[e] = u[o + e];
  }
  __syncthreads();
  const int g = t / d, c = t - g * d;
  const int di = mirrn_diag(c, d);
  if (g < G) {
    const float* cw = W.of(q);
    const float a = cw[di], bb = cw[di + 1];
    float da = 0.f, db = 0.f;
    for (int s = g; s < k; s += G) {
      const float gy = sdy[s * d + c];
      // H is antisymmetric: (H^T gy)_s = -(H gy)_s
      const float v = dres[o + s * d + c] + fmaf(a, gy, -bb * mirrn_circ(sh, sdy, s, c, d, k));
      du[o + s * d + c] = v;
      atomicAdd(dpos + (int64_t) (L - sp[s]) * d + c, __fmul_rn(v, 0.02f));
      da = fmaf(gy, su[s * d + c], da);
      db = fmaf(gy, mirrn_circ(sh, su, s, c, d, k), db);
    }
    part[g * 2 * d + c] = da;
    part[g * 2 * d + d + c] = db;
  }
  __syncthreads();
  if (t < d) {
    float da = 0.f, db = 0.f;
    for (int r = 0; r < G; ++r) {
      da += part[r * 2 * d + t];
      db += part[r * 2 * d + d + t];
    }
    const int dt = mirrn_diag(t, d);
    float* dcw = dW.of(q);
    atomicAdd(dcw + dt, da);
    atomicAdd(dcw + dt + 1, db);
  }
}

static int mirrn_filter_check(int64_t batch, int L, int d, int k, int pos_rows, size_t* smem_out, bool bwd) {
  if (int rc = mirrn_check(batch, L, d, k)) return rc;
  B2_REQUIRE(pos_rows > L, "MIRRN: the position table has %d rows, the history length L = %d needs L + 1 (max_len "
             ">= L)", pos_rows, L);
  const size_t smem = (size_t) k * d * 4 * (bwd ? 2 : 1) + (size_t) k * 8 +
                      (bwd ? (size_t) (MIRRN_THREADS / d) * 2 * d * 4 : 0);
  B2_REQUIRE(smem <= B2_LSH_MAX_SMEM, "MIRRN: k d = %d needs more shared memory than a CTA has", k * d);
  *smem_out = smem;
  return B2_OK;
}

extern "C" B2_API int b2_mirrn_filter_fwd(const float* x, const int32_t* topk_pos, const float* pos_table,
                                          int pos_rows, const float* cw0, const float* cw1, const float* cw2,
                                          const float* htab, int64_t batch, int L, int d, int k, float* u, float* y,
                                          void* stream) {
  size_t smem = 0;
  if (int rc = mirrn_filter_check(batch, L, d, k, pos_rows, &smem, false)) return rc;
  B2_REQUIRE(x && topk_pos && pos_table && cw0 && cw1 && cw2 && htab && u && y, "NULL pointer");
  if (batch == 0) return B2_OK;
  B2_REQUIRE(cudaFuncSetAttribute(mirrn_filter_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) smem) ==
                 cudaSuccess, "MIRRN: cannot reserve %zu bytes of shared memory", smem);
  MirrnWeights W = {{cw0, cw1, cw2}};
  B2_LAUNCH(mirrn_filter_fwd_kernel, dim3((unsigned) batch, 3), MIRRN_THREADS, smem, (cudaStream_t) stream, x,
            topk_pos, pos_table, W, htab, batch, L, d, k, u, y);
  B2_CUDA_LAUNCH_CHECK("b2_mirrn_filter_fwd");
  return B2_OK;
}

extern "C" B2_API int b2_mirrn_filter_bwd(const float* dy, const float* dres, const float* u, const int32_t* topk_pos,
                                          int pos_rows, const float* cw0, const float* cw1, const float* cw2,
                                          const float* htab, int64_t batch, int L, int d, int k, float* du,
                                          float* dcw0, float* dcw1, float* dcw2, float* dpos, void* stream) {
  size_t smem = 0;
  if (int rc = mirrn_filter_check(batch, L, d, k, pos_rows, &smem, true)) return rc;
  B2_REQUIRE(dy && dres && u && topk_pos && cw0 && cw1 && cw2 && htab && du && dcw0 && dcw1 && dcw2 && dpos,
             "NULL pointer");
  if (batch == 0) return B2_OK;
  B2_REQUIRE(cudaFuncSetAttribute(mirrn_filter_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) smem) ==
                 cudaSuccess, "MIRRN: cannot reserve %zu bytes of shared memory", smem);
  MirrnWeights W = {{cw0, cw1, cw2}};
  MirrnGrads dW = {{dcw0, dcw1, dcw2}};
  B2_LAUNCH(mirrn_filter_bwd_kernel, dim3((unsigned) batch, 3), MIRRN_THREADS, smem, (cudaStream_t) stream, dy, dres,
            u, topk_pos, W, htab, batch, L, d, k, du, dW, dpos);
  B2_CUDA_LAUNCH_CHECK("b2_mirrn_filter_bwd");
  return B2_OK;
}

// ---------------------------------------------------------------------------------------------------------------
// Mean over the k slots: out[b, q, :] = mean_s z[q, b, s, :] (z (3, B, k, d)), and its backward.
__global__ void __launch_bounds__(MIRRN_THREADS)
mirrn_mean_fwd_kernel(const float* __restrict__ z, int64_t batch, int d, int k, float* __restrict__ out) {
  b2_pdl_wait();
  const int64_t n = batch * 3 * d;
  for (int64_t e = blockIdx.x * (int64_t) blockDim.x + threadIdx.x; e < n; e += (int64_t) gridDim.x * blockDim.x) {
    const int64_t bq = e / d;
    const int c = (int) (e - bq * d);
    const int64_t b = bq / 3;
    const int q = (int) (bq - b * 3);
    const float* zr = z + ((q * batch + b) * k) * d + c;
    float s = 0.f;
    for (int r = 0; r < k; ++r) s += zr[(int64_t) r * d];
    out[e] = s / (float) k;
  }
}

__global__ void __launch_bounds__(MIRRN_THREADS)
mirrn_mean_bwd_kernel(const float* __restrict__ g, int64_t batch, int d, int k, float* __restrict__ dz) {
  b2_pdl_wait();
  const int64_t n = 3 * batch * k * d;
  for (int64_t e = blockIdx.x * (int64_t) blockDim.x + threadIdx.x; e < n; e += (int64_t) gridDim.x * blockDim.x) {
    const int64_t row = e / d;
    const int c = (int) (e - row * d);
    const int64_t qb = row / k;                 // q B + b
    const int64_t q = qb / batch, b = qb - q * batch;
    dz[e] = g[(b * 3 + q) * d + c] / (float) k;
  }
}

static unsigned mirrn_grid(int64_t n) {
  return (unsigned) std::min<int64_t>((n + MIRRN_THREADS - 1) / MIRRN_THREADS, (int64_t) B2_NUM_SMS * 16);
}

extern "C" B2_API int b2_mirrn_mean_fwd(const float* z, int64_t batch, int d, int k, float* out, void* stream) {
  B2_REQUIRE(z && out, "NULL pointer");
  B2_REQUIRE(batch >= 0 && d >= 1 && d <= B2_LSH_MAX_DIM && k >= 1 && k <= B2_LSH_MAX_TOPK,
             "MIRRN: mean over k = %d slots of width d = %d outside the range", k, d);
  if (batch == 0) return B2_OK;
  B2_LAUNCH(mirrn_mean_fwd_kernel, mirrn_grid(batch * 3 * d), MIRRN_THREADS, 0, (cudaStream_t) stream, z, batch, d, k,
            out);
  B2_CUDA_LAUNCH_CHECK("b2_mirrn_mean_fwd");
  return B2_OK;
}

extern "C" B2_API int b2_mirrn_mean_bwd(const float* g, int64_t batch, int d, int k, float* dz, void* stream) {
  B2_REQUIRE(g && dz, "NULL pointer");
  B2_REQUIRE(batch >= 0 && d >= 1 && d <= B2_LSH_MAX_DIM && k >= 1 && k <= B2_LSH_MAX_TOPK,
             "MIRRN: mean over k = %d slots of width d = %d outside the range", k, d);
  if (batch == 0) return B2_OK;
  B2_LAUNCH(mirrn_mean_bwd_kernel, mirrn_grid(3 * batch * k * d), MIRRN_THREADS, 0, (cudaStream_t) stream, g, batch, d,
            k, dz);
  B2_CUDA_LAUNCH_CHECK("b2_mirrn_mean_bwd");
  return B2_OK;
}

// ---------------------------------------------------------------------------------------------------------------
// Gradient assembly: dx (B, L + 1, d) "=", every row written once.  Row L: dt0 + dt1 + dt2.  Rows [L - S, L): dshort.
// Row l also adds du[q, b, s] for each retrieval q that picked l at slot s, in the order q = 0, 1, 2.
// shared: inv (3 L) i16
__global__ void __launch_bounds__(MIRRN_THREADS)
mirrn_assemble_kernel(const float* __restrict__ dt0, const float* __restrict__ dt1, const float* __restrict__ dt2,
                      const float* __restrict__ dshort, int S, const float* __restrict__ du,
                      const int32_t* __restrict__ topk_pos, int64_t batch, int L, int d, int k,
                      float* __restrict__ dx) {
  extern __shared__ float smem[];
  b2_pdl_wait();
  int16_t* inv = (int16_t*) smem;
  const int64_t b = blockIdx.x;
  const int t = threadIdx.x;
  for (int e = t; e < 3 * L; e += blockDim.x) inv[e] = -1;
  __syncthreads();
  for (int e = t; e < 3 * k; e += blockDim.x) {
    const int q = e / k;
    inv[q * L + topk_pos[b * 3 * k + e]] = (int16_t) (e - q * k);
  }
  __syncthreads();
  float* ob = dx + b * (int64_t) (L + 1) * d;
  const int w0 = L - S;
  for (int64_t e = t; e < (int64_t) (L + 1) * d; e += blockDim.x) {
    const int l = (int) (e / d), c = (int) (e - (int64_t) l * d);
    float v;
    if (l == L) {
      v = dt0[b * d + c] + dt1[b * d + c] + dt2[b * d + c];
    } else {
      v = l >= w0 ? dshort[(b * S + (l - w0)) * d + c] : 0.f;
#pragma unroll
      for (int q = 0; q < 3; ++q) {
        const int s = inv[q * L + l];
        if (s >= 0) v += du[(((int64_t) q * batch + b) * k + s) * d + c];
      }
    }
    ob[e] = v;
  }
}

extern "C" B2_API int b2_mirrn_assemble_bwd(const float* dt0, const float* dt1, const float* dt2, const float* dshort,
                                            int S, const float* du, const int32_t* topk_pos, int64_t batch, int L,
                                            int d, int k, float* dx, void* stream) {
  if (int rc = mirrn_check(batch, L, d, k)) return rc;
  B2_REQUIRE(dt0 && dt1 && dt2 && dshort && du && topk_pos && dx, "NULL pointer");
  B2_REQUIRE(S >= 1 && S <= L, "MIRRN: the short window S must lie in [1, L], got %d (L = %d)", S, L);
  if (batch == 0) return B2_OK;
  const size_t smem = (size_t) 3 * L * 2;
  B2_REQUIRE(cudaFuncSetAttribute(mirrn_assemble_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) smem) ==
                 cudaSuccess, "MIRRN: cannot reserve %zu bytes of shared memory", smem);
  B2_LAUNCH(mirrn_assemble_kernel, (unsigned) batch, MIRRN_THREADS, smem, (cudaStream_t) stream, dt0, dt1, dt2, dshort,
            S, du, topk_pos, batch, L, d, k, dx);
  B2_CUDA_LAUNCH_CHECK("b2_mirrn_assemble_bwd");
  return B2_OK;
}

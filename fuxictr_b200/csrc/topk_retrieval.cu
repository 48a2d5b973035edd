// topk_retrieval.cu — learned-score top-k retrieval over a long behaviour sequence, sm_90a: SIM's soft-search GSU
// (model_zoo/LongCTR/SIM/SIM.py) and TWIN's MultiHeadTopKAttention (model_zoo/LongCTR/TWIN/TWIN.py).
//
// x is item_feat_emb (B, L + 1, d): positions [0, L) are the history, position L the target.  One CTA per sample.
// Both select with b2_topk_select (topk_select.cuh): descending score, ties to the lower position, -0.0 == +0.0.
// Every score is an fp32 FMA dot product over the d columns in ascending order, so the backward recomputes exactly
// the forward's scores.  Every sum over positions runs in a fixed order (column groups, then the groups in order), so
// the results are deterministic, and each kernel writes its outputs once, with no atomics to global memory.
// SIM: qk_l = (u . x_l) mask_l with u = W_b^T W_a t; masked positions score 0, as in the reference, so they outrank
// negatively scored valid rows and fill the selection when fewer than k valid rows score above 0.
// TWIN: score_hl = q'_h . x_l, exactly -1e9 where masked (the reference fills after the scale, which q' carries); the
// softmax runs over the k chosen per head, so a head whose chosen rows are all masked weights them uniformly.
// Each kernel waits for its predecessor (programmatic dependent launch) before its first read and never triggers its
// successor early.
#include "b2_common.cuh"
#include "topk_select.cuh"

#define TOPK_THREADS 256

static int topk_check(int64_t batch, int L, int d) {
  B2_REQUIRE(d >= 1 && d <= B2_TOPK_MAX_DIM, "top-k: the item width d must lie in [1, %d], got %d", B2_TOPK_MAX_DIM,
             d);
  B2_REQUIRE(L >= 1 && L <= B2_TOPK_MAX_LEN, "top-k: the history length L must lie in [1, %d], got %d",
             B2_TOPK_MAX_LEN, L);
  B2_REQUIRE(batch >= 0, "top-k: negative batch %lld", (long long) batch);
  B2_REQUIRE(batch * (L + 1) < ((int64_t) 1 << 31), "top-k: batch (L + 1) must stay below 2^31");
  return B2_OK;
}

static int topk_k_check(int k, int L) {
  B2_REQUIRE(k >= 1 && k <= L && k <= B2_TOPK_MAX_K, "top-k: k must lie in [1, min(L, %d)], got %d (L = %d)",
             B2_TOPK_MAX_K, k, L);
  return B2_OK;
}

template <typename K>
static int topk_smem_attr(K kernel, size_t smem, const char* name) {
  B2_REQUIRE(smem <= B2_TOPK_MAX_SMEM, "%s: needs %zu bytes of shared memory, more than a CTA has", name, smem);
  B2_REQUIRE(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) smem) == cudaSuccess,
             "%s: cannot reserve %zu bytes of shared memory", name, smem);
  return B2_OK;
}

__device__ __forceinline__ float topk_dot(const float* __restrict__ v, const float* s, int d) {
  float acc = 0.f;
  for (int i = 0; i < d; ++i) acc = fmaf(__ldg(v + i), s[i], acc);
  return acc;
}

// out[c] = sum_l w[l] x_l[c] over positions pos ? pos[j] : j for j < n, in a fixed order: thread t sums column t % d
// over j = t / d mod G (G = blockDim / d column groups) into part, then the groups are added in order.  Ends
// synchronised; out is shared or global.
__device__ void topk_pool(const float* __restrict__ xb, const float* w, const int32_t* pos, int n, int d,
                          float* part, float* out) {
  const int G = blockDim.x / d, t = threadIdx.x, i = t % d, g = t / d;
  if (g < G) {
    float acc = 0.f;
    for (int j = g; j < n; j += G) acc = fmaf(w[j], xb[(int64_t) (pos ? pos[j] : j) * d + i], acc);
    part[g * d + i] = acc;
  }
  __syncthreads();
  for (int c = t; c < d; c += blockDim.x) {
    float s = 0.f;
    for (int q = 0; q < G; ++q) s += part[q * d + c];
    out[c] = s;
  }
  __syncthreads();
}

static size_t topk_part_bytes(int d) { return (size_t) (TOPK_THREADS / d) * d * 4; }

// ---------------------------------------------------------------------------------------------------------------
// SIM forward: GSU scores, pooled, selection and the compact rows.
// shared: key (L) u32 | qk (L) f32 | u (d) f32 | part | sel (k) i32
__global__ void __launch_bounds__(TOPK_THREADS)
sim_retrieve_kernel(const float* __restrict__ x, const uint8_t* __restrict__ mask, const float* __restrict__ u,
                    int L, int d, int k, float* __restrict__ qk, float* __restrict__ pooled,
                    float* __restrict__ topk_emb, uint8_t* __restrict__ topk_mask, int32_t* __restrict__ topk_pos) {
  extern __shared__ float smem[];
  __shared__ B2TopkSmem ts;
  b2_pdl_wait();
  uint32_t* key = (uint32_t*) smem;
  float* sqk = smem + L;
  float* su = sqk + L;
  float* part = su + d;
  int32_t* sel = (int32_t*) (part + (blockDim.x / d) * d);
  const int64_t b = blockIdx.x;
  const float* xb = x + b * (int64_t) (L + 1) * d;
  const uint8_t* mb = mask + b * (int64_t) L;
  for (int c = threadIdx.x; c < d; c += blockDim.x) su[c] = u[b * d + c];
  __syncthreads();
  for (int l = threadIdx.x; l < L; l += blockDim.x) {
    const float s = mb[l] ? topk_dot(xb + (int64_t) l * d, su, d) : 0.f;
    sqk[l] = s;
    key[l] = b2_topk_key(s);
    qk[b * L + l] = s;
  }
  __syncthreads();
  topk_pool(xb, sqk, nullptr, L, d, part, pooled + b * d);
  b2_topk_select(key, L, k, sel, ts);
  for (int s = threadIdx.x; s < k; s += blockDim.x) {
    const int p = sel[s];
    topk_pos[b * k + s] = p;
    topk_mask[b * k + s] = mb[p] != 0;
  }
  float* ob = topk_emb + b * (int64_t) k * d;
  for (int e = threadIdx.x; e < k * d; e += blockDim.x) {
    const int s = e / d, i = e - s * d;
    ob[e] = xb[(int64_t) sel[s] * d + i];
  }
}

static size_t sim_retrieve_smem(int L, int d, int k) {
  return (size_t) L * 8 + (size_t) d * 4 + topk_part_bytes(d) + (size_t) k * 4;
}

extern "C" B2_API int b2_sim_retrieve_fwd(const float* x, const uint8_t* mask, const float* u, int64_t batch, int L,
                                          int d, int k, float* qk, float* pooled, float* topk_emb,
                                          uint8_t* topk_mask, int32_t* topk_pos, void* stream) {
  if (int rc = topk_check(batch, L, d)) return rc;
  if (int rc = topk_k_check(k, L)) return rc;
  B2_REQUIRE(x && mask && u && qk && pooled && topk_emb && topk_mask && topk_pos, "NULL pointer");
  if (batch == 0) return B2_OK;
  const size_t smem = sim_retrieve_smem(L, d, k);
  if (int rc = topk_smem_attr(sim_retrieve_kernel, smem, "b2_sim_retrieve_fwd")) return rc;
  B2_LAUNCH(sim_retrieve_kernel, (unsigned) batch, TOPK_THREADS, smem, (cudaStream_t) stream, x, mask, u, L, d, k, qk,
            pooled, topk_emb, topk_mask, topk_pos);
  B2_CUDA_LAUNCH_CHECK("b2_sim_retrieve_fwd");
  return B2_OK;
}

// ---------------------------------------------------------------------------------------------------------------
// SIM backward of pooled = sum_l qk_l x_l into the scores: dqk_l = (dpooled . x_l) mask_l, du = sum_l dqk_l x_l.
// shared: dqk (L) f32 | dpooled (d) f32 | part
__global__ void __launch_bounds__(TOPK_THREADS)
sim_gsu_bwd_kernel(const float* __restrict__ x, const uint8_t* __restrict__ mask, const float* __restrict__ dpooled,
                   int L, int d, float* __restrict__ dqk, float* __restrict__ du) {
  extern __shared__ float smem[];
  b2_pdl_wait();
  float* sdq = smem;
  float* sdp = sdq + L;
  float* part = sdp + d;
  const int64_t b = blockIdx.x;
  const float* xb = x + b * (int64_t) (L + 1) * d;
  const uint8_t* mb = mask + b * (int64_t) L;
  for (int c = threadIdx.x; c < d; c += blockDim.x) sdp[c] = dpooled[b * d + c];
  __syncthreads();
  for (int l = threadIdx.x; l < L; l += blockDim.x) {
    const float s = mb[l] ? topk_dot(xb + (int64_t) l * d, sdp, d) : 0.f;
    sdq[l] = s;
    dqk[b * L + l] = s;
  }
  __syncthreads();
  topk_pool(xb, sdq, nullptr, L, d, part, du + b * d);
}

extern "C" B2_API int b2_sim_gsu_bwd(const float* x, const uint8_t* mask, const float* dpooled, int64_t batch, int L,
                                     int d, float* dqk, float* du, void* stream) {
  if (int rc = topk_check(batch, L, d)) return rc;
  B2_REQUIRE(x && mask && dpooled && dqk && du, "NULL pointer");
  if (batch == 0) return B2_OK;
  const size_t smem = (size_t) L * 4 + (size_t) d * 4 + topk_part_bytes(d);
  if (int rc = topk_smem_attr(sim_gsu_bwd_kernel, smem, "b2_sim_gsu_bwd")) return rc;
  B2_LAUNCH(sim_gsu_bwd_kernel, (unsigned) batch, TOPK_THREADS, smem, (cudaStream_t) stream, x, mask, dpooled, L, d,
            dqk, du);
  B2_CUDA_LAUNCH_CHECK("b2_sim_gsu_bwd");
  return B2_OK;
}

// ---------------------------------------------------------------------------------------------------------------
// SIM gradient assembly: every row of dx written once.  Row L: dt0 + dt1 + dt2 + dt3.  Rows [0, L): dshort on the
// window [L - S, L), dlong (B, k, d) at the chosen positions (an inverse map in shared memory; a sample's positions
// are distinct), and the GSU's qk_l dpooled + dqk_l u.
// shared: inv (L) i32 | u (d) f32 | dpooled (d) f32
__global__ void __launch_bounds__(TOPK_THREADS)
sim_assemble_kernel(const float* __restrict__ dt0, const float* __restrict__ dt1, const float* __restrict__ dt2,
                    const float* __restrict__ dt3, const float* __restrict__ dshort, int S,
                    const float* __restrict__ dlong, const int32_t* __restrict__ pos, int k,
                    const float* __restrict__ qk, const float* __restrict__ dqk, const float* __restrict__ u,
                    const float* __restrict__ dpooled, int L, int d, float* __restrict__ dx) {
  extern __shared__ float smem[];
  b2_pdl_wait();
  int32_t* inv = (int32_t*) smem;
  float* su = smem + L;
  float* sdp = su + d;
  const int64_t b = blockIdx.x;
  const int t = threadIdx.x;
  for (int l = t; l < L; l += blockDim.x) inv[l] = -1;
  for (int c = t; c < d; c += blockDim.x) {
    su[c] = u[b * d + c];
    sdp[c] = dpooled[b * d + c];
  }
  __syncthreads();
  for (int s = t; s < k; s += blockDim.x) inv[pos[b * k + s]] = s;
  __syncthreads();
  float* ob = dx + b * (int64_t) (L + 1) * d;
  const int w0 = L - S;
  for (int64_t e = t; e < (int64_t) (L + 1) * d; e += blockDim.x) {
    const int l = (int) (e / d), c = (int) (e - (int64_t) l * d);
    float v;
    if (l == L) {
      v = dt0[b * d + c] + dt1[b * d + c] + dt2[b * d + c] + dt3[b * d + c];
    } else {
      v = l >= w0 ? dshort[(b * S + (l - w0)) * d + c] : 0.f;
      const int s = inv[l];
      if (s >= 0) v += dlong[(b * k + s) * (int64_t) d + c];
      v += qk[b * L + l] * sdp[c] + dqk[b * L + l] * su[c];
    }
    ob[e] = v;
  }
}

extern "C" B2_API int b2_sim_assemble_bwd(const float* dt0, const float* dt1, const float* dt2, const float* dt3,
                                          const float* dshort, int S, const float* dlong, const int32_t* pos,
                                          const float* qk, const float* dqk, const float* u, const float* dpooled,
                                          int64_t batch, int L, int d, int k, float* dx, void* stream) {
  if (int rc = topk_check(batch, L, d)) return rc;
  if (int rc = topk_k_check(k, L)) return rc;
  B2_REQUIRE(dt0 && dt1 && dt2 && dt3 && dshort && dlong && pos && qk && dqk && u && dpooled && dx, "NULL pointer");
  B2_REQUIRE(S >= 1 && S <= L, "SIM: the short window S must lie in [1, L], got %d (L = %d)", S, L);
  if (batch == 0) return B2_OK;
  const size_t smem = (size_t) L * 4 + (size_t) d * 8;
  if (int rc = topk_smem_attr(sim_assemble_kernel, smem, "b2_sim_assemble_bwd")) return rc;
  B2_LAUNCH(sim_assemble_kernel, (unsigned) batch, TOPK_THREADS, smem, (cudaStream_t) stream, dt0, dt1, dt2, dt3,
            dshort, S, dlong, pos, k, qk, dqk, u, dpooled, L, d, dx);
  B2_CUDA_LAUNCH_CHECK("b2_sim_assemble_bwd");
  return B2_OK;
}

// ---------------------------------------------------------------------------------------------------------------
// TWIN forward, heads one after another: scores, selection, softmax over the k chosen, p_h = sum_s a_hs x_{pos_hs}.
// shared: key (L) u32 | q'_h (d) f32 | a (k) f32 | part | sel (k) i32
__global__ void __launch_bounds__(TOPK_THREADS)
twin_topk_fwd_kernel(const float* __restrict__ q, const float* __restrict__ x, const uint8_t* __restrict__ mask,
                     int L, int d, int H, int k, float* __restrict__ p, float* __restrict__ stats,
                     int32_t* __restrict__ topk_pos) {
  extern __shared__ float smem[];
  __shared__ B2TopkSmem ts;
  b2_pdl_wait();
  uint32_t* key = (uint32_t*) smem;
  float* sq = smem + L;
  float* sa = sq + d;
  float* part = sa + k;
  int32_t* sel = (int32_t*) (part + (blockDim.x / d) * d);
  const int64_t b = blockIdx.x;
  const float* xb = x + b * (int64_t) (L + 1) * d;
  const uint8_t* mb = mask + b * (int64_t) L;
  for (int h = 0; h < H; ++h) {
    for (int c = threadIdx.x; c < d; c += blockDim.x) sq[c] = q[(b * H + h) * d + c];
    __syncthreads();
    for (int l = threadIdx.x; l < L; l += blockDim.x)
      key[l] = b2_topk_key(mb[l] ? topk_dot(xb + (int64_t) l * d, sq, d) : -1e9f);
    b2_topk_select(key, L, k, sel, ts);                  // begins with a barrier, so the keys are visible
    if (threadIdx.x < 32) {
      const float m = b2_topk_value(key[sel[0]]);
      float sum = 0.f;
      for (int s = threadIdx.x; s < k; s += 32) {
        const float e = expf(b2_topk_value(key[sel[s]]) - m);
        sa[s] = e;
        sum += e;
      }
      sum = b2_warp_sum(sum);
      for (int s = threadIdx.x; s < k; s += 32) sa[s] = sa[s] / sum;
      if (threadIdx.x == 0) {
        stats[(b * H + h) * 2] = m;
        stats[(b * H + h) * 2 + 1] = sum;
      }
    }
    for (int s = threadIdx.x; s < k; s += blockDim.x) topk_pos[(b * H + h) * k + s] = sel[s];
    __syncthreads();
    topk_pool(xb, sa, sel, k, d, part, p + (b * H + h) * d);
  }
}

static size_t twin_fwd_smem(int L, int d, int k) {
  return (size_t) L * 4 + (size_t) d * 4 + (size_t) k * 8 + topk_part_bytes(d);
}

static int twin_check(int64_t batch, int L, int d, int heads, int k) {
  if (int rc = topk_check(batch, L, d)) return rc;
  if (int rc = topk_k_check(k, L)) return rc;
  B2_REQUIRE(heads >= 1 && heads <= B2_MHTA_MAX_HEADS && heads * d <= B2_MHTA_MAX_WIDTH,
             "TWIN: heads must lie in [1, %d] with heads d <= %d, got heads %d, d %d", B2_MHTA_MAX_HEADS,
             B2_MHTA_MAX_WIDTH, heads, d);
  return B2_OK;
}

extern "C" B2_API int b2_twin_topk_fwd(const float* q, const float* x, const uint8_t* mask, int64_t batch, int L,
                                       int d, int heads, int k, float* p, float* stats, int32_t* topk_pos,
                                       void* stream) {
  if (int rc = twin_check(batch, L, d, heads, k)) return rc;
  B2_REQUIRE(q && x && mask && p && stats && topk_pos, "NULL pointer");
  if (batch == 0) return B2_OK;
  const size_t smem = twin_fwd_smem(L, d, k);
  if (int rc = topk_smem_attr(twin_topk_fwd_kernel, smem, "b2_twin_topk_fwd")) return rc;
  B2_LAUNCH(twin_topk_fwd_kernel, (unsigned) batch, TOPK_THREADS, smem, (cudaStream_t) stream, q, x, mask, L, d,
            heads, k, p, stats, topk_pos);
  B2_CUDA_LAUNCH_CHECK("b2_twin_topk_fwd");
  return B2_OK;
}

// ---------------------------------------------------------------------------------------------------------------
// TWIN backward over the chosen positions.  a_hs recomputed from the saved stats and the forward's own scores;
// ds_hs = a_hs (dp_h . x_l - dp_h . p_h), 0 where l is masked (the -1e9 fill is constant); dq'_h = sum_s ds_hs x_l;
// dx_l = sum over the heads h that chose l of (a_hs dp_h + ds_hs q'_h), plus dshort on the window; row L =
// dt0 + dt1 + dq' W_M (GEMM1's data gradient, fp32 here as GEMM1 is).  A head's slot of position l sits in a (H, L)
// u16 map, 0xffff where the head did not choose l.
// shared: slot (H L) u16 | q' (H d) | dp (H d) | dq' (H d) | a (H k) | ds (H k) | pos (H k) i32 | dp.p (H)
__global__ void __launch_bounds__(TOPK_THREADS)
twin_topk_bwd_kernel(const float* __restrict__ q, const float* __restrict__ x, const uint8_t* __restrict__ mask,
                     const float* __restrict__ p, const float* __restrict__ stats, const int32_t* __restrict__ topk_pos,
                     const float* __restrict__ dp, const float* __restrict__ WM, const float* __restrict__ dt0,
                     const float* __restrict__ dt1, const float* __restrict__ dshort, int S, int L, int d, int H, int k,
                     float* __restrict__ dq, float* __restrict__ dx) {
  extern __shared__ float smem[];
  b2_pdl_wait();
  const int Hd = H * d, Hk = H * k;
  uint16_t* slot = (uint16_t*) smem;
  float* sq = smem + ((H * L + 1) >> 1);
  float* sdp = sq + Hd;
  float* sdq = sdp + Hd;
  float* sa = sdq + Hd;
  float* sds = sa + Hk;
  int32_t* spos = (int32_t*) (sds + Hk);
  float* dpp = (float*) (spos + Hk);
  const int64_t b = blockIdx.x;
  const int t = threadIdx.x;
  const float* xb = x + b * (int64_t) (L + 1) * d;
  const uint8_t* mb = mask + b * (int64_t) L;
  for (int e = t; e < H * L; e += blockDim.x) slot[e] = 0xffff;
  for (int e = t; e < Hd; e += blockDim.x) {
    sq[e] = q[b * Hd + e];
    sdp[e] = dp[b * Hd + e];
  }
  for (int e = t; e < Hk; e += blockDim.x) spos[e] = topk_pos[b * Hk + e];
  for (int h = t >> 5; h < H; h += blockDim.x >> 5) {    // dp_h . p_h, one warp per head
    float v = 0.f;
    for (int c = t & 31; c < d; c += 32) v = fmaf(dp[b * Hd + h * d + c], p[b * Hd + h * d + c], v);
    v = b2_warp_sum(v);
    if ((t & 31) == 0) dpp[h] = v;
  }
  __syncthreads();
  for (int e = t; e < Hk; e += blockDim.x) {
    const int h = e / k, l = spos[e];
    slot[h * L + l] = (uint16_t) (e - h * k);
    const float* xl = xb + (int64_t) l * d;
    const float sc = mb[l] ? topk_dot(xl, sq + h * d, d) : -1e9f;
    const float a = expf(sc - stats[(b * H + h) * 2]) / stats[(b * H + h) * 2 + 1];
    sa[e] = a;
    sds[e] = mb[l] ? a * (topk_dot(xl, sdp + h * d, d) - dpp[h]) : 0.f;
  }
  __syncthreads();
  for (int e = t; e < Hd; e += blockDim.x) {
    const int h = e / d, c = e - h * d;
    float v = 0.f;
    for (int s = 0; s < k; ++s) v = fmaf(sds[h * k + s], xb[(int64_t) spos[h * k + s] * d + c], v);
    sdq[e] = v;
    dq[b * Hd + e] = v;
  }
  __syncthreads();
  float* ob = dx + b * (int64_t) (L + 1) * d;
  const int w0 = L - S;
  for (int64_t e = t; e < (int64_t) (L + 1) * d; e += blockDim.x) {
    const int l = (int) (e / d), c = (int) (e - (int64_t) l * d);
    float v;
    if (l == L) {
      v = dt0[b * d + c] + dt1[b * d + c];
      for (int j = 0; j < Hd; ++j) v = fmaf(sdq[j], __ldg(WM + (int64_t) j * d + c), v);
    } else {
      v = l >= w0 ? dshort[(b * S + (l - w0)) * d + c] : 0.f;
      for (int h = 0; h < H; ++h) {
        const int s = slot[h * L + l];
        if (s != 0xffff) v += sa[h * k + s] * sdp[h * d + c] + sds[h * k + s] * sq[h * d + c];
      }
    }
    ob[e] = v;
  }
}

static size_t twin_bwd_smem(int L, int d, int H, int k) {
  return (size_t) ((H * L + 1) >> 1) * 4 + (size_t) H * d * 12 + (size_t) H * k * 12 + (size_t) H * 4;
}

extern "C" B2_API int b2_twin_topk_bwd(const float* q, const float* x, const uint8_t* mask, const float* p,
                                       const float* stats, const int32_t* topk_pos, const float* dp, const float* WM,
                                       const float* dt0, const float* dt1, const float* dshort, int S, int64_t batch,
                                       int L, int d, int heads, int k, float* dq, float* dx, void* stream) {
  if (int rc = twin_check(batch, L, d, heads, k)) return rc;
  B2_REQUIRE(q && x && mask && p && stats && topk_pos && dp && WM && dt0 && dt1 && dshort && dq && dx,
             "NULL pointer");
  B2_REQUIRE(S >= 1 && S <= L, "TWIN: the short window S must lie in [1, L], got %d (L = %d)", S, L);
  if (batch == 0) return B2_OK;
  const size_t smem = twin_bwd_smem(L, d, heads, k);
  if (int rc = topk_smem_attr(twin_topk_bwd_kernel, smem, "b2_twin_topk_bwd")) return rc;
  B2_LAUNCH(twin_topk_bwd_kernel, (unsigned) batch, TOPK_THREADS, smem, (cudaStream_t) stream, q, x, mask, p, stats,
            topk_pos, dp, WM, dt0, dt1, dshort, S, L, d, heads, k, dq, dx);
  B2_CUDA_LAUNCH_CHECK("b2_twin_topk_bwd");
  return B2_OK;
}

// lsh.cu — SimHash retrieval (ETA, model_zoo/LongCTR/ETA/ETA.py) and hash-collision pooling (SDIM,
// model_zoo/LongCTR/SDIM/SDIM.py) over a long behaviour sequence, sm_90a.
//
// x is item_feat_emb (B, L + 1, d): positions [0, L) are the history, position L the target.  One CTA per sample.
// SimHash bit j of a row v is v . R[:, j] > 0, the reference's argmax([-r, r]) (bit 0 at r = 0, so a zero padding row
// hashes to all zeros).  The projection is fp32 FMA over the d columns in ascending order, in every matmul mode: a TF32
// or bf16 projection would flip bits near a hyperplane.  A thread takes one position and keeps up to 32 projections
// (one code word) in registers; R sits in shared memory and every thread of a warp reads the same element.
//
// ETA: the distance is popc(code_l ^ code_t), 1 + bits where mask is 0.  The k smallest are found by a counting sort
// over the bits + 2 possible distances: a shared histogram, its prefix sum, then one warp walks the positions in
// ascending order and ranks each within its distance with __match_any_sync.  Ties are thus broken by ascending
// position and the output is sorted by (distance, position); torch.topk leaves tie order unspecified.
// SDIM: bucket h of a row is its bits-bit code under R[:, h, :]; position l collides in hash h when its bucket equals
// the target's and mask[l] != 0, one bit per hash in a 32-bit word per position.  The sums over colliding rows are
// formed column by column in a fixed order, so the result is deterministic.
// The backward of either model is one assembly launch that writes d(item_feat_emb) once: the target row (three
// gradients added), the short-attention window and the long-interest rows.  A sample's positions are distinct, so no
// atomics.  Each kernel waits for its predecessor (programmatic dependent launch) before its first read and never
// triggers its successor early.
#include "b2_common.cuh"
#include "lsh_common.cuh"

#define LSH_THREADS 256
#define LSH_WARPS (LSH_THREADS / 32)

static int lsh_check(int64_t batch, int L, int d) {
  B2_REQUIRE(d >= 1 && d <= B2_LSH_MAX_DIM, "LSH: the item width d must lie in [1, %d], got %d", B2_LSH_MAX_DIM, d);
  B2_REQUIRE(L >= 1 && L <= B2_LSH_MAX_LEN, "LSH: the history length L must lie in [1, %d], got %d", B2_LSH_MAX_LEN,
             L);
  B2_REQUIRE(batch >= 0, "LSH: negative batch %lld", (long long) batch);
  B2_REQUIRE(batch * (L + 1) < ((int64_t) 1 << 31), "LSH: batch (L + 1) must stay below 2^31");
  return B2_OK;
}

// ---------------------------------------------------------------------------------------------------------------
// ETA retrieval
// shared: R (d bits) f32 | pos (k) i32 | hist (bits + 2) i32 | tcode (2) u32 | dist (L) u8
__global__ void __launch_bounds__(LSH_THREADS)
eta_retrieve_kernel(const float* __restrict__ x, const uint8_t* __restrict__ mask, const float* __restrict__ R,
                    int64_t r_stride, int L, int d, int bits, int k, float* __restrict__ topk_emb,
                    uint8_t* __restrict__ topk_mask, int32_t* __restrict__ topk_pos) {
  extern __shared__ float smem[];
  b2_pdl_wait();
  float* sR = smem;
  int32_t* spos = (int32_t*) (sR + d * bits);
  int32_t* hist = spos + k;
  uint32_t* tcode = (uint32_t*) (hist + bits + 2);
  uint8_t* dist = (uint8_t*) (tcode + 2);
  const int64_t b = blockIdx.x;
  const float* xb = x + b * (int64_t) (L + 1) * d;
  const uint8_t* mb = mask + b * (int64_t) L;
  const int words = (bits + 31) >> 5;
  lsh_stage(R + b * r_stride, d * bits, sR);
  for (int e = threadIdx.x; e < bits + 2; e += blockDim.x) hist[e] = 0;
  __syncthreads();
  if (threadIdx.x < words) {
    const int w = threadIdx.x;
    tcode[w] = lsh_word(xb + (int64_t) L * d, sR, d, bits, 32 * w, min(32, bits - 32 * w));
  }
  __syncthreads();
  const uint32_t t0 = tcode[0], t1 = words > 1 ? tcode[1] : 0u;
  for (int l = threadIdx.x; l < L; l += blockDim.x) {
    int dl = bits + 1;
    if (mb[l]) {
      const float* v = xb + (int64_t) l * d;
      dl = __popc(lsh_word(v, sR, d, bits, 0, min(32, bits)) ^ t0);
      if (words > 1) dl += __popc(lsh_word(v, sR, d, bits, 32, bits - 32) ^ t1);
    }
    dist[l] = (uint8_t) dl;
    atomicAdd(hist + dl, 1);
  }
  __syncthreads();
  if (threadIdx.x < 32) {
    const int lane = threadIdx.x;
    if (lane == 0) {               // exclusive prefix: the first output slot of each distance
      int run = 0;
      for (int e = 0; e < bits + 2; ++e) {
        const int c = hist[e];
        hist[e] = run;
        run += c;
      }
    }
    __syncwarp();
    const uint32_t lt = (1u << lane) - 1u;
    for (int c0 = 0; c0 < L; c0 += 32) {
      const int l = c0 + lane;
      const int dl = l < L ? dist[l] : 255;
      const uint32_t peers = __match_any_sync(0xffffffffu, dl);
      if (l < L) {
        const int slot = hist[dl] + __popc(peers & lt);
        if (slot < k) spos[slot] = l;
      }
      __syncwarp();
      if (l < L && (peers & lt) == 0) hist[dl] += __popc(peers);
      __syncwarp();
    }
  }
  __syncthreads();
  for (int s = threadIdx.x; s < k; s += blockDim.x) {
    const int p = spos[s];
    topk_pos[b * k + s] = p;
    topk_mask[b * k + s] = mb[p] != 0;
  }
  float* ob = topk_emb + b * (int64_t) k * d;
  for (int e = threadIdx.x; e < k * d; e += blockDim.x) {
    const int s = e / d, i = e - s * d;
    ob[e] = xb[(int64_t) spos[s] * d + i];
  }
}

static size_t eta_smem(int L, int d, int bits, int k) {
  return (size_t) d * bits * 4 + (size_t) k * 4 + (size_t) (bits + 2) * 4 + 8 + (size_t) L;
}

extern "C" B2_API int b2_eta_retrieve_fwd(const float* x, const uint8_t* mask, const float* R, int64_t r_stride,
                                          int64_t batch, int L, int d, int bits, int k, float* topk_emb,
                                          uint8_t* topk_mask, int32_t* topk_pos, void* stream) {
  if (int rc = lsh_check(batch, L, d)) return rc;
  B2_REQUIRE(x && mask && R && topk_emb && topk_mask && topk_pos, "NULL pointer");
  B2_REQUIRE(bits >= 1 && bits <= B2_ETA_MAX_BITS, "ETA: hash_bits must lie in [1, %d], got %d", B2_ETA_MAX_BITS,
             bits);
  B2_REQUIRE(k >= 1 && k <= L && k <= B2_LSH_MAX_TOPK, "ETA: k must lie in [1, min(L, %d)], got %d (L = %d)",
             B2_LSH_MAX_TOPK, k, L);
  B2_REQUIRE(r_stride == 0 || r_stride >= (int64_t) d * bits, "ETA: r_stride must be 0 or >= d bits");
  if (batch == 0) return B2_OK;
  const size_t smem = eta_smem(L, d, bits, k);
  B2_REQUIRE(smem <= B2_LSH_MAX_SMEM, "ETA: d hash_bits = %d needs more shared memory than a CTA has", d * bits);
  B2_REQUIRE(cudaFuncSetAttribute(eta_retrieve_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) smem) ==
                 cudaSuccess, "ETA: cannot reserve %zu bytes of shared memory", smem);
  B2_LAUNCH(eta_retrieve_kernel, (unsigned) batch, LSH_THREADS, smem, (cudaStream_t) stream, x, mask, R, r_stride, L,
            d, bits, k, topk_emb, topk_mask, topk_pos);
  B2_CUDA_LAUNCH_CHECK("b2_eta_retrieve_fwd");
  return B2_OK;
}

// ---------------------------------------------------------------------------------------------------------------
// SDIM pooling
// shared: R (d nh bits) f32 | part (G nh d) f32 | tcode (nh) u32 | words (L) u32
__global__ void __launch_bounds__(LSH_THREADS)
sdim_pool_kernel(const float* __restrict__ x, const uint8_t* __restrict__ mask, const float* __restrict__ R,
                 int64_t r_stride, int L, int d, int nh, int bits, int l2norm, float* __restrict__ out,
                 float* __restrict__ sums, uint32_t* __restrict__ collide) {
  extern __shared__ float smem[];
  b2_pdl_wait();
  const int G = blockDim.x / d;             // column groups: thread t sums column t % d over positions = t / d mod G
  float* sR = smem;
  float* part = sR + d * nh * bits;
  uint32_t* tcode = (uint32_t*) (part + G * nh * d);
  uint32_t* cw = tcode + nh;
  const int64_t b = blockIdx.x;
  const float* xb = x + b * (int64_t) (L + 1) * d;
  const uint8_t* mb = mask + b * (int64_t) L;
  const int ldr = nh * bits;
  lsh_stage(R + b * r_stride, d * ldr, sR);
  __syncthreads();
  if (threadIdx.x < nh) tcode[threadIdx.x] = lsh_word(xb + (int64_t) L * d, sR, d, ldr, threadIdx.x * bits, bits);
  __syncthreads();
  for (int l = threadIdx.x; l < L; l += blockDim.x) {
    uint32_t w = 0;
    if (mb[l]) {
      const float* v = xb + (int64_t) l * d;
      for (int h = 0; h < nh; ++h)
        if (lsh_word(v, sR, d, ldr, h * bits, bits) == tcode[h]) w |= 1u << h;
    }
    cw[l] = w;
    collide[b * L + l] = w;
  }
  __syncthreads();
  const int t = threadIdx.x, i = t % d, g = t / d;
  if (g < G) {
    float* pg = part + g * nh * d;
    for (int h = 0; h < nh; ++h) pg[h * d + i] = 0.f;
    for (int l = g; l < L; l += G) {
      const uint32_t w = cw[l];
      if (w) {
        const float v = xb[(int64_t) l * d + i];
        for (int h = 0; h < nh; ++h)
          if (w >> h & 1u) pg[h * d + i] += v;
      }
    }
  }
  __syncthreads();
  for (int e = t; e < nh * d; e += blockDim.x) {
    float s = 0.f;
    for (int q = 0; q < G; ++q) s += part[q * nh * d + e];
    part[e] = s;                            // group 0's slot: only this thread reads or writes column e from here
    sums[b * nh * d + e] = s;
  }
  __syncthreads();
  __shared__ float inv[32];
  if (l2norm) {
    for (int h = t >> 5; h < nh; h += LSH_WARPS) {
      float q = 0.f;
      for (int c = t & 31; c < d; c += 32) q = fmaf(part[h * d + c], part[h * d + c], q);
      q = b2_warp_sum(q);
      if ((t & 31) == 0) inv[h] = 1.f / fmaxf(sqrtf(q), 1e-12f);
    }
    __syncthreads();
  }
  for (int c = t; c < d; c += blockDim.x) {
    float s = 0.f;
    for (int h = 0; h < nh; ++h) s += l2norm ? part[h * d + c] * inv[h] : part[h * d + c];
    out[b * d + c] = s / (float) nh;
  }
}

static int sdim_check(int64_t batch, int L, int d, int nh, int bits) {
  if (int rc = lsh_check(batch, L, d)) return rc;
  B2_REQUIRE(nh >= 1 && nh <= B2_SDIM_MAX_HASHES, "SDIM: num_hashes must lie in [1, %d], got %d", B2_SDIM_MAX_HASHES,
             nh);
  B2_REQUIRE(bits >= 1 && bits <= B2_SDIM_MAX_BITS, "SDIM: hash_bits must lie in [1, %d], got %d", B2_SDIM_MAX_BITS,
             bits);
  return B2_OK;
}

static size_t sdim_smem(int L, int d, int nh, int bits) {
  const int G = LSH_THREADS / d;
  return (size_t) d * nh * bits * 4 + (size_t) G * nh * d * 4 + (size_t) nh * 4 + (size_t) L * 4;
}

extern "C" B2_API int b2_sdim_pool_fwd(const float* x, const uint8_t* mask, const float* R, int64_t r_stride,
                                       int64_t batch, int L, int d, int num_hashes, int bits, int l2norm, float* out,
                                       float* sums, uint32_t* collide, void* stream) {
  if (int rc = sdim_check(batch, L, d, num_hashes, bits)) return rc;
  B2_REQUIRE(x && mask && R && out && sums && collide, "NULL pointer");
  B2_REQUIRE(r_stride == 0 || r_stride >= (int64_t) d * num_hashes * bits,
             "SDIM: r_stride must be 0 or >= d num_hashes hash_bits");
  if (batch == 0) return B2_OK;
  const size_t smem = sdim_smem(L, d, num_hashes, bits);
  B2_REQUIRE(smem <= B2_LSH_MAX_SMEM, "SDIM: d num_hashes hash_bits = %d needs more shared memory than a CTA has",
             d * num_hashes * bits);
  B2_REQUIRE(cudaFuncSetAttribute(sdim_pool_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) smem) ==
                 cudaSuccess, "SDIM: cannot reserve %zu bytes of shared memory", smem);
  B2_LAUNCH(sdim_pool_kernel, (unsigned) batch, LSH_THREADS, smem, (cudaStream_t) stream, x, mask, R, r_stride, L, d,
            num_hashes, bits, l2norm, out, sums, collide);
  B2_CUDA_LAUNCH_CHECK("b2_sdim_pool_fwd");
  return B2_OK;
}

// ---------------------------------------------------------------------------------------------------------------
// Gradient assembly.  Rows [0, L): the short window's gradient on rows [L - S, L), plus the long interest's.  Row L:
// dt0 + dt1 + dt2.  ETA: long = the retrieved rows' gradient dlong (B, k, d) at their positions, through an inverse map
// in shared memory.  SDIM: long = sum over the hashes h that position l collides in of u_h, u_h the gradient of the
// pooled vector with respect to sum h: g / nh, times the normalize Jacobian (g - v (v . g)) / |s| when |s| >= eps, or
// g / eps below it (F.normalize's clamp_min).
// shared ETA: inv (L) i32; SDIM: u (nh d) f32 | words (L) u32 | scratch
__global__ void __launch_bounds__(LSH_THREADS)
lsh_assemble_kernel(const float* __restrict__ dt0, const float* __restrict__ dt1, const float* __restrict__ dt2,
                    const float* __restrict__ dshort, int S, const float* __restrict__ dlong,
                    const int32_t* __restrict__ pos, int k, const float* __restrict__ sums,
                    const uint32_t* __restrict__ collide, int nh, int l2norm, int L, int d, float* __restrict__ dx) {
  extern __shared__ float smem[];
  __shared__ float coef[32][2];
  b2_pdl_wait();
  const int64_t b = blockIdx.x;
  const int t = threadIdx.x;
  const bool eta = pos != nullptr;
  int32_t* inv = (int32_t*) smem;
  float* u = smem;
  uint32_t* cw = (uint32_t*) (smem + nh * d);
  if (eta) {
    for (int l = t; l < L; l += blockDim.x) inv[l] = -1;
    __syncthreads();
    for (int s = t; s < k; s += blockDim.x) inv[pos[b * k + s]] = s;
  } else {
    const float* g = dlong + b * d;
    const float* sb = sums + b * (int64_t) nh * d;
    if (l2norm) {                           // per hash: |s| and v . g, one warp each
      for (int h = t >> 5; h < nh; h += LSH_WARPS) {
        float q = 0.f, p = 0.f;
        for (int c = t & 31; c < d; c += 32) {
          const float s = sb[h * d + c];
          q = fmaf(s, s, q);
          p = fmaf(s, g[c], p);
        }
        q = b2_warp_sum(q);
        p = b2_warp_sum(p);
        if ((t & 31) == 0) {
          const float n = sqrtf(q);
          coef[h][0] = n;
          coef[h][1] = p;
        }
      }
      __syncthreads();
    }
    const float inh = 1.f / (float) nh;
    for (int e = t; e < nh * d; e += blockDim.x) {
      const int h = e / d, c = e - h * d;
      float v = g[c] * inh;
      if (l2norm) {
        const float n = coef[h][0];
        if (n >= 1e-12f) {
          const float in = 1.f / n;
          v = (g[c] - sb[e] * in * (coef[h][1] * in)) * in * inh;
        } else {
          v = g[c] * 1e12f * inh;
        }
      }
      u[e] = v;
    }
    for (int l = t; l < L; l += blockDim.x) cw[l] = collide[b * L + l];
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
      if (eta) {
        const int s = inv[l];
        if (s >= 0) v += dlong[(b * k + s) * (int64_t) d + c];
      } else {
        const uint32_t w = cw[l];
        for (int h = 0; h < nh; ++h)
          if (w >> h & 1u) v += u[h * d + c];
      }
    }
    ob[e] = v;
  }
}

static int lsh_assemble_check(int64_t batch, int L, int d, int S, const float* dt0, const float* dt1,
                              const float* dt2, const float* dshort, const float* dlong, float* dx) {
  if (int rc = lsh_check(batch, L, d)) return rc;
  B2_REQUIRE(dt0 && dt1 && dt2 && dshort && dlong && dx, "NULL pointer");
  B2_REQUIRE(S >= 1 && S <= L, "LSH: the short window S must lie in [1, L], got %d (L = %d)", S, L);
  return B2_OK;
}

extern "C" B2_API int b2_eta_assemble_bwd(const float* dt0, const float* dt1, const float* dt2, const float* dshort,
                                          int S, const float* dlong, const int32_t* pos, int64_t batch, int L, int d,
                                          int k, float* dx, void* stream) {
  if (int rc = lsh_assemble_check(batch, L, d, S, dt0, dt1, dt2, dshort, dlong, dx)) return rc;
  B2_REQUIRE(pos, "NULL pointer");
  B2_REQUIRE(k >= 1 && k <= L && k <= B2_LSH_MAX_TOPK, "ETA: k must lie in [1, min(L, %d)], got %d (L = %d)",
             B2_LSH_MAX_TOPK, k, L);
  if (batch == 0) return B2_OK;
  const size_t smem = (size_t) L * 4;
  // the kernel is shared with b2_sdim_assemble_bwd: each entry point sets the dynamic shared memory limit it needs
  B2_REQUIRE(cudaFuncSetAttribute(lsh_assemble_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) smem) ==
                 cudaSuccess, "ETA: cannot reserve %zu bytes of shared memory", smem);
  B2_LAUNCH(lsh_assemble_kernel, (unsigned) batch, LSH_THREADS, smem, (cudaStream_t) stream, dt0, dt1, dt2, dshort, S,
            dlong, pos, k, (const float*) nullptr, (const uint32_t*) nullptr, 0, 0, L, d, dx);
  B2_CUDA_LAUNCH_CHECK("b2_eta_assemble_bwd");
  return B2_OK;
}

extern "C" B2_API int b2_sdim_assemble_bwd(const float* dt0, const float* dt1, const float* dt2, const float* dshort,
                                           int S, const float* dlong, const float* sums, const uint32_t* collide,
                                           int64_t batch, int L, int d, int num_hashes, int l2norm, float* dx,
                                           void* stream) {
  if (int rc = lsh_assemble_check(batch, L, d, S, dt0, dt1, dt2, dshort, dlong, dx)) return rc;
  B2_REQUIRE(sums && collide, "NULL pointer");
  B2_REQUIRE(num_hashes >= 1 && num_hashes <= B2_SDIM_MAX_HASHES, "SDIM: num_hashes must lie in [1, %d], got %d",
             B2_SDIM_MAX_HASHES, num_hashes);
  if (batch == 0) return B2_OK;
  const size_t smem = (size_t) num_hashes * d * 4 + (size_t) L * 4;
  B2_REQUIRE(smem <= B2_LSH_MAX_SMEM, "SDIM: num_hashes d = %d needs more shared memory than a CTA has",
             num_hashes * d);
  B2_REQUIRE(cudaFuncSetAttribute(lsh_assemble_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) smem) ==
                 cudaSuccess, "SDIM: cannot reserve %zu bytes of shared memory", smem);
  B2_LAUNCH(lsh_assemble_kernel, (unsigned) batch, LSH_THREADS, smem, (cudaStream_t) stream, dt0, dt1, dt2, dshort, S,
            dlong, (const int32_t*) nullptr, 0, sums, collide, num_hashes, l2norm, L, d, dx);
  B2_CUDA_LAUNCH_CHECK("b2_sdim_assemble_bwd");
  return B2_OK;
}

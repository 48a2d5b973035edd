// target_attention.cu — MultiHeadTargetAttention (one query per sample over its history), sm_90a.
//
// Reference semantics (reczoo/FuxiCTR v2.3.10):
//   MultiHeadTargetAttention.forward   fuxictr/pytorch/layers/attentions/target_attention.py:137-172
//   ScaledDotProductAttention.forward  fuxictr/pytorch/layers/attentions/dot_product_attention.py:32-58
//
// With the projections (use_qkvo) the layer is linear in the history x_l everywhere but the softmax, so the
// projections fold into weight-only d x d products per head and the history is never projected:
//   score_hl = q'_h . x_l,  q' = t W_M^T            (W_M^T stacks s W_q,h^T W_k,h)
//   out      = p W_N^T,     p_h = sum_l a_hl x_l     (W_N   stacks W_o,h W_v,h)
// The two contractions with t and p are the wgmma GEMM (or the SIMT GEMM); this file holds what lies between
// them: the pack of W_M, W_N, the per-row attention kernel in both directions, and the scatter of the packed
// weight gradients back to W_q, W_k, W_v, W_o.  Without the projections the same row kernels run "sliced":
// head h reads columns [h*hd, (h+1)*hd) of t and x and the scale is applied in the kernel.
// Layouts: include/fuxictr_b200.h "MultiHeadTargetAttention".
//
// Row kernels: one warp per row.  The history is read in chunks of TA_CHUNK positions (16-byte loads when
// d % 4 == 0) into shared memory with an odd row pitch, so lane l computing position l's dot products walks
// its own bank.  The softmax is online (running max and sum per head), so any L works in one pass; the
// backward recomputes a_hl from the saved max and sum and uses sum_l a_hl da_hl = dp_h . p_h, so it too reads
// the history once.  expf (not __expf: its error would show at the layer's 1e-5 bar).
#include "b2_common.cuh"

#define TA_CHUNK 32                              // history positions per chunk: one per lane for the scores
#define TA_COLS (B2_MHTA_MAX_WIDTH / 32)         // per-row columns (q', p, dp, dq') per lane
#define TA_MAX_WARPS 8
#define TA_SMEM_TARGET (64 * 1024)               // warps per CTA are halved until the CTA fits this

__device__ __forceinline__ void ta_store_aux(void* aux, int aux_dtype, int64_t off, float v) {
  if (aux_dtype == B2_BF16) reinterpret_cast<__nv_bfloat16*>(aux)[off] = __float2bfloat16_rn(v);
  else reinterpret_cast<float*>(aux)[off] = b2_tf32_small(v);
}

__device__ __forceinline__ float ta_warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

__device__ __forceinline__ float ta_dot(const float* a, const float* b, int w) {
  float s = 0.f;
  for (int k = 0; k < w; ++k) s = fmaf(a[k], b[k], s);
  return s;
}

// count = n*d contiguous floats of the history -> sx[l * pitch + k]
__device__ __forceinline__ void ta_load_chunk(const float* __restrict__ src, int count, int d, int pitch, float* sx,
                                              bool vec) {
  const int lane = threadIdx.x & 31;
  if (vec) {
#pragma unroll 4
    for (int e = 4 * lane; e < count; e += 128) {
      const float4 v = b2_ldg_stream(reinterpret_cast<const float4*>(src + e));
      const int l = e / d;
      float* o = sx + l * pitch + (e - l * d);
      o[0] = v.x; o[1] = v.y; o[2] = v.z; o[3] = v.w;
    }
  } else {
#pragma unroll 4
    for (int e = lane; e < count; e += 32) {
      const int l = e / d;
      sx[l * pitch + (e - l * d)] = __ldg(src + e);
    }
  }
}

// Lane l's score of head h at chunk position l (valid: l < n; keep: not masked).
__device__ __forceinline__ float ta_score(const float* sq, const float* sx, int pitch, int h, int w, int xs,
                                          float scale, bool keep) {
  const int lane = threadIdx.x & 31;
  return keep ? scale * ta_dot(sq + h * w, sx + lane * pitch + h * xs, w) : -1.e9f;
}

static __host__ __device__ __forceinline__ int ta_fwd_warp_floats(int d, int H, int w) {
  return TA_CHUNK * (d | 1) + H * w + H * TA_CHUNK + 3 * H;
}
static __host__ __device__ __forceinline__ int ta_bwd_warp_floats(int d, int H, int w) {
  return TA_CHUNK * (d | 1) + 2 * H * w + 2 * H * TA_CHUNK + 3 * H;
}

// p (B, H*w) "=", stats (B, H, 2) "=" {running max m_h, sum l_h = sum_l exp(s_hl - m_h)}.
__global__ void __launch_bounds__(TA_MAX_WARPS * 32)
mhta_fwd_kernel(const float* __restrict__ q, const float* __restrict__ x, const uint8_t* __restrict__ mask,
                int64_t batch, int L, int d, int H, int w, int xs, float scale, float* __restrict__ p,
                float* __restrict__ stats, void* p_aux, int aux_dtype, int64_t ld_aux) {
  extern __shared__ float sm[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  const int HW = H * w, pitch = d | 1;
  float* sx = sm + warp * ta_fwd_warp_floats(d, H, w);   // TA_CHUNK x pitch
  float* sq = sx + TA_CHUNK * pitch;                      // H*w
  float* sa = sq + HW;                                    // H x TA_CHUNK: exp(s - m) of the chunk
  float* smax = sa + H * TA_CHUNK;                        // H
  float* ssum = smax + H;                                 // H
  float* salpha = ssum + H;                               // H: exp(m_old - m_new) of the chunk
  const bool vec = (d % 4 == 0) && ((reinterpret_cast<uintptr_t>(x) & 15) == 0);
  b2_pdl_wait();
  for (int64_t row = (int64_t) blockIdx.x * nw + warp; row < batch; row += (int64_t) gridDim.x * nw) {
    __syncwarp();
    for (int c = lane; c < HW; c += 32) sq[c] = __ldg(q + row * HW + c);
    if (lane == 0)
      for (int h = 0; h < H; ++h) { smax[h] = -INFINITY; ssum[h] = 0.f; }
    float acc[TA_COLS];
#pragma unroll
    for (int i = 0; i < TA_COLS; ++i) acc[i] = 0.f;
    const float* xrow = x + row * L * d;
    const uint8_t* mrow = mask ? mask + row * L : nullptr;
    for (int l0 = 0; l0 < L; l0 += TA_CHUNK) {
      const int n = min(TA_CHUNK, L - l0);
      __syncwarp();
      ta_load_chunk(xrow + (int64_t) l0 * d, n * d, d, pitch, sx, vec);
      __syncwarp();
      const bool valid = lane < n;
      const bool keep = valid && (mrow == nullptr || mrow[l0 + lane] != 0);
      for (int h = 0; h < H; ++h) {
        const float s = valid ? ta_score(sq, sx, pitch, h, w, xs, scale, keep) : -INFINITY;
        const float m_old = smax[h];
        const float m_new = fmaxf(m_old, ta_warp_max(s));
        const float a = valid ? expf(s - m_new) : 0.f;
        const float sum = b2_warp_sum(a);
        sa[h * TA_CHUNK + lane] = a;
        __syncwarp();
        if (lane == 0) {
          const float alpha = expf(m_old - m_new);
          salpha[h] = alpha;
          smax[h] = m_new;
          ssum[h] = ssum[h] * alpha + sum;
        }
      }
      __syncwarp();
#pragma unroll
      for (int i = 0; i < TA_COLS; ++i) {
        const int c = lane + 32 * i;
        if (c < HW) {
          const int h = c / w;
          const float* xc = sx + h * xs + (c - h * w);
          const float* ah = sa + h * TA_CHUNK;
          float v = acc[i] * salpha[h];
          for (int j = 0; j < n; ++j) v = fmaf(ah[j], xc[j * pitch], v);
          acc[i] = v;
        }
      }
    }
    __syncwarp();
#pragma unroll
    for (int i = 0; i < TA_COLS; ++i) {
      const int c = lane + 32 * i;
      if (c < HW) {
        const float v = acc[i] / ssum[c / w];
        p[row * HW + c] = v;
        if (p_aux) ta_store_aux(p_aux, aux_dtype, row * ld_aux + c, v);
      }
    }
    for (int h = lane; h < H; h += 32) {
      stats[(row * H + h) * 2] = smax[h];
      stats[(row * H + h) * 2 + 1] = ssum[h];
    }
  }
  b2_pdl_trigger();
}

// Backward per row, from q, x, mask, p, stats and dp:
//   a_hl = exp(s_hl - m_h) / l_h,  da_hl = dp_h . x_l,  ds_hl = a_hl (da_hl - dp_h . p_h) (0 where masked),
//   dx_l = sum_h (a_hl dp_h + scale ds_hl q_h) on head h's columns,  dq_h = scale sum_l ds_hl x_l.
__global__ void __launch_bounds__(TA_MAX_WARPS * 32)
mhta_bwd_kernel(const float* __restrict__ q, const float* __restrict__ x, const uint8_t* __restrict__ mask,
                const float* __restrict__ p, const float* __restrict__ stats, const float* __restrict__ dp,
                int64_t batch, int L, int d, int H, int w, int xs, float scale, float* __restrict__ dq,
                float* __restrict__ dx, void* dq_aux, int aux_dtype, int64_t ld_aux) {
  extern __shared__ float sm[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  const int HW = H * w, pitch = d | 1;
  float* sx = sm + warp * ta_bwd_warp_floats(d, H, w);   // TA_CHUNK x pitch
  float* sq = sx + TA_CHUNK * pitch;                      // H*w
  float* sdp = sq + HW;                                   // H*w
  float* sa = sdp + HW;                                   // H x TA_CHUNK: a_hl
  float* sds = sa + H * TA_CHUNK;                         // H x TA_CHUNK: scale * ds_hl
  float* smax = sds + H * TA_CHUNK;                       // H
  float* sinv = smax + H;                                 // H: 1 / l_h
  float* sD = sinv + H;                                   // H: dp_h . p_h
  const bool vec = (d % 4 == 0) && ((reinterpret_cast<uintptr_t>(x) & 15) == 0) &&
                   ((reinterpret_cast<uintptr_t>(dx) & 15) == 0);
  b2_pdl_wait();
  for (int64_t row = (int64_t) blockIdx.x * nw + warp; row < batch; row += (int64_t) gridDim.x * nw) {
    __syncwarp();
    for (int c = lane; c < HW; c += 32) {
      sq[c] = __ldg(q + row * HW + c);
      sdp[c] = __ldg(dp + row * HW + c);
    }
    for (int h = lane; h < H; h += 32) {
      smax[h] = __ldg(stats + (row * H + h) * 2);
      sinv[h] = 1.f / __ldg(stats + (row * H + h) * 2 + 1);
    }
    for (int h = 0; h < H; ++h) {
      float t = 0.f;
      for (int k = lane; k < w; k += 32) t = fmaf(__ldg(dp + row * HW + h * w + k), __ldg(p + row * HW + h * w + k), t);
      t = b2_warp_sum(t);
      if (lane == 0) sD[h] = t;
    }
    float acc[TA_COLS];
#pragma unroll
    for (int i = 0; i < TA_COLS; ++i) acc[i] = 0.f;
    const float* xrow = x + row * L * d;
    float* dxrow = dx + row * L * d;
    const uint8_t* mrow = mask ? mask + row * L : nullptr;
    for (int l0 = 0; l0 < L; l0 += TA_CHUNK) {
      const int n = min(TA_CHUNK, L - l0);
      __syncwarp();
      ta_load_chunk(xrow + (int64_t) l0 * d, n * d, d, pitch, sx, vec);
      __syncwarp();
      const bool valid = lane < n;
      const bool keep = valid && (mrow == nullptr || mrow[l0 + lane] != 0);
      for (int h = 0; h < H; ++h) {
        float a = 0.f, ds = 0.f;
        if (valid) {
          a = expf(ta_score(sq, sx, pitch, h, w, xs, scale, keep) - smax[h]) * sinv[h];
          if (keep) ds = scale * a * (ta_dot(sdp + h * w, sx + lane * pitch + h * xs, w) - sD[h]);
        }
        sa[h * TA_CHUNK + lane] = a;
        sds[h * TA_CHUNK + lane] = ds;
      }
      __syncwarp();
#pragma unroll
      for (int i = 0; i < TA_COLS; ++i) {
        const int c = lane + 32 * i;
        if (c < HW) {
          const int h = c / w;
          const float* xc = sx + h * xs + (c - h * w);
          const float* dh = sds + h * TA_CHUNK;
          float v = acc[i];
          for (int j = 0; j < n; ++j) v = fmaf(dh[j], xc[j * pitch], v);
          acc[i] = v;
        }
      }
      // dx of the chunk's n*d elements, 4 consecutive ones per lane when d % 4 == 0 (same position l)
      const int step = vec ? 4 : 1, count = n * d;
      for (int e = lane * step; e < count; e += 32 * step) {
        const int l = e / d, k0 = e - l * d;
        float v[4];
#pragma unroll
        for (int t = 0; t < 4; ++t) {
          const int k = k0 + t;
          float s = 0.f;
          if (t >= step) { v[t] = 0.f; continue; }
          if (xs == 0) {
            for (int h = 0; h < H; ++h)
              s = fmaf(sa[h * TA_CHUNK + l], sdp[h * w + k], fmaf(sds[h * TA_CHUNK + l], sq[h * w + k], s));
          } else {
            const int h = k / xs;
            if (h < H) s = fmaf(sa[h * TA_CHUNK + l], sdp[k], sds[h * TA_CHUNK + l] * sq[k]);
          }
          v[t] = s;
        }
        float* o = dxrow + (int64_t) l0 * d + e;
        if (vec) b2_stg_stream(reinterpret_cast<float4*>(o), make_float4(v[0], v[1], v[2], v[3]));
        else o[0] = v[0];
      }
    }
#pragma unroll
    for (int i = 0; i < TA_COLS; ++i) {
      const int c = lane + 32 * i;
      if (c < HW) {
        dq[row * HW + c] = acc[i];
        if (dq_aux) ta_store_aux(dq_aux, aux_dtype, row * ld_aux + c, acc[i]);
      }
    }
  }
  b2_pdl_trigger();
}

// W_M (H*d, d): W_M[h*d + j, i] = s sum_k Wq[h*hd + k, i] Wk[h*hd + k, j]
// W_N (d, H*d): W_N[j, h*d + i] = sum_k Wo[j, h*hd + k] Wv[h*hd + k, i]
__global__ void __launch_bounds__(256)
mhta_pack_kernel(const float* __restrict__ Wq, const float* __restrict__ Wk, const float* __restrict__ Wv,
                 const float* __restrict__ Wo, int d, int H, int hd, float scale, float* __restrict__ WM,
                 float* __restrict__ WN) {
  const int A = H * hd;
  const int64_t n_m = (int64_t) H * d * d, total = 2 * n_m;
  b2_pdl_wait();
  for (int64_t t = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (int64_t) gridDim.x * blockDim.x) {
    float s = 0.f;
    if (t < n_m) {
      const int r = (int) (t / d), i = (int) (t - (int64_t) r * d), h = r / d, j = r - h * d;
      for (int k = 0; k < hd; ++k)
        s = fmaf(__ldg(Wq + (int64_t) (h * hd + k) * d + i), __ldg(Wk + (int64_t) (h * hd + k) * d + j), s);
      WM[t] = scale * s;
    } else {
      const int64_t u = t - n_m;
      const int j = (int) (u / ((int64_t) H * d)), c = (int) (u - (int64_t) j * H * d), h = c / d, i = c - h * d;
      for (int k = 0; k < hd; ++k)
        s = fmaf(__ldg(Wo + (int64_t) j * A + h * hd + k), __ldg(Wv + (int64_t) (h * hd + k) * d + i), s);
      WN[u] = s;
    }
  }
  b2_pdl_trigger();
}

// gWq[h*hd + k, i] = s sum_j Wk[h*hd + k, j] dWM[h*d + j, i]     gWk[h*hd + k, j] = s sum_i Wq[h*hd + k, i] dWM[h*d + j, i]
// gWv[h*hd + k, i] = sum_j Wo[j, h*hd + k] dWN[j, h*d + i]       gWo[j, h*hd + k] = sum_i dWN[j, h*d + i] Wv[h*hd + k, i]
__global__ void __launch_bounds__(256)
mhta_unpack_kernel(const float* __restrict__ Wq, const float* __restrict__ Wk, const float* __restrict__ Wv,
                   const float* __restrict__ Wo, const float* __restrict__ dWM, const float* __restrict__ dWN, int d,
                   int H, int hd, float scale, float* __restrict__ gWq, float* __restrict__ gWk,
                   float* __restrict__ gWv, float* __restrict__ gWo) {
  const int A = H * hd, HD = H * d;
  const int64_t n = (int64_t) A * d, total = 4 * n;
  b2_pdl_wait();
  for (int64_t t = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (int64_t) gridDim.x * blockDim.x) {
    const int which = (int) (t / n);
    const int64_t u = t - which * n;
    float s = 0.f;
    if (which < 3) {           // (A, d) row-major: row r = h*hd + k, column c
      const int r = (int) (u / d), c = (int) (u - (int64_t) r * d), h = r / hd;
      if (which == 0) {
        for (int j = 0; j < d; ++j) s = fmaf(__ldg(Wk + (int64_t) r * d + j), __ldg(dWM + (int64_t) (h * d + j) * d + c), s);
        gWq[u] = scale * s;
      } else if (which == 1) {
        for (int i = 0; i < d; ++i) s = fmaf(__ldg(Wq + (int64_t) r * d + i), __ldg(dWM + (int64_t) (h * d + c) * d + i), s);
        gWk[u] = scale * s;
      } else {
        for (int j = 0; j < d; ++j) s = fmaf(__ldg(Wo + (int64_t) j * A + r), __ldg(dWN + (int64_t) j * HD + h * d + c), s);
        gWv[u] = s;
      }
    } else {                   // (d, A) row-major: row j, column r = h*hd + k
      const int j = (int) (u / A), r = (int) (u - (int64_t) j * A), h = r / hd;
      for (int i = 0; i < d; ++i) s = fmaf(__ldg(dWN + (int64_t) j * HD + h * d + i), __ldg(Wv + (int64_t) r * d + i), s);
      gWo[u] = s;
    }
  }
  b2_pdl_trigger();
}

// ---------------------------------------------------------------------------------
// Host side
// ---------------------------------------------------------------------------------
static int ta_check_rows(int64_t batch, int L, int d, int H, int w, int xs) {
  B2_REQUIRE(batch >= 0, "negative batch");
  B2_REQUIRE(L >= 1, "history length %d < 1", L);
  B2_REQUIRE(batch * (int64_t) L <= INT32_MAX, "batch * history length %lld exceeds the int32 bound",
             (long long) (batch * (int64_t) L));
  B2_REQUIRE(H >= 1 && H <= B2_MHTA_MAX_HEADS, "heads %d outside [1, %d]", H, B2_MHTA_MAX_HEADS);
  B2_REQUIRE(w >= 1 && (int64_t) H * w <= B2_MHTA_MAX_WIDTH, "heads * width = %lld outside [1, %d]",
             (long long) H * w, B2_MHTA_MAX_WIDTH);
  B2_REQUIRE(d >= 1 && d <= B2_MHTA_MAX_WIDTH, "input_dim %d outside [1, %d]", d, B2_MHTA_MAX_WIDTH);
  B2_REQUIRE(xs == 0 || xs == w, "x_step %d must be 0 (folded) or the head width %d (sliced)", xs, w);
  B2_REQUIRE((int64_t) xs * (H - 1) + w <= d, "the heads' columns exceed input_dim %d", d);
  return B2_OK;
}

static int ta_check_weights(int d, int H, int hd) {
  B2_REQUIRE(H >= 1 && H <= B2_MHTA_MAX_HEADS, "heads %d outside [1, %d]", H, B2_MHTA_MAX_HEADS);
  B2_REQUIRE(d >= 1 && (int64_t) H * d <= B2_MHTA_MAX_WIDTH, "heads * input_dim = %lld outside [1, %d]",
             (long long) H * d, B2_MHTA_MAX_WIDTH);
  B2_REQUIRE(hd >= 1, "head_dim %d < 1", hd);
  B2_REQUIRE((int64_t) H * hd * d <= INT32_MAX, "heads * head_dim * input_dim exceeds the int32 bound");
  return B2_OK;
}

static int ta_check_aux(const void* aux, int aux_dtype, int64_t ld_aux, int width) {
  if (aux == nullptr) return B2_OK;
  B2_REQUIRE(aux_dtype == B2_F32 || aux_dtype == B2_BF16, "aux_dtype must be B2_F32 or B2_BF16");
  B2_REQUIRE(ld_aux >= width, "ld_aux %lld < row width %d", (long long) ld_aux, width);
  return B2_OK;
}

static int ta_grid(int64_t blocks, int per_sm) {
  const int64_t cap = (int64_t) B2_NUM_SMS * per_sm;
  return (int) (blocks < 1 ? 1 : (blocks > cap ? cap : blocks));
}

// Warps per CTA: TA_MAX_WARPS, halved while the CTA's shared memory exceeds TA_SMEM_TARGET (one warp at least).
static int ta_warps(int warp_floats) {
  int nw = TA_MAX_WARPS;
  while (nw > 1 && (size_t) nw * warp_floats * sizeof(float) > TA_SMEM_TARGET) nw >>= 1;
  return nw;
}

template <typename K>
static void ta_smem_attr(K kernel, size_t smem) {
  if (smem > 48 * 1024) cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) smem);
}

extern "C" B2_API int b2_mhta_pack(const float* Wq, const float* Wk, const float* Wv, const float* Wo, int d,
                                   int heads, int head_dim, float scale, float* WM, float* WN, void* stream) {
  B2_REQUIRE(Wq && Wk && Wv && Wo && WM && WN, "NULL pointer");
  if (int rc = ta_check_weights(d, heads, head_dim)) return rc;
  const int64_t total = 2 * (int64_t) heads * d * d;
  B2_LAUNCH(mhta_pack_kernel, ta_grid(b2_ceil_div(total, 256), 8), 256, 0, (cudaStream_t) stream,
            Wq, Wk, Wv, Wo, d, heads, head_dim, scale, WM, WN);
  B2_CUDA_LAUNCH_CHECK("b2_mhta_pack");
  return B2_OK;
}

extern "C" B2_API int b2_mhta_fwd(const float* q, const float* x, const uint8_t* mask, int64_t batch, int L, int d,
                                  int heads, int width, int x_step, float scale, float* p, float* stats,
                                  void* p_aux, int aux_dtype, int64_t ld_aux, void* stream) {
  B2_REQUIRE(q && x && p && stats, "NULL pointer");
  if (int rc = ta_check_rows(batch, L, d, heads, width, x_step)) return rc;
  if (int rc = ta_check_aux(p_aux, aux_dtype, ld_aux, heads * width)) return rc;
  if (batch == 0) return B2_OK;
  const int wf = ta_fwd_warp_floats(d, heads, width), nw = ta_warps(wf);
  const size_t smem = (size_t) nw * wf * sizeof(float);
  ta_smem_attr(mhta_fwd_kernel, smem);
  B2_LAUNCH(mhta_fwd_kernel, ta_grid(b2_ceil_div(batch, nw), 16), nw * 32, smem, (cudaStream_t) stream,
            q, x, mask, batch, L, d, heads, width, x_step, scale, p, stats, p_aux, aux_dtype, ld_aux);
  B2_CUDA_LAUNCH_CHECK("b2_mhta_fwd");
  return B2_OK;
}

extern "C" B2_API int b2_mhta_bwd(const float* q, const float* x, const uint8_t* mask, const float* p,
                                  const float* stats, const float* dp, int64_t batch, int L, int d, int heads,
                                  int width, int x_step, float scale, float* dq, float* dx, void* dq_aux,
                                  int aux_dtype, int64_t ld_aux, void* stream) {
  B2_REQUIRE(q && x && p && stats && dp && dq && dx, "NULL pointer");
  if (int rc = ta_check_rows(batch, L, d, heads, width, x_step)) return rc;
  if (int rc = ta_check_aux(dq_aux, aux_dtype, ld_aux, heads * width)) return rc;
  if (batch == 0) return B2_OK;
  const int wf = ta_bwd_warp_floats(d, heads, width), nw = ta_warps(wf);
  const size_t smem = (size_t) nw * wf * sizeof(float);
  ta_smem_attr(mhta_bwd_kernel, smem);
  B2_LAUNCH(mhta_bwd_kernel, ta_grid(b2_ceil_div(batch, nw), 16), nw * 32, smem, (cudaStream_t) stream,
            q, x, mask, p, stats, dp, batch, L, d, heads, width, x_step, scale, dq, dx, dq_aux, aux_dtype, ld_aux);
  B2_CUDA_LAUNCH_CHECK("b2_mhta_bwd");
  return B2_OK;
}

extern "C" B2_API int b2_mhta_unpack(const float* Wq, const float* Wk, const float* Wv, const float* Wo,
                                     const float* dWM, const float* dWN, int d, int heads, int head_dim, float scale,
                                     float* gWq, float* gWk, float* gWv, float* gWo, void* stream) {
  B2_REQUIRE(Wq && Wk && Wv && Wo && dWM && dWN && gWq && gWk && gWv && gWo, "NULL pointer");
  if (int rc = ta_check_weights(d, heads, head_dim)) return rc;
  const int64_t total = 4 * (int64_t) heads * head_dim * d;
  B2_LAUNCH(mhta_unpack_kernel, ta_grid(b2_ceil_div(total, 256), 8), 256, 0, (cudaStream_t) stream,
            Wq, Wk, Wv, Wo, dWM, dWN, d, heads, head_dim, scale, gWq, gWk, gWv, gWo);
  B2_CUDA_LAUNCH_CHECK("b2_mhta_unpack");
  return B2_OK;
}

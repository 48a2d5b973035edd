// attention.cu — Dice activation and the non-GEMM parts of DIN target attention, sm_90a.
//
// Reference semantics (reczoo/FuxiCTR v2.3.10):
//   Dice.forward           fuxictr/pytorch/layers/activations.py:37,49-50
//       p = sigmoid(BatchNorm1d(affine=False, eps=1e-9, momentum=0.01)(x));  out = p*x + alpha*(1-p)*x
//   DIN_Attention.forward  fuxictr/pytorch/layers/attentions/target_attention.py:79-92
//       att_in = cat([t, h, t-h, t*h], -1)  ->  MLP (our GEMM + Dice)  ->  w * mask  ->  sum_l w*h
//
// HBM-bound elementwise + column/row reductions: no tensor cores.  Train-mode Dice needs batch
// statistics over all B*L rows: a column-statistics pass (fp64 block partials, one atomic per
// column per CTA) followed by one elementwise pass; the backward mirrors it.
#include "bn_common.cuh"

namespace {
// ---- column sums of up to three derived quantities -------------------------------------------------
// stats[0*C + c] += sum_m q0(m,c), stats[1*C+c] += sum_m q1, stats[2*C+c] += sum_m q2   (fp64)
// MODE 0: q0 = x, q1 = x*x                                   (forward: mean / variance)
// MODE 1: q0 = u, q1 = u*xhat, q2 = g*x*(1-p)                (backward), u = g*x*(1-alpha)*p*(1-p)
template <int MODE>
__global__ void __launch_bounds__(256)
dice_stats_kernel(const float* __restrict__ x, const float* __restrict__ g,
                  const float* __restrict__ mean, const float* __restrict__ rstd,
                  const float* __restrict__ alpha, int64_t M, int C, int64_t rows_per_cta,
                  double* __restrict__ stats) {
  __shared__ double sm[3][8][33];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int c = blockIdx.x * 32 + tx;
  const int64_t r0 = (int64_t) blockIdx.y * rows_per_cta;
  const int64_t r1 = min(M, r0 + rows_per_cta);
  double a0 = 0.0, a1 = 0.0, a2 = 0.0;
  if (c < C) {
    float mu = 0.f, rs = 0.f, al = 0.f;
    if (MODE == 1) { mu = mean[c]; rs = rstd[c]; al = alpha[c]; }
    for (int64_t m = r0 + ty; m < r1; m += 8) {
      const float xv = __ldg(x + m * C + c);
      if (MODE == 0) {
        a0 += (double) xv;
        a1 += (double) xv * (double) xv;
      } else {
        const float gv = __ldg(g + m * C + c);
        const float xhat = (xv - mu) * rs;
        const float p = 1.f / (1.f + expf(-xhat));
        const float u = gv * xv * (1.f - al) * (p * (1.f - p));
        a0 += (double) u;
        a1 += (double) u * (double) xhat;
        a2 += (double) (gv * xv * (1.f - p));
      }
    }
  }
  sm[0][ty][tx] = a0; sm[1][ty][tx] = a1; sm[2][ty][tx] = a2;
  __syncthreads();
  if (ty < 3 && c < C && (MODE == 1 || ty < 2)) {
    double t = 0.0;
#pragma unroll
    for (int i = 0; i < 8; ++i) t += sm[ty][i][tx];
    atomicAdd(stats + (int64_t) ty * C + c, t);
  }
}

// mean/rstd from the sums; running statistics updated like nn.BatchNorm1d (unbiased variance).
__global__ void dice_finalize_kernel(const double* __restrict__ stats, int64_t M, int C, float eps,
                                     float momentum, float* __restrict__ mean, float* __restrict__ rstd,
                                     float* __restrict__ running_mean, float* __restrict__ running_var) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  b2_bn_finalize(stats[c], stats[C + c], M, eps, momentum, mean + c, rstd + c,
                 running_mean != nullptr ? running_mean + c : nullptr, running_mean != nullptr ? running_var + c : nullptr);
}

// eval mode: normalise with the running statistics
__global__ void dice_eval_stats_kernel(const float* __restrict__ rm, const float* __restrict__ rv, int C,
                                       float eps, float* __restrict__ mean, float* __restrict__ rstd) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c < C) {
    mean[c] = rm[c];
    rstd[c] = 1.f / sqrtf(rv[c] + eps);
  }
}

__global__ void __launch_bounds__(256)
dice_fwd_kernel(const float* __restrict__ x, const float* __restrict__ mean,
                const float* __restrict__ rstd, const float* __restrict__ alpha, int64_t n, int C,
                float* __restrict__ out) {
  for (int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (int64_t) gridDim.x * blockDim.x) {
    const int c = (int) (i % C);
    const float xv = __ldg(x + i);
    const float p = 1.f / (1.f + expf(-(xv - mean[c]) * rstd[c]));
    out[i] = p * xv + alpha[c] * (1.f - p) * xv;   // activations.py:50
  }
}

// gx = g*s + rstd*(u - [train] (mean_u + xhat*mean_uxhat)),  s = p + alpha*(1-p)
__global__ void __launch_bounds__(256)
dice_bwd_kernel(const float* __restrict__ x, const float* __restrict__ g,
                const float* __restrict__ mean, const float* __restrict__ rstd,
                const float* __restrict__ alpha, const double* __restrict__ stats, int64_t M, int C,
                int training, float* __restrict__ gx) {
  const int64_t n = M * C;
  for (int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (int64_t) gridDim.x * blockDim.x) {
    const int c = (int) (i % C);
    const float xv = __ldg(x + i), gv = __ldg(g + i);
    const float rs = rstd[c], al = alpha[c];
    const float xhat = (xv - mean[c]) * rs;
    const float p = 1.f / (1.f + expf(-xhat));
    const float u = gv * xv * (1.f - al) * (p * (1.f - p));
    float du = u;
    if (training) du -= (float) (stats[c] / (double) M) + xhat * (float) (stats[C + c] / (double) M);
    gx[i] = gv * (p + al * (1.f - p)) + rs * du;
  }
}

__global__ void dice_galpha_kernel(const double* __restrict__ stats, int C, float* __restrict__ galpha) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c < C) galpha[c] = (float) stats[2 * C + c];
}

// ---- DIN attention glue ---------------------------------------------------------------------------------
// att_in[(b,l), :] = [t, h, t-h, t*h]   (target_attention.py:81-82)
__global__ void __launch_bounds__(256)
din_input_fwd_kernel(const float* __restrict__ target, const float* __restrict__ hist, int64_t B, int L,
                     int d, float* __restrict__ out) {
  const int64_t n = B * (int64_t) L * d;
  for (int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (int64_t) gridDim.x * blockDim.x) {
    const int64_t bl = i / d;
    const int c = (int) (i - bl * d);
    const int64_t b = bl / L;
    const float t = __ldg(target + b * d + c), h = __ldg(hist + i);
    float* o = out + bl * 4 * d;
    o[c] = t; o[d + c] = h; o[2 * d + c] = t - h; o[3 * d + c] = t * h;
  }
}

// ghist[(b,l),c] (+)= g1 - g2 + g3*t ;  gtarget[b,c] = sum_l (g0 + g2 + g3*h)
__global__ void __launch_bounds__(256)
din_input_bwd_kernel(const float* __restrict__ target, const float* __restrict__ hist,
                     const float* __restrict__ gin, int64_t B, int L, int d,
                     float* __restrict__ gtarget, float* __restrict__ ghist, int accumulate_hist) {
  const int64_t n = B * (int64_t) d;
  for (int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (int64_t) gridDim.x * blockDim.x) {
    const int64_t b = i / d;
    const int c = (int) (i - b * d);
    const float t = __ldg(target + i);
    float gt = 0.f;
    for (int l = 0; l < L; ++l) {
      const int64_t bl = b * L + l;
      const float* gi = gin + bl * 4 * d;
      const float h = __ldg(hist + bl * d + c);
      const float g0 = __ldg(gi + c), g1 = __ldg(gi + d + c), g2 = __ldg(gi + 2 * d + c), g3 = __ldg(gi + 3 * d + c);
      gt += g0 + g2 + g3 * h;
      const float gh = g1 - g2 + g3 * t;
      if (accumulate_hist) ghist[bl * d + c] += gh; else ghist[bl * d + c] = gh;
    }
    gtarget[i] = gt;
  }
}

// out[b,c] = sum_l (w[b,l]*mask[b,l]) * hist[b,l,c]      (target_attention.py:85-86,91)
__global__ void __launch_bounds__(256)
din_wsum_fwd_kernel(const float* __restrict__ w, const unsigned char* __restrict__ mask,
                    const float* __restrict__ hist, int64_t B, int L, int d, float* __restrict__ out) {
  const int64_t n = B * (int64_t) d;
  for (int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (int64_t) gridDim.x * blockDim.x) {
    const int64_t b = i / d;
    const int c = (int) (i - b * d);
    float acc = 0.f;
    for (int l = 0; l < L; ++l) {
      float wv = __ldg(w + b * L + l);
      if (mask != nullptr) wv *= (float) mask[b * L + l];
      acc = fmaf(wv, __ldg(hist + (b * L + l) * d + c), acc);
    }
    out[i] = acc;
  }
}

// gw[b,l] = mask * sum_c gout[b,c]*hist[b,l,c] ;  ghist[b,l,c] = w*mask*gout[b,c]
__global__ void __launch_bounds__(256)
din_wsum_bwd_kernel(const float* __restrict__ w, const unsigned char* __restrict__ mask,
                    const float* __restrict__ hist, const float* __restrict__ gout, int64_t B, int L, int d,
                    float* __restrict__ gw, float* __restrict__ ghist) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t) blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t) gridDim.x * blockDim.x) >> 5;
  const int64_t nbl = B * (int64_t) L;
  for (int64_t bl = warp; bl < nbl; bl += nwarps) {
    const int64_t b = bl / L;
    const float m = (mask != nullptr) ? (float) mask[bl] : 1.f;
    const float wm = __ldg(w + bl) * m;
    float dot = 0.f;
    for (int c = lane; c < d; c += 32) {
      const float go = __ldg(gout + b * d + c);
      dot = fmaf(go, __ldg(hist + bl * d + c), dot);
      ghist[bl * d + c] = wm * go;
    }
    dot = b2_warp_sum(dot);
    if (lane == 0) gw[bl] = dot * m;
  }
}

int grid1d(int64_t n) {
  int64_t blocks = b2_ceil_div(n, 256);
  if (blocks > (int64_t) B2_NUM_SMS * 8) blocks = (int64_t) B2_NUM_SMS * 8;
  return (int) (blocks < 1 ? 1 : blocks);
}
}  // namespace

extern "C" B2_API int b2_dice_fwd(const float* x, const float* alpha, int64_t M, int C, float eps,
                                  float momentum, int training, float* running_mean, float* running_var,
                                  float* mean, float* rstd, double* stats_ws, float* out, void* stream) {
  B2_REQUIRE(x && alpha && mean && rstd && out, "NULL pointer");
  B2_REQUIRE(M >= 1 && C >= 1, "bad shape");
  cudaStream_t st = (cudaStream_t) stream;
  if (training) {
    B2_REQUIRE(stats_ws != nullptr, "training mode needs the fp64 workspace (3*C doubles)");
    cudaError_t e = cudaMemsetAsync(stats_ws, 0, sizeof(double) * 3 * C, st);
    if (e != cudaSuccess) return b2_fail(B2_E_CUDA, "b2_dice_fwd: memset: %s", cudaGetErrorString(e));
    const int64_t col_blocks = b2_ceil_div(C, 32);
    int64_t row_splits = b2_ceil_div(4 * B2_NUM_SMS, col_blocks);
    if (row_splits > b2_ceil_div(M, 64)) row_splits = b2_ceil_div(M, 64);
    const int64_t rows_per_cta = b2_ceil_div(M, row_splits);
    dim3 grid((unsigned) col_blocks, (unsigned) b2_ceil_div(M, rows_per_cta));
    dice_stats_kernel<0><<<grid, 256, 0, st>>>(x, nullptr, nullptr, nullptr, nullptr, M, C, rows_per_cta, stats_ws);
    dice_finalize_kernel<<<(C + 127) / 128, 128, 0, st>>>(stats_ws, M, C, eps, momentum, mean, rstd, running_mean, running_var);
  } else {
    B2_REQUIRE(running_mean && running_var, "eval mode needs running statistics");
    dice_eval_stats_kernel<<<(C + 127) / 128, 128, 0, st>>>(running_mean, running_var, C, eps, mean, rstd);
  }
  dice_fwd_kernel<<<grid1d(M * C), 256, 0, st>>>(x, mean, rstd, alpha, M * C, C, out);
  B2_CUDA_LAUNCH_CHECK("b2_dice_fwd");
  return B2_OK;
}

extern "C" B2_API int b2_dice_bwd(const float* x, const float* gout, const float* alpha, const float* mean,
                                  const float* rstd, int64_t M, int C, int training, double* stats_ws,
                                  float* gx, float* galpha, void* stream) {
  B2_REQUIRE(x && gout && alpha && mean && rstd && stats_ws && gx && galpha, "NULL pointer");
  B2_REQUIRE(M >= 1 && C >= 1, "bad shape");
  cudaStream_t st = (cudaStream_t) stream;
  cudaError_t e = cudaMemsetAsync(stats_ws, 0, sizeof(double) * 3 * C, st);
  if (e != cudaSuccess) return b2_fail(B2_E_CUDA, "b2_dice_bwd: memset: %s", cudaGetErrorString(e));
  const int64_t col_blocks = b2_ceil_div(C, 32);
  int64_t row_splits = b2_ceil_div(4 * B2_NUM_SMS, col_blocks);
  if (row_splits > b2_ceil_div(M, 64)) row_splits = b2_ceil_div(M, 64);
  const int64_t rows_per_cta = b2_ceil_div(M, row_splits);
  dim3 grid((unsigned) col_blocks, (unsigned) b2_ceil_div(M, rows_per_cta));
  dice_stats_kernel<1><<<grid, 256, 0, st>>>(x, gout, mean, rstd, alpha, M, C, rows_per_cta, stats_ws);
  dice_bwd_kernel<<<grid1d(M * C), 256, 0, st>>>(x, gout, mean, rstd, alpha, stats_ws, M, C, training, gx);
  dice_galpha_kernel<<<(C + 127) / 128, 128, 0, st>>>(stats_ws, C, galpha);
  B2_CUDA_LAUNCH_CHECK("b2_dice_bwd");
  return B2_OK;
}

extern "C" B2_API int b2_din_input_fwd(const float* target, const float* hist, int64_t B, int L, int d,
                                       float* out, void* stream) {
  B2_REQUIRE(target && hist && out, "NULL pointer");
  if (B <= 0) return B2_OK;
  din_input_fwd_kernel<<<grid1d(B * L * d), 256, 0, (cudaStream_t) stream>>>(target, hist, B, L, d, out);
  B2_CUDA_LAUNCH_CHECK("b2_din_input_fwd");
  return B2_OK;
}

extern "C" B2_API int b2_din_input_bwd(const float* target, const float* hist, const float* gin, int64_t B,
                                       int L, int d, float* gtarget, float* ghist, int accumulate_hist,
                                       void* stream) {
  B2_REQUIRE(target && hist && gin && gtarget && ghist, "NULL pointer");
  if (B <= 0) return B2_OK;
  din_input_bwd_kernel<<<grid1d(B * d), 256, 0, (cudaStream_t) stream>>>(target, hist, gin, B, L, d, gtarget, ghist, accumulate_hist);
  B2_CUDA_LAUNCH_CHECK("b2_din_input_bwd");
  return B2_OK;
}

extern "C" B2_API int b2_din_wsum_fwd(const float* w, const unsigned char* mask, const float* hist, int64_t B,
                                      int L, int d, float* out, void* stream) {
  B2_REQUIRE(w && hist && out, "NULL pointer");
  if (B <= 0) return B2_OK;
  din_wsum_fwd_kernel<<<grid1d(B * d), 256, 0, (cudaStream_t) stream>>>(w, mask, hist, B, L, d, out);
  B2_CUDA_LAUNCH_CHECK("b2_din_wsum_fwd");
  return B2_OK;
}

extern "C" B2_API int b2_din_wsum_bwd(const float* w, const unsigned char* mask, const float* hist,
                                      const float* gout, int64_t B, int L, int d, float* gw, float* ghist,
                                      void* stream) {
  B2_REQUIRE(w && hist && gout && gw && ghist, "NULL pointer");
  if (B <= 0) return B2_OK;
  din_wsum_bwd_kernel<<<grid1d(B * L * 32), 256, 0, (cudaStream_t) stream>>>(w, mask, hist, gout, B, L, d, gw, ghist);
  B2_CUDA_LAUNCH_CHECK("b2_din_wsum_bwd");
  return B2_OK;
}

// ---------------------------------------------------------------------------------
// DIN attention, use_softmax = True (target_attention.py:85-90):
//   s = w * mask;  s = s + (-1e9) * (1 - mask);  p = softmax_L(s)
// One warp per (sample) row of L scores: masked scale, row max, exp, row sum — in registers.
// Backward: ds = p * (g - sum_l g p);  dw = ds * mask   (the additive fill has no gradient).
// ---------------------------------------------------------------------------------
namespace {
__global__ void __launch_bounds__(256)
din_softmax_fwd_kernel(const float* __restrict__ w, const unsigned char* __restrict__ mask, int64_t B, int L,
                       float* __restrict__ p) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t) blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t) gridDim.x * blockDim.x) >> 5;
  for (int64_t b = warp; b < B; b += nwarps) {
    float mx = -INFINITY;
    for (int l = lane; l < L; l += 32) {
      float s = __ldg(w + b * L + l);
      if (mask != nullptr) {
        const float m = (float) mask[b * L + l];
        s = s * m + (-1.e9f) * (1.f - m);
      }
      mx = fmaxf(mx, s);
    }
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    float sum = 0.f;
    for (int l = lane; l < L; l += 32) {
      float s = __ldg(w + b * L + l);
      if (mask != nullptr) {
        const float m = (float) mask[b * L + l];
        s = s * m + (-1.e9f) * (1.f - m);
      }
      const float e = expf(s - mx);
      p[b * L + l] = e;
      sum += e;
    }
    sum = b2_warp_sum(sum);
    const float inv = 1.f / sum;
    for (int l = lane; l < L; l += 32) p[b * L + l] *= inv;   // each lane re-reads only its own writes
  }
}

__global__ void __launch_bounds__(256)
din_softmax_bwd_kernel(const float* __restrict__ p, const float* __restrict__ g,
                       const unsigned char* __restrict__ mask, int64_t B, int L, float* __restrict__ gw) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t) blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t) gridDim.x * blockDim.x) >> 5;
  for (int64_t b = warp; b < B; b += nwarps) {
    float dot = 0.f;
    for (int l = lane; l < L; l += 32) dot = fmaf(__ldg(g + b * L + l), __ldg(p + b * L + l), dot);
    dot = b2_warp_sum(dot);
    for (int l = lane; l < L; l += 32) {
      float ds = __ldg(p + b * L + l) * (__ldg(g + b * L + l) - dot);
      if (mask != nullptr) ds *= (float) mask[b * L + l];
      gw[b * L + l] = ds;
    }
  }
}
}  // namespace

extern "C" B2_API int b2_din_softmax_fwd(const float* w, const unsigned char* mask, int64_t B, int L, float* p,
                                         void* stream) {
  B2_REQUIRE(w && p && L >= 1, "bad argument");
  if (B <= 0) return B2_OK;
  int64_t blocks = b2_ceil_div(B * 32, 256);
  if (blocks > (int64_t) B2_NUM_SMS * 8) blocks = (int64_t) B2_NUM_SMS * 8;
  din_softmax_fwd_kernel<<<(int) blocks, 256, 0, (cudaStream_t) stream>>>(w, mask, B, L, p);
  B2_CUDA_LAUNCH_CHECK("b2_din_softmax_fwd");
  return B2_OK;
}

extern "C" B2_API int b2_din_softmax_bwd(const float* p, const float* g, const unsigned char* mask, int64_t B,
                                         int L, float* gw, void* stream) {
  B2_REQUIRE(p && g && gw && L >= 1, "bad argument");
  if (B <= 0) return B2_OK;
  int64_t blocks = b2_ceil_div(B * 32, 256);
  if (blocks > (int64_t) B2_NUM_SMS * 8) blocks = (int64_t) B2_NUM_SMS * 8;
  din_softmax_bwd_kernel<<<(int) blocks, 256, 0, (cudaStream_t) stream>>>(p, g, mask, B, L, gw);
  B2_CUDA_LAUNCH_CHECK("b2_din_softmax_bwd");
  return B2_OK;
}

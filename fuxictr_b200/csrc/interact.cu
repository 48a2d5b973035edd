// interact.cu — feature-interaction kernels over the (fields x emb_dim) tile, sm_90a.
//
// Reference semantics (reczoo/FuxiCTR v2.3.10):
//   InnerProductInteraction.forward  fuxictr/pytorch/layers/interactions/inner_product.py:41-70
//   CrossInteraction / CrossNet      fuxictr/pytorch/layers/interactions/cross_net.py:44-55, 80-92
//
// HBM-bound elementwise + small reductions: no tensor cores.  One group of lanes
// owns one sample, reads its (F, D) tile coalesced, reduces with warp shuffles.
#include "b2_common.cuh"

// ---------------------------------------------------------------------------------
// product_sum / bi_interaction.  DP = 2^k lanes per sample (DP >= min(D,32)); lane j
// owns embedding columns d = j, j+DP, ...; it walks the F fields sequentially so the
// per-column sums use the same left-to-right order as a scalar loop over dim=1.
// ---------------------------------------------------------------------------------
template <bool BWD>
__global__ void __launch_bounds__(256)
fm_sum_kernel(const float* __restrict__ emb, const float* __restrict__ gout, int64_t batch, int F,
              int D, int mode, int dp_log2, float* __restrict__ out, float* __restrict__ gemb) {
  const int DP = 1 << dp_log2;
  const int lane = threadIdx.x & 31;
  const int sub = lane & (DP - 1);
  const unsigned gmask = (DP == 32) ? 0xffffffffu : (((1u << DP) - 1u) << (lane & ~(DP - 1)));
  const int64_t ngroups = ((int64_t) gridDim.x * blockDim.x) >> dp_log2;
  const int64_t group = ((int64_t) blockIdx.x * blockDim.x + threadIdx.x) >> dp_log2;
  const int64_t FD = (int64_t) F * D;
  for (int64_t b = group; b < batch; b += ngroups) {
    const float* e = emb + b * FD;
    float total = 0.f;
    for (int d = sub; d < D; d += DP) {
      float s = 0.f, q = 0.f;
      for (int f = 0; f < F; ++f) {
        const float v = __ldg(e + (int64_t) f * D + d);
        s += v;
        q += v * v;
      }
      if (!BWD) {
        const float bi = (s * s - q) * 0.5f;  // inner_product.py:56-58
        if (mode == 1) out[b * D + d] = bi; else total += bi;
      } else {
        // d/de_{f,d} 0.5*(s^2 - q) = s - e_{f,d}
        const float g = (mode == 1) ? __ldg(gout + b * D + d) : __ldg(gout + b);
        float* ge = gemb + b * FD;
        for (int f = 0; f < F; ++f) {
          const float v = __ldg(e + (int64_t) f * D + d);
          ge[(int64_t) f * D + d] = g * (s - v);
        }
      }
    }
    if (!BWD && mode == 0) {
      for (int o = DP >> 1; o > 0; o >>= 1) total += __shfl_xor_sync(gmask, total, o);
      if (sub == 0) out[b] = total;  // bi_interaction.sum(dim=-1, keepdim=True), inner_product.py:62
    }
  }
}

// ---------------------------------------------------------------------------------
// inner_product (DLRM "dot"): out[b, p] = <e_i, e_j> for i<j in row-major triu order
// (torch.masked_select over triu(ones(F,F),1), inner_product.py:64-66).
// One CTA handles SPB samples; the (F, D) tile is staged in shared memory with an
// odd row pitch so that lanes reading different rows hit different banks.
// ---------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
fm_dot_fwd_kernel(const float* __restrict__ emb, int64_t batch, int F, int D, int spb,
                  float* __restrict__ out) {
  extern __shared__ float sm[];
  const int pitch = D | 1;
  const int P = F * (F - 1) / 2;
  const int64_t FD = (int64_t) F * D;
  int* pair_i = reinterpret_cast<int*>(sm + (size_t) spb * F * pitch);
  int* pair_j = pair_i + P;
  for (int p = threadIdx.x; p < P; p += blockDim.x) {
    // invert p -> (i, j): rows of lengths F-1, F-2, ...
    int i = 0, rem = p;
    while (rem >= F - 1 - i) { rem -= F - 1 - i; ++i; }
    pair_i[p] = i;
    pair_j[p] = i + 1 + rem;
  }
  for (int64_t b0 = (int64_t) blockIdx.x * spb; b0 < batch; b0 += (int64_t) gridDim.x * spb) {
    const int ns = (int) min((int64_t) spb, batch - b0);
    __syncthreads();
    for (int t = threadIdx.x; t < ns * (int) FD; t += blockDim.x) {
      const int s = t / (int) FD, r = t - s * (int) FD;
      sm[(s * F + r / D) * pitch + (r % D)] = __ldg(emb + (b0 + s) * FD + r);
    }
    __syncthreads();
    for (int t = threadIdx.x; t < ns * P; t += blockDim.x) {
      const int s = t / P, p = t - s * P;
      const float* ei = sm + (s * F + pair_i[p]) * pitch;
      const float* ej = sm + (s * F + pair_j[p]) * pitch;
      float acc = 0.f;
      for (int d = 0; d < D; ++d) acc = fmaf(ei[d], ej[d], acc);
      out[(b0 + s) * P + p] = acc;
    }
  }
}

// gemb[b, i, :] = sum_{j != i} gZ[b, pair(i,j)] * e_j
__global__ void __launch_bounds__(256)
fm_dot_bwd_kernel(const float* __restrict__ emb, const float* __restrict__ gout, int64_t batch,
                  int F, int D, int spb, float* __restrict__ gemb) {
  extern __shared__ float sm[];
  const int pitch = D | 1;
  const int P = F * (F - 1) / 2;
  const int64_t FD = (int64_t) F * D;
  float* sg = sm + (size_t) spb * F * pitch;  // spb * P incoming grads
  for (int64_t b0 = (int64_t) blockIdx.x * spb; b0 < batch; b0 += (int64_t) gridDim.x * spb) {
    const int ns = (int) min((int64_t) spb, batch - b0);
    __syncthreads();
    for (int t = threadIdx.x; t < ns * (int) FD; t += blockDim.x) {
      const int s = t / (int) FD, r = t - s * (int) FD;
      sm[(s * F + r / D) * pitch + (r % D)] = __ldg(emb + (b0 + s) * FD + r);
    }
    for (int t = threadIdx.x; t < ns * P; t += blockDim.x) sg[t] = __ldg(gout + b0 * P + t);
    __syncthreads();
    for (int t = threadIdx.x; t < ns * (int) FD; t += blockDim.x) {
      const int s = t / (int) FD, r = t - s * (int) FD;
      const int i = r / D, d = r - i * D;
      const float* g = sg + s * P;
      float acc = 0.f;
      // pairs (j, i) with j < i: index = j*(2F-j-1)/2 + (i-j-1)
      for (int j = 0; j < i; ++j)
        acc = fmaf(g[j * (2 * F - j - 1) / 2 + (i - j - 1)], sm[(s * F + j) * pitch + d], acc);
      // pairs (i, j) with j > i
      const int base = i * (2 * F - i - 1) / 2 - i - 1;
      for (int j = i + 1; j < F; ++j) acc = fmaf(g[base + j], sm[(s * F + j) * pitch + d], acc);
      gemb[(b0 + s) * FD + r] = acc;
    }
  }
}

// ---------------------------------------------------------------------------------
// CrossNet (rank-1 cross): x_{i+1} = x_i + (w_i . x_i) x_0 + b_i, all layers fused.
// One warp per sample keeps x_0 and x_i in registers (<= CH chunks of 32 columns).
// Because x_i = alpha_i * x_0 + beta_i with alpha_i = 1 + sum_{j<i} s_j and
// beta_i = sum_{j<i} b_j, the backward needs only x_0, the saved scalars s (B, L)
// and the parameters — no per-layer activations are stored.
// ---------------------------------------------------------------------------------
template <int CH>
__global__ void __launch_bounds__(256)
crossnet_fwd_kernel(const float* __restrict__ x0, const float* __restrict__ w,
                    const float* __restrict__ bvec, int64_t batch, int d, int L,
                    float* __restrict__ out, float* __restrict__ s_out) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t) blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t) gridDim.x * blockDim.x) >> 5;
  for (int64_t b = warp; b < batch; b += nwarps) {
    float a0[CH], xi[CH];
#pragma unroll
    for (int c = 0; c < CH; ++c) {
      const int col = c * 32 + lane;
      a0[c] = (col < d) ? __ldg(x0 + b * d + col) : 0.f;
      xi[c] = a0[c];
    }
    for (int l = 0; l < L; ++l) {
      float dot = 0.f;
#pragma unroll
      for (int c = 0; c < CH; ++c) {
        const int col = c * 32 + lane;
        if (col < d) dot = fmaf(__ldg(w + (int64_t) l * d + col), xi[c], dot);
      }
      dot = b2_warp_sum(dot);
      if (lane == 0 && s_out != nullptr) s_out[b * L + l] = dot;
#pragma unroll
      for (int c = 0; c < CH; ++c) {
        const int col = c * 32 + lane;
        if (col < d) xi[c] = xi[c] + (dot * a0[c] + __ldg(bvec + (int64_t) l * d + col));  // cross_net.py:54,91
      }
    }
#pragma unroll
    for (int c = 0; c < CH; ++c) {
      const int col = c * 32 + lane;
      if (col < d) out[b * d + col] = xi[c];
    }
  }
}

// Backward.  With g_{L} = gout and, going down, for layer l (input x_l, output x_{l+1}):
//   t_l   = g_{l+1} . x_0
//   gw_l += t_l * x_l            gb_l += g_{l+1}
//   gx0  += s_l * g_{l+1}        g_l   = g_{l+1} + t_l * w_l
// and finally gx0 += g_0.  gw/gb are accumulated per CTA in shared memory, then one
// atomic per (layer, column) per CTA.
template <int CH>
__global__ void __launch_bounds__(256)
crossnet_bwd_kernel(const float* __restrict__ x0, const float* __restrict__ w,
                    const float* __restrict__ bvec, const float* __restrict__ s,
                    const float* __restrict__ gout, int64_t batch, int d, int L,
                    float* __restrict__ gx0, float* __restrict__ gw, float* __restrict__ gb) {
  extern __shared__ float sm[];  // [L*d] gw partial, [L*d] gb partial
  float* sgw = sm;
  float* sgb = sm + (size_t) L * d;
  for (int t = threadIdx.x; t < 2 * L * d; t += blockDim.x) sm[t] = 0.f;
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t) blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t) gridDim.x * blockDim.x) >> 5;
  for (int64_t b = warp; b < batch; b += nwarps) {
    float a0[CH], g[CH], gx[CH];
#pragma unroll
    for (int c = 0; c < CH; ++c) {
      const int col = c * 32 + lane;
      a0[c] = (col < d) ? __ldg(x0 + b * d + col) : 0.f;
      g[c] = (col < d) ? __ldg(gout + b * d + col) : 0.f;
      gx[c] = 0.f;
    }
    // alpha_l = 1 + sum_{j<l} s_j ; start from alpha_L and peel one s per layer.
    float alpha = 1.f;
    for (int l = 0; l < L; ++l) alpha += __ldg(s + b * L + l);
    for (int l = L - 1; l >= 0; --l) {
      const float sl = __ldg(s + b * L + l);
      alpha -= sl;  // now alpha_l
      float t = 0.f;
#pragma unroll
      for (int c = 0; c < CH; ++c) t = fmaf(g[c], a0[c], t);
      t = b2_warp_sum(t);
#pragma unroll
      for (int c = 0; c < CH; ++c) {
        const int col = c * 32 + lane;
        if (col < d) {
          // beta_l[col] = sum_{j<l} b_j[col]
          float beta = 0.f;
          for (int j = 0; j < l; ++j) beta += __ldg(bvec + (int64_t) j * d + col);
          const float xl = alpha * a0[c] + beta;
          atomicAdd(sgw + l * d + col, t * xl);
          atomicAdd(sgb + l * d + col, g[c]);
          gx[c] = fmaf(sl, g[c], gx[c]);
          g[c] = fmaf(t, __ldg(w + (int64_t) l * d + col), g[c]);
        }
      }
    }
#pragma unroll
    for (int c = 0; c < CH; ++c) {
      const int col = c * 32 + lane;
      if (col < d) gx0[b * d + col] = gx[c] + g[c];
    }
  }
  __syncthreads();
  for (int t = threadIdx.x; t < L * d; t += blockDim.x) {
    if (sgw[t] != 0.f) b2_red_add(gw + t, sgw[t]);
    if (sgb[t] != 0.f) b2_red_add(gb + t, sgb[t]);
  }
}

// ---------------------------------------------------------------------------------
// Host side
// ---------------------------------------------------------------------------------
static int pow2_log2_ge(int v) {
  int l = 0;
  while ((1 << l) < v) ++l;
  return l;
}
static int grid_cap(int64_t blocks, int per_sm) {
  const int64_t cap = (int64_t) B2_NUM_SMS * per_sm;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  return (int) blocks;
}

extern "C" B2_API int b2_fm_fwd(const float* emb, int64_t batch, int nfields, int dim, int mode,
                         float* out, void* stream) {
  B2_REQUIRE(emb != nullptr && out != nullptr, "NULL pointer");
  B2_REQUIRE(nfields >= 1 && dim >= 1 && mode >= 0 && mode <= 2, "bad nfields/dim/mode");
  if (batch == 0) return B2_OK;
  cudaStream_t st = (cudaStream_t) stream;
  if (mode == 2) {
    B2_REQUIRE(nfields >= 2, "inner_product needs >= 2 fields");
    const int P = nfields * (nfields - 1) / 2, pitch = dim | 1;
    int spb = 8;
    size_t smem;
    while (true) {
      smem = sizeof(float) * (size_t) spb * nfields * pitch + sizeof(int) * 2 * (size_t) P;
      if (smem <= 48 * 1024 || spb == 1) break;
      spb >>= 1;
    }
    B2_REQUIRE(smem <= 48 * 1024, "inner_product tile (F=%d, D=%d) exceeds 48 KB smem", nfields, dim);
    const int grid = grid_cap(b2_ceil_div(batch, spb), 8);
    fm_dot_fwd_kernel<<<grid, 256, smem, st>>>(emb, batch, nfields, dim, spb, out);
  } else {
    int dp_log2 = pow2_log2_ge(dim);
    if (dp_log2 > 5) dp_log2 = 5;
    const int grid = grid_cap(b2_ceil_div(batch << dp_log2, 256), 8);
    fm_sum_kernel<false><<<grid, 256, 0, st>>>(emb, nullptr, batch, nfields, dim, mode, dp_log2, out, nullptr);
  }
  B2_CUDA_LAUNCH_CHECK("b2_fm_fwd");
  return B2_OK;
}

extern "C" B2_API int b2_fm_bwd(const float* emb, const float* gout, int64_t batch, int nfields, int dim,
                         int mode, float* gemb, void* stream) {
  B2_REQUIRE(emb != nullptr && gout != nullptr && gemb != nullptr, "NULL pointer");
  B2_REQUIRE(nfields >= 1 && dim >= 1 && mode >= 0 && mode <= 2, "bad nfields/dim/mode");
  if (batch == 0) return B2_OK;
  cudaStream_t st = (cudaStream_t) stream;
  if (mode == 2) {
    B2_REQUIRE(nfields >= 2, "inner_product needs >= 2 fields");
    const int P = nfields * (nfields - 1) / 2, pitch = dim | 1;
    int spb = 8;
    size_t smem;
    while (true) {
      smem = sizeof(float) * ((size_t) spb * nfields * pitch + (size_t) spb * P);
      if (smem <= 48 * 1024 || spb == 1) break;
      spb >>= 1;
    }
    B2_REQUIRE(smem <= 48 * 1024, "inner_product tile (F=%d, D=%d) exceeds 48 KB smem", nfields, dim);
    const int grid = grid_cap(b2_ceil_div(batch, spb), 8);
    fm_dot_bwd_kernel<<<grid, 256, smem, st>>>(emb, gout, batch, nfields, dim, spb, gemb);
  } else {
    int dp_log2 = pow2_log2_ge(dim);
    if (dp_log2 > 5) dp_log2 = 5;
    const int grid = grid_cap(b2_ceil_div(batch << dp_log2, 256), 8);
    fm_sum_kernel<true><<<grid, 256, 0, st>>>(emb, gout, batch, nfields, dim, mode, dp_log2, nullptr, gemb);
  }
  B2_CUDA_LAUNCH_CHECK("b2_fm_bwd");
  return B2_OK;
}

extern "C" B2_API int b2_crossnet_fwd(const float* x0, const float* w, const float* b, int64_t batch,
                               int d, int nlayers, float* out, float* s, void* stream) {
  B2_REQUIRE(x0 && w && b && out, "NULL pointer");
  B2_REQUIRE(d >= 1 && d <= 32 * 32, "input_dim %d outside [1,1024]", d);
  B2_REQUIRE(nlayers >= 0, "negative num_layers");
  if (batch == 0) return B2_OK;
  cudaStream_t st = (cudaStream_t) stream;
  const int grid = grid_cap(b2_ceil_div(batch * 32, 256), 8);
  const int ch = (d + 31) / 32;
  if (ch <= 4) crossnet_fwd_kernel<4><<<grid, 256, 0, st>>>(x0, w, b, batch, d, nlayers, out, s);
  else if (ch <= 8) crossnet_fwd_kernel<8><<<grid, 256, 0, st>>>(x0, w, b, batch, d, nlayers, out, s);
  else if (ch <= 20) crossnet_fwd_kernel<20><<<grid, 256, 0, st>>>(x0, w, b, batch, d, nlayers, out, s);
  else crossnet_fwd_kernel<32><<<grid, 256, 0, st>>>(x0, w, b, batch, d, nlayers, out, s);
  B2_CUDA_LAUNCH_CHECK("b2_crossnet_fwd");
  return B2_OK;
}

extern "C" B2_API int b2_crossnet_bwd(const float* x0, const float* w, const float* b, const float* s,
                               const float* gout, int64_t batch, int d, int nlayers, float* gx0,
                               float* gw, float* gb, void* stream) {
  B2_REQUIRE(x0 && w && b && s && gout && gx0 && gw && gb, "NULL pointer");
  B2_REQUIRE(d >= 1 && d <= 32 * 32, "input_dim %d outside [1,1024]", d);
  B2_REQUIRE(nlayers >= 1, "num_layers must be >= 1 for backward");
  if (batch == 0) return B2_OK;
  cudaStream_t st = (cudaStream_t) stream;
  const size_t smem = sizeof(float) * 2 * (size_t) nlayers * d;
  B2_REQUIRE(smem <= 200 * 1024, "L*d too large for the shared-memory gradient staging");
  // Few, fat CTAs: each one issues L*d global atomics at the end.
  const int grid = grid_cap(b2_ceil_div(batch * 32, 256), 1);
  const int ch = (d + 31) / 32;
#define B2_LAUNCH_CROSS_BWD(CHV)                                                                  \
  do {                                                                                            \
    if (smem > 48 * 1024)                                                                         \
      cudaFuncSetAttribute(crossnet_bwd_kernel<CHV>, cudaFuncAttributeMaxDynamicSharedMemorySize, \
                           (int) smem);                                                           \
    crossnet_bwd_kernel<CHV><<<grid, 256, smem, st>>>(x0, w, b, s, gout, batch, d, nlayers, gx0,  \
                                                      gw, gb);                                    \
  } while (0)
  if (ch <= 4) B2_LAUNCH_CROSS_BWD(4);
  else if (ch <= 8) B2_LAUNCH_CROSS_BWD(8);
  else if (ch <= 20) B2_LAUNCH_CROSS_BWD(20);
  else B2_LAUNCH_CROSS_BWD(32);
#undef B2_LAUNCH_CROSS_BWD
  B2_CUDA_LAUNCH_CHECK("b2_crossnet_bwd");
  return B2_OK;
}

// cin.cu — one Compressed-Interaction-Network layer without ever materialising the
// (B, F*H, D) Hadamard tensor, sm_90a.
//
// Reference (reczoo/FuxiCTR v2.3.10), fuxictr/pytorch/layers/interactions/compressed_interaction_net.py:70-73:
//     hadamard = einsum("bhd,bmd->bhmd", X_0, X_i).view(B, F*H, D)
//     X_next   = Conv1d(F*H, H', kernel_size=1)(hadamard)          # (B, H', D)
// i.e. per "column" (b, d):  X_next[h'] = bias[h'] + sum_{f,m} W[h', f*H + m] * X_0[f] * X_i[m].
// The reference writes and re-reads B*F*H*D floats (400 MB at C2 shape, layer 1); here a column's
// products live in registers only.
//
//   cin_fwd_kernel   thread = column; x0 / xk tiles in shared memory (coalesced along d);
//                    W streamed through shared memory one field f at a time (broadcast reads).
//   cin_bwd_x_kernel thread = column; t(f,m) = sum_h' G[h'] W[h',f,m] on the fly;
//                    dX0[f] = sum_m t*xk[m] and dXk[m] = sum_f t*x0[f] accumulate in registers.
//   cin_bwd_w_kernel thread = a few (f,m) pairs x all h'; loops over the columns of its tiles,
//                    accumulates in registers, one `red` per weight per CTA at the end.
// Compute-bound on the FP32 pipe (2*F*H*H' flops per column): no tensor cores in this round — the
// A operand would have to be generated in the swizzled UMMA layout by a producer warp (next step).
#include "b2_common.cuh"

namespace {
constexpr int COLS = 256;      // columns (= threads) per tile
constexpr int PITCH = COLS + 1;  // odd pitch: tile rows f / m land in different banks

__device__ __forceinline__ void load_tile(const float* __restrict__ x, int64_t col0, int64_t ncols_total,
                                          int R, int D, float* __restrict__ s) {
  // s[r * PITCH + c] = x[b, r, d] for column col0 + c = b*D + d
  for (int i = threadIdx.x; i < R * COLS; i += blockDim.x) {
    const int r = i / COLS, c = i - r * COLS;
    const int64_t col = col0 + c;
    float v = 0.f;
    if (col < ncols_total) {
      const int64_t b = col / D;
      const int d = (int) (col - b * D);
      v = __ldg(x + (b * R + r) * D + d);
    }
    s[r * PITCH + c] = v;
  }
}

// ---------------------------------------------------------------------------------
template <int HP>  // HP >= H' (accumulators per thread)
__global__ void __launch_bounds__(COLS)
cin_fwd_kernel(const float* __restrict__ x0, const float* __restrict__ xk, const float* __restrict__ w,
               const float* __restrict__ bias, int64_t batch, int F, int H, int HO, int D,
               float* __restrict__ out) {
  extern __shared__ float sm[];
  float* sx0 = sm;                       // F * PITCH
  float* sxk = sx0 + F * PITCH;          // H * PITCH
  float* sw = sm + (((F + H) * PITCH + 3) & ~3);  // 16-byte aligned: 2 buffers of H * HP (W[:, f, :] as [m][h'])
  const int64_t ncols = batch * (int64_t) D;
  const int tid = threadIdx.x;
  for (int64_t col0 = (int64_t) blockIdx.x * COLS; col0 < ncols; col0 += (int64_t) gridDim.x * COLS) {
    __syncthreads();
    load_tile(x0, col0, ncols, F, D, sx0);
    load_tile(xk, col0, ncols, H, D, sxk);
    float acc[HP];
#pragma unroll
    for (int h = 0; h < HP; ++h) acc[h] = (h < HO && bias != nullptr) ? __ldg(bias + h) : 0.f;
    for (int f = 0; f < F; ++f) {
      float* swf = sw + (f & 1) * H * HP;
      // stage W[h', f*H + m] as swf[m*HP + h'] (zero padded)
      for (int i = tid; i < H * HP; i += COLS) {
        const int m = i / HP, h = i - m * HP;
        swf[i] = (h < HO) ? __ldg(w + (int64_t) h * F * H + (int64_t) f * H + m) : 0.f;
      }
      __syncthreads();   // also orders the tile loads before the first use
      const float x0f = sx0[f * PITCH + tid];
      for (int m = 0; m < H; ++m) {
        const float p = x0f * sxk[m * PITCH + tid];
        const float4* wv = reinterpret_cast<const float4*>(swf + m * HP);
#pragma unroll
        for (int h4 = 0; h4 < HP / 4; ++h4) {
          const float4 wq = wv[h4];   // same address in every lane: broadcast
          acc[4 * h4 + 0] = fmaf(wq.x, p, acc[4 * h4 + 0]);
          acc[4 * h4 + 1] = fmaf(wq.y, p, acc[4 * h4 + 1]);
          acc[4 * h4 + 2] = fmaf(wq.z, p, acc[4 * h4 + 2]);
          acc[4 * h4 + 3] = fmaf(wq.w, p, acc[4 * h4 + 3]);
        }
      }
    }
    const int64_t col = col0 + tid;
    if (col < ncols) {
      const int64_t b = col / D;
      const int d = (int) (col - b * D);
#pragma unroll
      for (int h = 0; h < HP; ++h)
        if (h < HO) out[(b * HO + h) * D + d] = acc[h];
    }
  }
}

// ---------------------------------------------------------------------------------
template <int HP, int HK>  // HK >= H (dXk accumulators per thread)
__global__ void __launch_bounds__(COLS)
cin_bwd_x_kernel(const float* __restrict__ x0, const float* __restrict__ xk, const float* __restrict__ w,
                 const float* __restrict__ g, int64_t batch, int F, int H, int HO, int D,
                 float* __restrict__ gx0, float* __restrict__ gxk, int accumulate_x0) {
  extern __shared__ float sm[];
  float* sx0 = sm;
  float* sxk = sx0 + F * PITCH;
  float* sw = sm + (((F + H) * PITCH + 3) & ~3);
  const int64_t ncols = batch * (int64_t) D;
  const int tid = threadIdx.x;
  for (int64_t col0 = (int64_t) blockIdx.x * COLS; col0 < ncols; col0 += (int64_t) gridDim.x * COLS) {
    __syncthreads();
    load_tile(x0, col0, ncols, F, D, sx0);
    load_tile(xk, col0, ncols, H, D, sxk);
    const int64_t col = col0 + tid;
    const bool live = col < ncols;
    const int64_t b = live ? col / D : 0;
    const int d = live ? (int) (col - b * D) : 0;
    float gv[HP];
#pragma unroll
    for (int h = 0; h < HP; ++h) gv[h] = (live && h < HO) ? __ldg(g + (b * HO + h) * D + d) : 0.f;
    float dxk[HK];
#pragma unroll
    for (int m = 0; m < HK; ++m) dxk[m] = 0.f;
    for (int f = 0; f < F; ++f) {
      float* swf = sw + (f & 1) * H * HP;
      for (int i = tid; i < H * HP; i += COLS) {
        const int m = i / HP, h = i - m * HP;
        swf[i] = (h < HO) ? __ldg(w + (int64_t) h * F * H + (int64_t) f * H + m) : 0.f;
      }
      __syncthreads();
      const float x0f = sx0[f * PITCH + tid];
      float dx0f = 0.f;
#pragma unroll
      for (int m = 0; m < HK; ++m) {
        if (m < H) {
          const float4* wv = reinterpret_cast<const float4*>(swf + m * HP);
          float t = 0.f;
#pragma unroll
          for (int h4 = 0; h4 < HP / 4; ++h4) {
            const float4 wq = wv[h4];
            t = fmaf(wq.x, gv[4 * h4 + 0], t);
            t = fmaf(wq.y, gv[4 * h4 + 1], t);
            t = fmaf(wq.z, gv[4 * h4 + 2], t);
            t = fmaf(wq.w, gv[4 * h4 + 3], t);
          }
          dx0f = fmaf(t, sxk[m * PITCH + tid], dx0f);
          dxk[m] = fmaf(t, x0f, dxk[m]);
        }
      }
      if (live) {
        float* p = gx0 + (b * F + f) * D + d;
        if (accumulate_x0) *p += dx0f; else *p = dx0f;
      }
    }
    if (live) {
#pragma unroll
      for (int m = 0; m < HK; ++m)
        if (m < H) gxk[(b * H + m) * D + d] = dxk[m];
    }
  }
}

// ---------------------------------------------------------------------------------
// dW[h', f*H+m] += sum_cols G[h', col] * x0[f, col] * xk[m, col]
template <int HP, int PAIRS>  // PAIRS (f,m) pairs per thread
__global__ void __launch_bounds__(COLS)
cin_bwd_w_kernel(const float* __restrict__ x0, const float* __restrict__ xk, const float* __restrict__ g,
                 int64_t batch, int F, int H, int HO, int D, float* __restrict__ gw) {
  extern __shared__ float sm[];
  float* sx0 = sm;
  float* sxk = sx0 + F * PITCH;
  float* sg = sm + (((F + H) * PITCH + 3) & ~3);  // 16-byte aligned: COLS * HP (sg[c*HP + h'])
  const int64_t ncols = batch * (int64_t) D;
  const int tid = threadIdx.x;
  const int K = F * H;
  // pairs of this thread within this CTA's K-slice
  const int kslice = blockIdx.y;         // each y-slice owns COLS*PAIRS consecutive (f,m) pairs
  int pf[PAIRS], pm[PAIRS];
  bool pok[PAIRS];
#pragma unroll
  for (int j = 0; j < PAIRS; ++j) {
    const int c = (kslice * PAIRS + j) * COLS + tid;
    pok[j] = c < K;
    pf[j] = pok[j] ? c / H : 0;
    pm[j] = pok[j] ? c - pf[j] * H : 0;
  }
  float acc[PAIRS][HP];
#pragma unroll
  for (int j = 0; j < PAIRS; ++j)
#pragma unroll
    for (int h = 0; h < HP; ++h) acc[j][h] = 0.f;

  for (int64_t col0 = (int64_t) blockIdx.x * COLS; col0 < ncols; col0 += (int64_t) gridDim.x * COLS) {
    __syncthreads();
    load_tile(x0, col0, ncols, F, D, sx0);
    load_tile(xk, col0, ncols, H, D, sxk);
    for (int i = tid; i < COLS * HP; i += COLS) {
      const int c = i / HP, h = i - c * HP;
      const int64_t col = col0 + c;
      float v = 0.f;
      if (col < ncols && h < HO) {
        const int64_t b = col / D;
        const int d = (int) (col - b * D);
        v = __ldg(g + (b * HO + h) * D + d);
      }
      sg[i] = v;
    }
    __syncthreads();
    for (int c = 0; c < COLS; ++c) {
      const float4* gq = reinterpret_cast<const float4*>(sg + c * HP);
#pragma unroll
      for (int j = 0; j < PAIRS; ++j) {
        const float p = sx0[pf[j] * PITCH + c] * sxk[pm[j] * PITCH + c];
#pragma unroll
        for (int h4 = 0; h4 < HP / 4; ++h4) {
          const float4 gvv = gq[h4];   // broadcast
          acc[j][4 * h4 + 0] = fmaf(gvv.x, p, acc[j][4 * h4 + 0]);
          acc[j][4 * h4 + 1] = fmaf(gvv.y, p, acc[j][4 * h4 + 1]);
          acc[j][4 * h4 + 2] = fmaf(gvv.z, p, acc[j][4 * h4 + 2]);
          acc[j][4 * h4 + 3] = fmaf(gvv.w, p, acc[j][4 * h4 + 3]);
        }
      }
    }
  }
#pragma unroll
  for (int j = 0; j < PAIRS; ++j) {
    if (!pok[j]) continue;
    const int c = pf[j] * H + pm[j];
#pragma unroll
    for (int h = 0; h < HP; ++h)
      if (h < HO) b2_red_add(gw + (int64_t) h * K + c, acc[j][h]);
  }
}

int round_hp(int ho) { return ho <= 8 ? 8 : (ho <= 16 ? 16 : 32); }
}  // namespace

#define B2_CIN_SET_SMEM(kernel, bytes)                                                          \
  do {                                                                                          \
    if ((bytes) > 48 * 1024) {                                                                  \
      cudaError_t e_ = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, \
                                            (int) (bytes));                                     \
      if (e_ != cudaSuccess) return b2_fail(B2_E_CUDA, "cin smem attribute: %s", cudaGetErrorString(e_)); \
    }                                                                                           \
  } while (0)

extern "C" B2_API int b2_cin_fwd(const float* x0, const float* xk, const float* w, const float* bias,
                                 int64_t batch, int F, int H, int HO, int D, float* out, void* stream) {
  B2_REQUIRE(x0 && xk && w && out, "NULL pointer");
  B2_REQUIRE(F >= 1 && H >= 1 && HO >= 1 && HO <= 32 && D >= 1, "unsupported CIN shape (H' must be <= 32)");
  if (batch <= 0) return B2_OK;
  const int hp = round_hp(HO);
  const size_t smem = sizeof(float) * ((size_t) (F + H) * PITCH + 4 + 2 * (size_t) H * hp);
  B2_REQUIRE(smem <= 220 * 1024, "CIN tile (F=%d, H=%d) exceeds shared memory", F, H);
  const int64_t tiles = b2_ceil_div(batch * (int64_t) D, COLS);
  const int grid = (int) (tiles < 2 * B2_NUM_SMS ? tiles : 2 * B2_NUM_SMS);
  cudaStream_t st = (cudaStream_t) stream;
  if (hp == 8) { B2_CIN_SET_SMEM(cin_fwd_kernel<8>, smem); cin_fwd_kernel<8><<<grid, COLS, smem, st>>>(x0, xk, w, bias, batch, F, H, HO, D, out); }
  else if (hp == 16) { B2_CIN_SET_SMEM(cin_fwd_kernel<16>, smem); cin_fwd_kernel<16><<<grid, COLS, smem, st>>>(x0, xk, w, bias, batch, F, H, HO, D, out); }
  else { B2_CIN_SET_SMEM(cin_fwd_kernel<32>, smem); cin_fwd_kernel<32><<<grid, COLS, smem, st>>>(x0, xk, w, bias, batch, F, H, HO, D, out); }
  B2_CUDA_LAUNCH_CHECK("b2_cin_fwd");
  return B2_OK;
}

extern "C" B2_API int b2_cin_bwd(const float* x0, const float* xk, const float* w, const float* g,
                                 int64_t batch, int F, int H, int HO, int D, float* gx0, int accumulate_x0,
                                 float* gxk, float* gw, void* stream) {
  B2_REQUIRE(x0 && xk && w && g && gx0 && gxk && gw, "NULL pointer");
  B2_REQUIRE(F >= 1 && H >= 1 && H <= 64 && HO >= 1 && HO <= 32 && D >= 1,
             "unsupported CIN shape (H <= 64, H' <= 32)");
  if (batch <= 0) return B2_OK;
  cudaStream_t st = (cudaStream_t) stream;
  const int hp = round_hp(HO);
  const int64_t tiles = b2_ceil_div(batch * (int64_t) D, COLS);
  {
    const size_t smem = sizeof(float) * ((size_t) (F + H) * PITCH + 4 + 2 * (size_t) H * hp);
    B2_REQUIRE(smem <= 220 * 1024, "CIN tile (F=%d, H=%d) exceeds shared memory", F, H);
    const int grid = (int) (tiles < 2 * B2_NUM_SMS ? tiles : 2 * B2_NUM_SMS);
#define B2_LAUNCH_BX(HPV, HKV)                                                                     \
  do {                                                                                             \
    B2_CIN_SET_SMEM((cin_bwd_x_kernel<HPV, HKV>), smem);                                            \
    cin_bwd_x_kernel<HPV, HKV><<<grid, COLS, smem, st>>>(x0, xk, w, g, batch, F, H, HO, D, gx0, gxk, \
                                                        accumulate_x0);                            \
  } while (0)
    const int hk = H <= 16 ? 16 : (H <= 40 ? 40 : 64);
    if (hp == 8) { if (hk == 16) B2_LAUNCH_BX(8, 16); else if (hk == 40) B2_LAUNCH_BX(8, 40); else B2_LAUNCH_BX(8, 64); }
    else if (hp == 16) { if (hk == 16) B2_LAUNCH_BX(16, 16); else if (hk == 40) B2_LAUNCH_BX(16, 40); else B2_LAUNCH_BX(16, 64); }
    else { if (hk == 16) B2_LAUNCH_BX(32, 16); else if (hk == 40) B2_LAUNCH_BX(32, 40); else B2_LAUNCH_BX(32, 64); }
#undef B2_LAUNCH_BX
    B2_CUDA_LAUNCH_CHECK("b2_cin_bwd(x)");
  }
  {
    constexpr int PAIRS = 2;
    const size_t smem = sizeof(float) * ((size_t) (F + H) * PITCH + 4 + (size_t) COLS * hp);
    B2_REQUIRE(smem <= 220 * 1024, "CIN tile (F=%d, H=%d) exceeds shared memory", F, H);
    const int K = F * H;
    const int kslices = (int) b2_ceil_div(K, COLS * PAIRS);
    int64_t gx = b2_ceil_div(2 * B2_NUM_SMS, kslices);
    if (gx > tiles) gx = tiles;
    if (gx < 1) gx = 1;
    dim3 grid((unsigned) gx, (unsigned) kslices);
    cudaError_t e = cudaMemsetAsync(gw, 0, sizeof(float) * (size_t) HO * K, st);
    if (e != cudaSuccess) return b2_fail(B2_E_CUDA, "b2_cin_bwd: memset: %s", cudaGetErrorString(e));
    if (hp == 8) { B2_CIN_SET_SMEM((cin_bwd_w_kernel<8, PAIRS>), smem); cin_bwd_w_kernel<8, PAIRS><<<grid, COLS, smem, st>>>(x0, xk, g, batch, F, H, HO, D, gw); }
    else if (hp == 16) { B2_CIN_SET_SMEM((cin_bwd_w_kernel<16, PAIRS>), smem); cin_bwd_w_kernel<16, PAIRS><<<grid, COLS, smem, st>>>(x0, xk, g, batch, F, H, HO, D, gw); }
    else { B2_CIN_SET_SMEM((cin_bwd_w_kernel<32, PAIRS>), smem); cin_bwd_w_kernel<32, PAIRS><<<grid, COLS, smem, st>>>(x0, xk, g, batch, F, H, HO, D, gw); }
    B2_CUDA_LAUNCH_CHECK("b2_cin_bwd(w)");
  }
  return B2_OK;
}

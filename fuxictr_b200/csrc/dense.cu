// dense.cu — fp32 dense layer (parity path), elementwise backward helpers, fused
// logit+BCE, and the dense clip+Adam step, sm_90a.
//
// Reference semantics (reczoo/FuxiCTR v2.3.10):
//   MLP_Block                fuxictr/pytorch/layers/blocks/mlp_block.py:64-96   (nn.Linear + act)
//   CrossNetV2.forward       fuxictr/pytorch/layers/interactions/cross_net.py:126-129
//   BaseModel.add_loss       fuxictr/pytorch/models/rank_model.py:120-131       (BCE, mean)
//   BaseModel.train_step     fuxictr/pytorch/models/rank_model.py:316-322       (clip + Adam)
//
// The fp32 GEMM here is the 1e-5-parity path: plain FFMA with fp32 accumulate, the
// same arithmetic class as the reference's ATen addmm.  The tensor-core (wgmma)
// GEMM for the bf16 throughput path lives in gemm_tc.cu.
#include "b2_common.cuh"
#include "adam_common.cuh"

// ---------------------------------------------------------------------------------
// SIMT SGEMM, 64x64x16 tile, 256 threads, 4x4 micro-tile, register-prefetched double
// buffer.  Operands are addressed through (row, col) element strides so the forward
// (X W^T), dgrad (dY W) and wgrad (dY^T X) layouts all run through one kernel.
// ---------------------------------------------------------------------------------
namespace {
constexpr int BM = 64, BN = 64, BK = 16, TM = 4, TN = 4;
constexpr int PAD = 4;  // keeps float4 alignment of the smem rows, halves store conflicts

struct GemmArgs {
  const float* a; int64_t a_rs, a_cs;
  const float* b; int64_t b_rs, b_cs;
  float* c; int64_t ldc;
  int64_t M, N, K;
  const float* bias; const float* mul; const float* add;
  int act; int beta; int k_per_split;
};

// Loads a (ROWS x BK) operand tile into registers: 4 elements per thread.
// KCONTIG: the reduction index is the unit-stride one.
template <bool KCONTIG>
__device__ __forceinline__ void load_tile(const float* __restrict__ p, int64_t rs, int64_t cs,
                                          int64_t r0, int64_t k0, int64_t R, int64_t Kend,
                                          float (&v)[4], int t, bool vec_ok) {
  // element (r, k) of the operand lives at p[r*rs + k*cs]
  if (KCONTIG) {
    const int r = t >> 2, k4 = (t & 3) * 4;  // 64 rows x 4 float4
    const int64_t rr = r0 + r, kk = k0 + k4;
    if (vec_ok && rr < R && kk + 3 < Kend) {
      const float4 q = __ldg(reinterpret_cast<const float4*>(p + rr * rs + kk));
      v[0] = q.x; v[1] = q.y; v[2] = q.z; v[3] = q.w;
    } else {
#pragma unroll
      for (int i = 0; i < 4; ++i)
        v[i] = (rr < R && kk + i < Kend) ? __ldg(p + rr * rs + (kk + i) * cs) : 0.f;
    }
  } else {
    const int k = t >> 4, r4 = (t & 15) * 4;  // 16 k x 16 float4 along rows
    const int64_t rr = r0 + r4, kk = k0 + k;
    if (vec_ok && kk < Kend && rr + 3 < R) {
      const float4 q = __ldg(reinterpret_cast<const float4*>(p + kk * cs + rr));
      v[0] = q.x; v[1] = q.y; v[2] = q.z; v[3] = q.w;
    } else {
#pragma unroll
      for (int i = 0; i < 4; ++i)
        v[i] = (kk < Kend && rr + i < R) ? __ldg(p + (rr + i) * rs + kk * cs) : 0.f;
    }
  }
}

template <bool KCONTIG>
__device__ __forceinline__ void store_tile(float (*s)[BM + PAD], const float (&v)[4], int t) {
  if (KCONTIG) {
    const int r = t >> 2, k4 = (t & 3) * 4;
#pragma unroll
    for (int i = 0; i < 4; ++i) s[k4 + i][r] = v[i];
  } else {
    const int k = t >> 4, r4 = (t & 15) * 4;
    *reinterpret_cast<float4*>(&s[k][r4]) = make_float4(v[0], v[1], v[2], v[3]);
  }
}

template <bool A_KC, bool B_KC>
__global__ void __launch_bounds__(256)
sgemm_kernel(const GemmArgs g, bool a_vec, bool b_vec) {
  __shared__ __align__(16) float As[2][BK][BM + PAD];
  __shared__ __align__(16) float Bs[2][BK][BN + PAD];
  const int t = threadIdx.x;
  const int tx = t & 15, ty = t >> 4;  // 16 x 16 threads, each 4 x 4 outputs
  const int64_t m0 = (int64_t) blockIdx.y * BM, n0 = (int64_t) blockIdx.x * BN;
  const int64_t kbeg = (int64_t) blockIdx.z * g.k_per_split;
  const int64_t kend = min(g.K, kbeg + g.k_per_split);

  float acc[TM][TN];
#pragma unroll
  for (int i = 0; i < TM; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

  float ra[4], rb[4];
  // B operand: element (k, n) at b[k*b_rs + n*b_cs]; as a "rows = n" operand its row
  // stride is b_cs and its k stride is b_rs.
  load_tile<A_KC>(g.a, g.a_rs, g.a_cs, m0, kbeg, g.M, kend, ra, t, a_vec);
  load_tile<B_KC>(g.b, g.b_cs, g.b_rs, n0, kbeg, g.N, kend, rb, t, b_vec);
  store_tile<A_KC>(As[0], ra, t);
  store_tile<B_KC>(Bs[0], rb, t);
  __syncthreads();

  int cur = 0;
  for (int64_t k0 = kbeg; k0 < kend; k0 += BK) {
    const bool more = (k0 + BK) < kend;
    if (more) {
      load_tile<A_KC>(g.a, g.a_rs, g.a_cs, m0, k0 + BK, g.M, kend, ra, t, a_vec);
      load_tile<B_KC>(g.b, g.b_cs, g.b_rs, n0, k0 + BK, g.N, kend, rb, t, b_vec);
    }
#pragma unroll
    for (int k = 0; k < BK; ++k) {
      const float4 av = *reinterpret_cast<const float4*>(&As[cur][k][ty * TM]);
      const float4 bv = *reinterpret_cast<const float4*>(&Bs[cur][k][tx * TN]);
      const float a4[4] = {av.x, av.y, av.z, av.w};
      const float b4[4] = {bv.x, bv.y, bv.z, bv.w};
#pragma unroll
      for (int i = 0; i < TM; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(a4[i], b4[j], acc[i][j]);
    }
    if (more) {
      store_tile<A_KC>(As[cur ^ 1], ra, t);
      store_tile<B_KC>(Bs[cur ^ 1], rb, t);
      __syncthreads();
      cur ^= 1;
    }
  }

  // Epilogue: C = act( add + mul * (acc + bias) ) [+ C]
  const bool split = gridDim.z > 1;
#pragma unroll
  for (int i = 0; i < TM; ++i) {
    const int64_t m = m0 + ty * TM + i;
    if (m >= g.M) continue;
#pragma unroll
    for (int j = 0; j < TN; ++j) {
      const int64_t n = n0 + tx * TN + j;
      if (n >= g.N) continue;
      float v = acc[i][j];
      if (g.bias != nullptr && blockIdx.z == 0) v += __ldg(g.bias + n);
      float* cp = g.c + m * g.ldc + n;
      if (split) {  // linear epilogue only; partial sums meet in memory
        b2_red_add(cp, v);
        continue;
      }
      if (g.mul != nullptr) v *= __ldg(g.mul + m * g.ldc + n);
      if (g.add != nullptr) v += __ldg(g.add + m * g.ldc + n);
      if (g.act == B2_ACT_RELU) v = fmaxf(v, 0.f);
      else if (g.act == B2_ACT_SIGMOID) v = 1.f / (1.f + expf(-v));
      if (g.beta) v += *cp;
      *cp = v;
    }
  }
}

__global__ void zero_strided_kernel(float* c, int64_t M, int64_t N, int64_t ldc) {
  const int64_t total = M * N;
  for (int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (int64_t) gridDim.x * blockDim.x)
    c[(i / N) * ldc + (i % N)] = 0.f;
}
}  // namespace

extern "C" B2_API int b2_gemm_f32(const float* a, int64_t a_rs, int64_t a_cs, const float* b,
                           int64_t b_rs, int64_t b_cs, float* c, int64_t ldc, int64_t M,
                           int64_t N, int64_t K, const float* bias, int act, const float* mul,
                           const float* add, int beta_accumulate, void* stream) {
  B2_REQUIRE(a && b && c, "NULL operand");
  B2_REQUIRE(M >= 0 && N >= 0 && K >= 0 && ldc >= N, "bad shape M=%lld N=%lld K=%lld ldc=%lld",
             (long long) M, (long long) N, (long long) K, (long long) ldc);
  B2_REQUIRE(a_rs == 1 || a_cs == 1, "A must have a unit stride");
  B2_REQUIRE(b_rs == 1 || b_cs == 1, "B must have a unit stride");
  B2_REQUIRE(act >= B2_ACT_NONE && act <= B2_ACT_SIGMOID, "bad activation code %d", act);
  if (M == 0 || N == 0) return B2_OK;
  cudaStream_t st = (cudaStream_t) stream;
  GemmArgs g;
  g.a = a; g.a_rs = a_rs; g.a_cs = a_cs;
  g.b = b; g.b_rs = b_rs; g.b_cs = b_cs;
  g.c = c; g.ldc = ldc; g.M = M; g.N = N; g.K = K;
  g.bias = bias; g.mul = mul; g.add = add; g.act = act; g.beta = beta_accumulate ? 1 : 0;
  const bool a_kc = (a_cs == 1);  // reduction index contiguous in A
  const bool b_kc = (b_rs == 1);  // reduction index contiguous in B
  const bool a_vec = ((uintptr_t) a % 16 == 0) && ((a_kc ? a_rs : a_cs) % 4 == 0);
  const bool b_vec = ((uintptr_t) b % 16 == 0) && ((b_kc ? b_cs : b_rs) % 4 == 0);
  const int64_t tiles = b2_ceil_div(M, BM) * b2_ceil_div(N, BN);
  // Split-K (atomic meet) only for purely linear epilogues with few output tiles: wgrad.
  int splits = 1;
  const bool linear = (act == B2_ACT_NONE && mul == nullptr && add == nullptr);
  if (linear && tiles < 2 * B2_NUM_SMS && K >= 8 * BK) {
    splits = (int) b2_ceil_div(3 * B2_NUM_SMS, tiles);
    const int64_t max_splits = K / (4 * BK);
    if (splits > max_splits) splits = (int) max_splits;
    if (splits < 1) splits = 1;
  }
  int64_t k_per = b2_ceil_div(b2_ceil_div(K, splits), BK) * BK;
  if (k_per < BK) k_per = BK;
  splits = (int) b2_ceil_div(K > 0 ? K : 1, k_per);
  g.k_per_split = (int) k_per;
  if (splits > 1 && !g.beta) {
    const int64_t total = M * N;
    int zgrid = (int) (b2_ceil_div(total, 256) < 1184 ? b2_ceil_div(total, 256) : 1184);
    zero_strided_kernel<<<zgrid, 256, 0, st>>>(c, M, N, ldc);
  }
  dim3 grid((unsigned) b2_ceil_div(N, BN), (unsigned) b2_ceil_div(M, BM), (unsigned) splits);
  B2_REQUIRE(grid.y <= 65535, "M too large for this launch geometry");
  if (a_kc && b_kc) sgemm_kernel<true, true><<<grid, 256, 0, st>>>(g, a_vec, b_vec);
  else if (a_kc && !b_kc) sgemm_kernel<true, false><<<grid, 256, 0, st>>>(g, a_vec, b_vec);
  else if (!a_kc && b_kc) sgemm_kernel<false, true><<<grid, 256, 0, st>>>(g, a_vec, b_vec);
  else sgemm_kernel<false, false><<<grid, 256, 0, st>>>(g, a_vec, b_vec);
  B2_CUDA_LAUNCH_CHECK("b2_gemm_f32");
  return B2_OK;
}

// ---------------------------------------------------------------------------------
// Elementwise backward of an activation given its OUTPUT y.
// ---------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
act_bwd_kernel(const float* __restrict__ y, const float* __restrict__ gy, float* __restrict__ gx,
               int64_t n, int act) {
  for (int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (int64_t) gridDim.x * blockDim.x) {
    const float yv = __ldg(y + i), g = __ldg(gy + i);
    float r;
    if (act == B2_ACT_RELU) r = (yv > 0.f) ? g : 0.f;             // threshold_backward
    else if (act == B2_ACT_SIGMOID) r = g * ((1.f - yv) * yv);   // sigmoid_backward
    else r = g;
    gx[i] = r;
  }
}

extern "C" B2_API int b2_act_bwd(const float* y, const float* gy, float* gx, int64_t n, int act,
                          void* stream) {
  B2_REQUIRE(y && gy && gx, "NULL pointer");
  B2_REQUIRE(act >= B2_ACT_NONE && act <= B2_ACT_SIGMOID, "bad activation code %d", act);
  if (n == 0) return B2_OK;
  int64_t blocks = b2_ceil_div(n, 256);
  if (blocks > (int64_t) B2_NUM_SMS * 8) blocks = (int64_t) B2_NUM_SMS * 8;
  act_bwd_kernel<<<(int) blocks, 256, 0, (cudaStream_t) stream>>>(y, gy, gx, n, act);
  B2_CUDA_LAUNCH_CHECK("b2_act_bwd");
  return B2_OK;
}

// ---------------------------------------------------------------------------------
// Column sums (bias gradients): out[n] (+)= sum_m x[m, n].
// CTA = 32 columns x 8 row-lanes; grid.y splits the rows; partials meet with `red`.
// ---------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
colsum_kernel(const float* __restrict__ x, int64_t M, int64_t N, int64_t ld,
              float* __restrict__ out, int64_t rows_per_cta) {
  __shared__ float sm[8][33];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int64_t n = (int64_t) blockIdx.x * 32 + tx;
  const int64_t r0 = (int64_t) blockIdx.y * rows_per_cta;
  const int64_t r1 = min(M, r0 + rows_per_cta);
  float acc = 0.f;
  if (n < N)
    for (int64_t m = r0 + ty; m < r1; m += 8) acc += __ldg(x + m * ld + n);
  sm[ty][tx] = acc;
  __syncthreads();
  if (ty == 0 && n < N) {
    float t = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) t += sm[i][tx];
    b2_red_add(out + n, t);
  }
}

extern "C" B2_API int b2_colsum(const float* x, int64_t M, int64_t N, int64_t ld, float* out,
                         int accumulate, void* stream) {
  B2_REQUIRE(x && out, "NULL pointer");
  B2_REQUIRE(M >= 0 && N >= 1 && ld >= N, "bad shape");
  cudaStream_t st = (cudaStream_t) stream;
  if (!accumulate) {
    cudaError_t e = cudaMemsetAsync(out, 0, sizeof(float) * N, st);
    if (e != cudaSuccess) return b2_fail(B2_E_CUDA, "b2_colsum: memset: %s", cudaGetErrorString(e));
  }
  if (M == 0) return B2_OK;
  const int64_t col_blocks = b2_ceil_div(N, 32);
  int64_t row_splits = b2_ceil_div(2 * B2_NUM_SMS, col_blocks);
  if (row_splits > b2_ceil_div(M, 64)) row_splits = b2_ceil_div(M, 64);
  if (row_splits < 1) row_splits = 1;
  const int64_t rows_per_cta = b2_ceil_div(M, row_splits);
  dim3 grid((unsigned) col_blocks, (unsigned) b2_ceil_div(M, rows_per_cta));
  colsum_kernel<<<grid, 256, 0, st>>>(x, M, N, ld, out, rows_per_cta);
  B2_CUDA_LAUNCH_CHECK("b2_colsum");
  return B2_OK;
}

// ---------------------------------------------------------------------------------
// Fused logit sum + sigmoid + binary cross entropy (mean) + dL/dlogit.
//   p = 1/(1+exp(-z))                                    nn.Sigmoid, rank_model.py:447-448
//   l = -(y*max(log p,-100) + (1-y)*max(log(1-p),-100))  F.binary_cross_entropy
//   dz = (p-y)/max((1-p)*p, 1e-12) * (1-p)*p / B         binary_cross_entropy_backward o sigmoid_backward
// ---------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
logit_bce_kernel(const float* __restrict__ t0, const float* __restrict__ t1,
                 const float* __restrict__ t2, const float* __restrict__ t3,
                 const float* __restrict__ label, int64_t batch, float* __restrict__ y_pred,
                 float* __restrict__ loss, float* __restrict__ glogit) {
  b2_pdl_wait();
  b2_pdl_trigger();
  __shared__ float red[32];
  const float inv_b = 1.f / (float) batch;
  float part = 0.f;
  for (int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; i < batch;
       i += (int64_t) gridDim.x * blockDim.x) {
    float z = __ldg(t0 + i);
    if (t1 != nullptr) z += __ldg(t1 + i);
    if (t2 != nullptr) z += __ldg(t2 + i);
    if (t3 != nullptr) z += __ldg(t3 + i);
    const float p = 1.f / (1.f + expf(-z));
    if (y_pred != nullptr) y_pred[i] = p;
    if (label != nullptr) {
      const float y = __ldg(label + i);
      const float lp = fmaxf(logf(p), -100.f), lq = fmaxf(logf(1.f - p), -100.f);
      part += -(y * lp + (1.f - y) * lq);
      if (glogit != nullptr) {
        const float pq = (1.f - p) * p;
        glogit[i] = ((p - y) / fmaxf(pq, 1e-12f)) * inv_b * pq;
      }
    }
  }
  if (loss != nullptr) {
    const float t = b2_block_sum(part, red);
    if (threadIdx.x == 0) b2_red_add(loss, t * inv_b);
  }
}

extern "C" B2_API int b2_logit_bce_fwd(const float* t0, const float* t1, const float* t2,
                                const float* t3, const float* label, int64_t batch,
                                float* y_pred, float* loss, float* glogit, void* stream) {
  B2_REQUIRE(t0 != nullptr, "first logit term is NULL");
  B2_REQUIRE(batch >= 1, "batch must be >= 1");
  B2_REQUIRE(label != nullptr || (loss == nullptr && glogit == nullptr), "loss/glogit need labels");
  cudaStream_t st = (cudaStream_t) stream;
  if (loss != nullptr) {
    cudaError_t e = cudaMemsetAsync(loss, 0, sizeof(float), st);
    if (e != cudaSuccess) return b2_fail(B2_E_CUDA, "b2_logit_bce_fwd: memset: %s", cudaGetErrorString(e));
  }
  int64_t blocks = b2_ceil_div(batch, 256);
  if (blocks > B2_NUM_SMS * 4) blocks = B2_NUM_SMS * 4;
  B2_LAUNCH(logit_bce_kernel, (int) blocks, 256, 0, st, t0, t1, t2, t3, label, batch, y_pred, loss, glogit);
  B2_CUDA_LAUNCH_CHECK("b2_logit_bce_fwd");
  return B2_OK;
}

// ---------------------------------------------------------------------------------
// Dense clip_grad_norm_ + Adam over a flat fp32 arena (rank_model.py:321-322).
// HBM-bound streaming: float4, grid = whole waves of B2_NUM_SMS (132) SMs.
// ---------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
sumsq_kernel(const float* __restrict__ g, int64_t n, float* __restrict__ out) {
  b2_pdl_wait();
  b2_pdl_trigger();
  __shared__ float red[32];
  float acc = 0.f;
  const int64_t n4 = n >> 2;
  const float4* g4 = reinterpret_cast<const float4*>(g);
  for (int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; i < n4;
       i += (int64_t) gridDim.x * blockDim.x) {
    const float4 v = b2_ldg_stream(g4 + i);
    acc += (v.x * v.x + v.y * v.y) + (v.z * v.z + v.w * v.w);
  }
  if (blockIdx.x == 0 && threadIdx.x < (n & 3)) {
    const float v = g[(n4 << 2) + threadIdx.x];
    acc += v * v;
  }
  const float t = b2_block_sum(acc, red);
  if (threadIdx.x == 0) b2_red_add(out, t);
}

extern "C" B2_API int b2_sumsq(const float* g, int64_t n, float* out, void* stream) {
  B2_REQUIRE(g && out, "NULL pointer");
  B2_REQUIRE(((uintptr_t) g % 16) == 0, "gradient arena must be 16-byte aligned");
  if (n <= 0) return B2_OK;
  int64_t blocks = b2_ceil_div(n >> 2, 256 * 4);
  if (blocks > (int64_t) B2_NUM_SMS * 8) blocks = (int64_t) B2_NUM_SMS * 8;
  if (blocks < 1) blocks = 1;
  B2_LAUNCH(sumsq_kernel, (int) blocks, 256, 0, (cudaStream_t) stream, g, n, out);
  B2_CUDA_LAUNCH_CHECK("b2_sumsq");
  return B2_OK;
}

// sched[step] is written first so that the dense pass and every later lazy catch-up of the same
// step read the SAME two scalars.
__global__ void adam_sched_kernel(const int64_t* __restrict__ step_dev, float lr, float beta1, float beta2,
                                  B2AdamSched* __restrict__ sched, int64_t sched_len) {
  const int64_t t = *step_dev;
  if (t < 1 || t >= sched_len) return;
  const double bc1 = 1.0 - pow((double) beta1, (double) t);
  const double bc2 = 1.0 - pow((double) beta2, (double) t);
  sched[t] = make_float2((float) ((double) lr / bc1), (float) (1.0 / sqrt(bc2)));
}

__global__ void __launch_bounds__(256)
adam_kernel(float* __restrict__ p, float* __restrict__ g, float* __restrict__ m,
            float* __restrict__ v, int64_t n, const float* __restrict__ sumsq, float max_norm,
            float lr, float beta1, float beta2, float eps, const int64_t* __restrict__ step_dev,
            int zero_grad, const B2AdamSched* __restrict__ sched) {
  b2_pdl_wait();
  b2_pdl_trigger();
  __shared__ B2AdamConst sc;
  __shared__ float s_clip, s_step, s_ibc2;
  if (threadIdx.x == 0) {
    const int64_t t = *step_dev;
    float clip = 1.f;
    if (sumsq != nullptr) {
      const float total_norm = sqrtf(*sumsq);
      clip = fminf(max_norm / (total_norm + 1e-6f), 1.f);
    }
    s_clip = clip;
    sc.w1 = (float) (1.0 - (double) beta1);
    sc.b2 = beta2;
    sc.w2 = (float) (1.0 - (double) beta2);
    sc.eps = eps;
    if (sched != nullptr) {
      const B2AdamSched e = sched[t];
      s_step = e.x;
      s_ibc2 = e.y;
    } else {
      const double bc1 = 1.0 - pow((double) beta1, (double) t);
      const double bc2 = 1.0 - pow((double) beta2, (double) t);
      s_step = (float) ((double) lr / bc1);
      s_ibc2 = (float) (1.0 / sqrt(bc2));
    }
  }
  __syncthreads();
  const B2AdamConst c = sc;
  const float clip = s_clip, step_size = s_step, ibc2 = s_ibc2;
  const int64_t n4 = n >> 2;
  float4* p4 = reinterpret_cast<float4*>(p);
  float4* g4 = reinterpret_cast<float4*>(g);
  float4* m4 = reinterpret_cast<float4*>(m);
  float4* v4 = reinterpret_cast<float4*>(v);
  for (int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; i < n4;
       i += (int64_t) gridDim.x * blockDim.x) {
    float4 pp = p4[i], gg = g4[i], mm = m4[i], vv = v4[i];
    b2_adam_apply(pp.x, __fmul_rn(gg.x, clip), mm.x, vv.x, c, step_size, ibc2);   // g.mul_(clip_coef) first
    b2_adam_apply(pp.y, __fmul_rn(gg.y, clip), mm.y, vv.y, c, step_size, ibc2);
    b2_adam_apply(pp.z, __fmul_rn(gg.z, clip), mm.z, vv.z, c, step_size, ibc2);
    b2_adam_apply(pp.w, __fmul_rn(gg.w, clip), mm.w, vv.w, c, step_size, ibc2);
    p4[i] = pp; m4[i] = mm; v4[i] = vv;
    // zero_grad fused in; rows no sample touched are already zero (most of a table): skip their 16-byte store
    if (zero_grad && (gg.x != 0.f || gg.y != 0.f || gg.z != 0.f || gg.w != 0.f)) g4[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
  if (blockIdx.x == 0 && threadIdx.x < (n & 3)) {
    const int64_t i = (n4 << 2) + threadIdx.x;
    float pp = p[i], mm = m[i], vv = v[i];
    b2_adam_apply(pp, __fmul_rn(g[i], clip), mm, vv, c, step_size, ibc2);
    p[i] = pp; m[i] = mm; v[i] = vv;
    if (zero_grad) g[i] = 0.f;
  }
}

extern "C" B2_API int b2_adam_step(float* p, float* g, float* m, float* v, int64_t n,
                            const float* sumsq, float max_norm, float lr, float beta1,
                            float beta2, float eps, const int64_t* step_dev, int zero_grad,
                            void* stream) {
  B2_REQUIRE(p && g && m && v && step_dev, "NULL pointer");
  B2_REQUIRE((((uintptr_t) p | (uintptr_t) g | (uintptr_t) m | (uintptr_t) v) % 16) == 0,
             "arenas must be 16-byte aligned");
  if (n <= 0) return B2_OK;
  int64_t blocks = b2_ceil_div(n >> 2, 256 * 2);
  if (blocks > (int64_t) B2_NUM_SMS * 8) blocks = (int64_t) B2_NUM_SMS * 8;
  if (blocks < 1) blocks = 1;
  const B2AdamSched* no_sched = nullptr;
  B2_LAUNCH(adam_kernel, (int) blocks, 256, 0, (cudaStream_t) stream, p, g, m, v, n, sumsq, max_norm, lr, beta1, beta2,
            eps, step_dev, zero_grad, no_sched);
  B2_CUDA_LAUNCH_CHECK("b2_adam_step");
  return B2_OK;
}

extern "C" B2_API int b2_adam_sched(const int64_t* step_dev, float lr, float beta1, float beta2, float* sched,
                                    int64_t sched_len, void* stream) {
  B2_REQUIRE(step_dev && sched && sched_len >= 2, "NULL pointer / empty schedule table");
  adam_sched_kernel<<<1, 1, 0, (cudaStream_t) stream>>>(step_dev, lr, beta1, beta2,
                                                        reinterpret_cast<B2AdamSched*>(sched), sched_len);
  B2_CUDA_LAUNCH_CHECK("b2_adam_sched");
  return B2_OK;
}

extern "C" B2_API int b2_adam_step_sched(float* p, float* g, float* m, float* v, int64_t n, const float* sumsq,
                                         float max_norm, float beta1, float beta2, float eps,
                                         const int64_t* step_dev, const float* sched, int zero_grad,
                                         void* stream) {
  B2_REQUIRE(p && g && m && v && step_dev && sched, "NULL pointer");
  B2_REQUIRE((((uintptr_t) p | (uintptr_t) g | (uintptr_t) m | (uintptr_t) v) % 16) == 0,
             "arenas must be 16-byte aligned");
  if (n <= 0) return B2_OK;
  int64_t blocks = b2_ceil_div(n >> 2, 256 * 2);
  if (blocks > (int64_t) B2_NUM_SMS * 8) blocks = (int64_t) B2_NUM_SMS * 8;
  if (blocks < 1) blocks = 1;
  const B2AdamSched* sched_tab = reinterpret_cast<const B2AdamSched*>(sched);
  B2_LAUNCH(adam_kernel, (int) blocks, 256, 0, (cudaStream_t) stream, p, g, m, v, n, sumsq, max_norm, 0.f, beta1, beta2,
            eps, step_dev, zero_grad, sched_tab);
  B2_CUDA_LAUNCH_CHECK("b2_adam_step_sched");
  return B2_OK;
}

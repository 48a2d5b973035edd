// dien.cu — the Deep Interest Evolution Network's recurrences and attention scores (model_zoo/DIEN/src/DIEN.py),
// sm_90a.
//
// GRU, AUGRU and AGRU are one cell, h' = h + g (n - h), selected by a cell code (include/fuxictr_b200.h "DIEN").
// A CTA of DIEN_THREADS threads takes S = DIEN_THREADS / G samples, G the power of two >= H: thread j of a sample's
// group owns hidden unit j, computes the three gate rows j, H + j, 2H + j of W_ih x_t and W_hh h, and keeps its h_j in
// a register.  W_ih and W_hh sit in shared memory row-major at an odd row pitch P, so a warp reading one column across
// rows (the gates) or one row across columns (the backward's W^T products) meets no bank conflict.  x_t and h are
// exchanged through shared memory.  The input projection is folded into the recurrence: at H <= 64 a tensor-core GEMM
// with K = H would write a (B L, 3H) gate tensor, three times the sequence's bytes, to save a few FMAs.
//
// Every thread of a CTA walks all L positions, so the barriers are uniform; a sample past its length only carries its
// state.  The forward double-buffers x_t and h (one barrier per step).  The backward recomputes the gates from the
// saved h_{t-1} and x_t, and accumulates the weight gradients of all its samples in shared memory (each thread owns a
// fixed set of elements, no atomics), then issues one float atomic per element and CTA.
// All arithmetic is fp32 on CUDA cores, expf and tanhf; the lengths come from the byte mask on the device.
#include "b2_common.cuh"

#define DIEN_THREADS 256

static inline int dien_group(int H) {
  int g = 1;
  while (g < H) g <<= 1;
  return g;
}
static inline int dien_pitch(int H) { return H | 1; }

__device__ __forceinline__ float dien_sigmoid(float v) { return 1.f / (1.f + expf(-v)); }

// Stage W_ih, W_hh (3H, H) at row pitch P and the biases; count each sample's length.
__device__ __forceinline__ void dien_stage(const float* __restrict__ W_ih, const float* __restrict__ b_ih,
                                           const float* __restrict__ W_hh, const float* __restrict__ b_hh, int H,
                                           int P, float* sWi, float* sWh, float* sbi, float* sbh) {
  for (int e = threadIdx.x; e < 3 * H * H; e += blockDim.x) {
    const int row = e / H, k = e - row * H;
    sWi[row * P + k] = __ldg(W_ih + e);
    sWh[row * P + k] = __ldg(W_hh + e);
  }
  for (int e = threadIdx.x; e < 3 * H; e += blockDim.x) {
    sbi[e] = b_ih ? __ldg(b_ih + e) : 0.f;
    sbh[e] = b_hh ? __ldg(b_hh + e) : 0.f;
  }
}

__device__ __forceinline__ void dien_count(const uint8_t* __restrict__ mask, int64_t b, int64_t batch, int L, int j,
                                           int G, int s, int* lens) {
  if (b < batch) {
    int c = 0;
    for (int t = j; t < L; t += G) c += mask[b * L + t] != 0;
    if (c) atomicAdd(lens + s, c);
  }
}

// The three gate rows c * H + j of W v + bias, for c in [c0, 3).
__device__ __forceinline__ void dien_gates(const float* sW, const float* sb, const float* v, int H, int P, int j,
                                           bool three, float& g0, float& g1, float& g2) {
  const float* w0 = sW + j * P;
  const float* w1 = sW + (H + j) * P;
  const float* w2 = sW + (2 * H + j) * P;
  float a0 = three ? sb[j] : 0.f, a1 = sb[H + j], a2 = sb[2 * H + j];
  if (three) {
#pragma unroll 4
    for (int k = 0; k < H; ++k) {
      const float vk = v[k];
      a0 = fmaf(w0[k], vk, a0);
      a1 = fmaf(w1[k], vk, a1);
      a2 = fmaf(w2[k], vk, a2);
    }
  } else {
#pragma unroll 4
    for (int k = 0; k < H; ++k) {
      const float vk = v[k];
      a1 = fmaf(w1[k], vk, a1);
      a2 = fmaf(w2[k], vk, a2);
    }
  }
  g0 = a0; g1 = a1; g2 = a2;
}

__global__ void __launch_bounds__(DIEN_THREADS)
dien_gru_fwd_kernel(const float* __restrict__ x, int64_t ld_x, const uint8_t* __restrict__ mask,
                    const float* __restrict__ W_ih, const float* __restrict__ b_ih, const float* __restrict__ W_hh,
                    const float* __restrict__ b_hh, const float* __restrict__ att, int cell, int64_t batch, int L,
                    int H, int G, float* __restrict__ h_seq, float* __restrict__ h_last) {
  extern __shared__ float smem[];
  const int P = H | 1, S = DIEN_THREADS / G;
  float* sWi = smem;
  float* sWh = sWi + 3 * H * P;
  float* sbi = sWh + 3 * H * P;
  float* sbh = sbi + 3 * H;
  float* xs = sbh + 3 * H;          // [2][S][H]
  float* hs = xs + 2 * S * H;       // [2][S][H]
  int* lens = reinterpret_cast<int*>(hs + 2 * S * H);
  const int s = threadIdx.x / G, j = threadIdx.x - s * G;
  const int64_t b = (int64_t) blockIdx.x * S + s;
  const bool active = b < batch && j < H;
  if (threadIdx.x < S) lens[threadIdx.x] = 0;
  b2_pdl_wait();
  dien_stage(W_ih, b_ih, W_hh, b_hh, H, P, sWi, sWh, sbi, sbh);
  __syncthreads();
  dien_count(mask, b, batch, L, j, G, s, lens);
  __syncthreads();
  const int len = b < batch ? lens[s] : 0;
  const float* xb = x + b * ld_x;
  float* hb = h_seq + b * (int64_t) L * H;
  float h = 0.f;
  if (active) {
    hs[s * H + j] = 0.f;
    if (len > 0) xs[s * H + j] = __ldg(xb + j);
  }
  const bool three = cell != B2_DIEN_AGRU;
  __syncthreads();
  for (int t = 0; t < L; ++t) {
    const int cur = t & 1, nxt = cur ^ 1;
    if (active) {
      if (t < len) {
        float i0, i1, i2, g0, g1, g2;
        dien_gates(sWi, sbi, xs + (cur * S + s) * H, H, P, j, three, i0, i1, i2);
        dien_gates(sWh, sbh, hs + (cur * S + s) * H, H, P, j, three, g0, g1, g2);
        float g, r;
        if (cell == B2_DIEN_GRU) {
          r = dien_sigmoid(i0 + g0);
          g = 1.f - dien_sigmoid(i1 + g1);
        } else {
          r = dien_sigmoid(i1 + g1);
          const float a = __ldg(att + b * L + t);
          g = cell == B2_DIEN_AUGRU ? a * dien_sigmoid(i0 + g0) : a;
        }
        const float n = tanhf(i2 + r * g2);
        h = h + g * (n - h);
        hb[(int64_t) t * H + j] = h;
        hs[(nxt * S + s) * H + j] = h;
        if (t + 1 < len) xs[(nxt * S + s) * H + j] = __ldg(xb + (int64_t) (t + 1) * H + j);
      } else {
        hb[(int64_t) t * H + j] = 0.f;
      }
    }
    __syncthreads();
  }
  b2_pdl_trigger();
  if (active && h_last) h_last[b * H + j] = h;
}

__global__ void __launch_bounds__(DIEN_THREADS)
dien_gru_bwd_kernel(const float* __restrict__ x, int64_t ld_x, const uint8_t* __restrict__ mask,
                    const float* __restrict__ W_ih, const float* __restrict__ b_ih, const float* __restrict__ W_hh,
                    const float* __restrict__ b_hh, const float* __restrict__ att, int cell, int64_t batch, int L,
                    int H, int G, const float* __restrict__ h_seq, const float* __restrict__ dh_seq,
                    const float* __restrict__ dh_last, float* __restrict__ dx, int accumulate, float* __restrict__ da,
                    float* __restrict__ dW_ih, float* __restrict__ db_ih, float* __restrict__ dW_hh,
                    float* __restrict__ db_hh) {
  extern __shared__ float smem[];
  const int P = H | 1, S = DIEN_THREADS / G, H3 = 3 * H;
  float* sWi = smem;
  float* sWh = sWi + H3 * P;
  float* sbi = sWh + H3 * P;
  float* sbh = sbi + H3;
  float* gWi = sbh + H3;            // [3H][H] weight-gradient partial sums of this CTA
  float* gWh = gWi + H3 * H;
  float* gbi = gWh + H3 * H;        // [3H]
  float* gbh = gbi + H3;
  float* xs = gbh + H3;             // [S][H] x_t
  float* hp = xs + S * H;           // [S][H] h_{t-1}
  float* dgi = hp + S * H;          // [S][3H]
  float* dgh = dgi + S * H3;        // [S][3H]
  float* dgu = dgh + S * H3;        // [S][H] the terms of da
  int* lens = reinterpret_cast<int*>(dgu + S * H);
  const int s = threadIdx.x / G, j = threadIdx.x - s * G;
  const int64_t b = (int64_t) blockIdx.x * S + s;
  const bool active = b < batch && j < H;
  if (threadIdx.x < S) lens[threadIdx.x] = 0;
  for (int e = threadIdx.x; e < 2 * H3 * H + 2 * H3; e += blockDim.x) gWi[e] = 0.f;
  b2_pdl_wait();
  dien_stage(W_ih, b_ih, W_hh, b_hh, H, P, sWi, sWh, sbi, sbh);
  __syncthreads();
  dien_count(mask, b, batch, L, j, G, s, lens);
  __syncthreads();
  const int len = b < batch ? lens[s] : 0;
  const float* xb = x + b * ld_x;
  const int64_t row0 = b * (int64_t) L;
  const bool three = cell != B2_DIEN_AGRU;
  float dh = (active && dh_last) ? __ldg(dh_last + b * H + j) : 0.f;
  for (int t = L - 1; t >= 0; --t) {
    const bool on = active && t < len;
    if (j < H) {
      xs[s * H + j] = on ? __ldg(xb + (int64_t) t * H + j) : 0.f;
      hp[s * H + j] = (on && t > 0) ? __ldg(h_seq + (row0 + t - 1) * H + j) : 0.f;
    }
    if (on && dh_seq) dh += __ldg(dh_seq + (row0 + t) * H + j);
    __syncthreads();
    float keep = 1.f;
    if (j < H) {
      float d0 = 0.f, d1 = 0.f, d2 = 0.f, e0 = 0.f, e1 = 0.f, e2 = 0.f, du = 0.f;
      if (on) {
        float i0, i1, i2, g0, g1, g2;
        dien_gates(sWi, sbi, xs + s * H, H, P, j, three, i0, i1, i2);
        dien_gates(sWh, sbh, hp + s * H, H, P, j, three, g0, g1, g2);
        const float h = hp[s * H + j];
        const bool gru = cell == B2_DIEN_GRU;
        const float r = dien_sigmoid(gru ? i0 + g0 : i1 + g1);
        const float n = tanhf(i2 + r * g2);
        const float a = gru ? 0.f : __ldg(att + row0 + t);
        const float z = three ? dien_sigmoid(gru ? i1 + g1 : i0 + g0) : 0.f;   // GRU: z; AUGRU: u
        const float g = gru ? 1.f - z : (cell == B2_DIEN_AUGRU ? a * z : a);
        const float dg = dh * (n - h);
        const float dpn = dh * g * (1.f - n * n);
        const float dpr = dpn * g2 * r * (1.f - r);
        d2 = dpn;
        e2 = dpn * r;
        keep = 1.f - g;
        if (gru) {
          const float dpz = -dg * z * (1.f - z);
          d0 = e0 = dpr;
          d1 = e1 = dpz;
        } else {
          d1 = e1 = dpr;
          if (cell == B2_DIEN_AUGRU) {
            d0 = e0 = dg * a * z * (1.f - z);
            du = dg * z;
          } else {
            du = dg;
          }
        }
      }
      float* di = dgi + s * H3;
      float* dhh = dgh + s * H3;
      di[j] = d0; di[H + j] = d1; di[2 * H + j] = d2;
      dhh[j] = e0; dhh[H + j] = e1; dhh[2 * H + j] = e2;
      dgu[s * H + j] = du;
    }
    __syncthreads();
    if (j < H) {
      const float* di = dgi + s * H3;
      const float* dhh = dgh + s * H3;
      if (on) {
        float ax = 0.f, ah = 0.f;
#pragma unroll 4
        for (int row = 0; row < H3; ++row) {
          ax = fmaf(sWi[row * P + j], di[row], ax);
          ah = fmaf(sWh[row * P + j], dhh[row], ah);
        }
        float* px = dx + (row0 + t) * H + j;
        *px = accumulate ? *px + ax : ax;
        dh = dh * keep + ah;
      } else if (active && !accumulate) {
        dx[(row0 + t) * H + j] = 0.f;
      }
      // this thread's weight-gradient elements: rows s, s + S, ..., column j, summed over the CTA's samples
      for (int row = s; row < H3; row += S) {
        float ai = 0.f, ah = 0.f;
        for (int q = 0; q < S; ++q) {
          ai = fmaf(dgi[q * H3 + row], xs[q * H + j], ai);
          ah = fmaf(dgh[q * H3 + row], hp[q * H + j], ah);
        }
        gWi[row * H + j] += ai;
        gWh[row * H + j] += ah;
      }
    }
    if (da && j == 0 && b < batch) {
      float acc = 0.f;
      if (t < len)
        for (int k = 0; k < H; ++k) acc += dgu[s * H + k];
      da[row0 + t] = acc;
    }
    for (int row = threadIdx.x; row < H3; row += blockDim.x) {
      float ai = 0.f, ah = 0.f;
      for (int q = 0; q < S; ++q) {
        ai += dgi[q * H3 + row];
        ah += dgh[q * H3 + row];
      }
      gbi[row] += ai;
      gbh[row] += ah;
    }
    __syncthreads();
  }
  b2_pdl_trigger();
  for (int e = threadIdx.x; e < H3 * H; e += blockDim.x) {
    b2_red_add(dW_ih + e, gWi[e]);
    b2_red_add(dW_hh + e, gWh[e]);
  }
  for (int e = threadIdx.x; e < H3; e += blockDim.x) {
    if (db_ih) b2_red_add(db_ih + e, gbi[e]);
    if (db_hh) b2_red_add(db_hh + e, gbh[e]);
  }
}

// ---------------------------------------------------------------------------------
// Attention scores (bilinear / dot) and sum pooling: a group of G threads per sample, as above
// ---------------------------------------------------------------------------------
__global__ void __launch_bounds__(DIEN_THREADS)
dien_scores_fwd_kernel(const float* __restrict__ h_seq, const float* __restrict__ tg, int64_t ld_t,
                       const float* __restrict__ W, const uint8_t* __restrict__ mask, int64_t batch, int L, int H,
                       int G, float* __restrict__ q, float* __restrict__ sc) {
  extern __shared__ float smem[];
  const int S = DIEN_THREADS / G;
  float* ts = smem;                 // [S][H]
  float* qs = ts + S * H;           // [S][H]
  const int s = threadIdx.x / G, j = threadIdx.x - s * G;
  const int64_t b = (int64_t) blockIdx.x * S + s;
  const bool active = b < batch && j < H;
  b2_pdl_wait();
  if (active) ts[s * H + j] = __ldg(tg + b * ld_t + j);
  __syncthreads();
  if (active) {
    float v;
    if (W) {
      v = 0.f;
      for (int k = 0; k < H; ++k) v = fmaf(__ldg(W + j * H + k), ts[s * H + k], v);
    } else {
      v = ts[s * H + j];
    }
    qs[s * H + j] = v;
    q[b * H + j] = v;
  }
  __syncthreads();
  b2_pdl_trigger();
  if (b >= batch) return;
  const float* hb = h_seq + b * (int64_t) L * H;
  for (int t = j; t < L; t += G) {
    float v = 0.f;
    if (mask[b * L + t]) {
      for (int k = 0; k < H; ++k) v = fmaf(__ldg(hb + (int64_t) t * H + k), qs[s * H + k], v);
    }
    sc[b * L + t] = v;
  }
}

__global__ void __launch_bounds__(DIEN_THREADS)
dien_scores_bwd_kernel(const float* __restrict__ h_seq, const float* __restrict__ W, const uint8_t* __restrict__ mask,
                       const float* __restrict__ q, const float* __restrict__ ds, int64_t batch, int L, int H, int G,
                       float* __restrict__ dh_seq, int accumulate, float* __restrict__ dq, float* __restrict__ dt) {
  extern __shared__ float smem[];
  const int S = DIEN_THREADS / G;
  float* dqs = smem;                // [S][H]
  const int s = threadIdx.x / G, j = threadIdx.x - s * G;
  const int64_t b = (int64_t) blockIdx.x * S + s;
  const bool active = b < batch && j < H;
  b2_pdl_wait();
  if (active) {
    const float qj = __ldg(q + b * H + j);
    const float* hb = h_seq + b * (int64_t) L * H;
    float* gb = dh_seq + b * (int64_t) L * H;
    float acc = 0.f;
    for (int t = 0; t < L; ++t) {
      const float d = mask[b * L + t] ? __ldg(ds + b * L + t) : 0.f;
      acc = fmaf(d, __ldg(hb + (int64_t) t * H + j), acc);
      float* p = gb + (int64_t) t * H + j;
      *p = accumulate ? fmaf(d, qj, *p) : d * qj;
    }
    dqs[s * H + j] = acc;
    dq[b * H + j] = acc;
  }
  __syncthreads();
  b2_pdl_trigger();
  if (active) {
    float v;
    if (W) {
      v = 0.f;
      for (int i = 0; i < H; ++i) v = fmaf(__ldg(W + i * H + j), dqs[s * H + i], v);
    } else {
      v = dqs[s * H + j];
    }
    dt[b * H + j] = v;
  }
}

__global__ void __launch_bounds__(DIEN_THREADS)
dien_sum_pool_fwd_kernel(const float* __restrict__ x, const float* __restrict__ tg, int64_t ld_t, int64_t batch, int L,
                         int H, int G, float* __restrict__ out, int64_t ld_out) {
  const int S = DIEN_THREADS / G;
  const int s = threadIdx.x / G, j = threadIdx.x - s * G;
  const int64_t b = (int64_t) blockIdx.x * S + s;
  b2_pdl_wait();
  b2_pdl_trigger();
  if (b >= batch || j >= H) return;
  const float* xb = x + b * (int64_t) L * H;
  float acc = 0.f;
  for (int t = 0; t < L; ++t) acc += __ldg(xb + (int64_t) t * H + j);
  out[b * ld_out + j] = acc;
  out[b * ld_out + H + j] = __ldg(tg + b * ld_t + j) * acc;
}

__global__ void __launch_bounds__(DIEN_THREADS)
dien_sum_pool_bwd_kernel(const float* __restrict__ x, const float* __restrict__ tg, int64_t ld_t,
                         const float* __restrict__ g, int64_t ld_g, int64_t batch, int L, int H, int G,
                         float* __restrict__ dx, float* __restrict__ dt, int accumulate) {
  const int S = DIEN_THREADS / G;
  const int s = threadIdx.x / G, j = threadIdx.x - s * G;
  const int64_t b = (int64_t) blockIdx.x * S + s;
  b2_pdl_wait();
  b2_pdl_trigger();
  if (b >= batch || j >= H) return;
  const float* xb = x + b * (int64_t) L * H;
  float* db = dx + b * (int64_t) L * H;
  const float g1 = __ldg(g + b * ld_g + j), g2 = __ldg(g + b * ld_g + H + j);
  const float d = fmaf(__ldg(tg + b * ld_t + j), g2, g1);
  float acc = 0.f;
  for (int t = 0; t < L; ++t) {
    acc += __ldg(xb + (int64_t) t * H + j);
    float* p = db + (int64_t) t * H + j;
    *p = accumulate ? *p + d : d;
  }
  float* pt = dt + b * H + j;
  *pt = accumulate ? fmaf(acc, g2, *pt) : acc * g2;
}

// ---------------------------------------------------------------------------------
// C-ABI
// ---------------------------------------------------------------------------------
static int dien_check(int64_t batch, int L, int H) {
  B2_REQUIRE(H >= 1 && H <= B2_DIEN_MAX_DIM, "DIEN: the GRU width H must lie in [1, %d], got %d", B2_DIEN_MAX_DIM, H);
  B2_REQUIRE(L >= 1 && L <= B2_DIEN_MAX_LEN, "DIEN: the sequence length L must lie in [1, %d], got %d",
             B2_DIEN_MAX_LEN, L);
  B2_REQUIRE(batch >= 0, "DIEN: negative batch %lld", (long long) batch);
  B2_REQUIRE(batch * L < ((int64_t) 1 << 31), "DIEN: batch L must stay below 2^31");
  return B2_OK;
}

static int dien_cell_check(int cell, const float* att) {
  B2_REQUIRE(cell == B2_DIEN_GRU || cell == B2_DIEN_AUGRU || cell == B2_DIEN_AGRU,
             "DIEN: cell code %d is not B2_DIEN_GRU, _AUGRU or _AGRU", cell);
  B2_REQUIRE(cell == B2_DIEN_GRU || att, "DIEN: AUGRU and AGRU need the attention (NULL pointer)");
  return B2_OK;
}

static size_t dien_fwd_smem(int H, int G) {
  const int S = DIEN_THREADS / G;
  return sizeof(float) * (size_t) (6 * H * dien_pitch(H) + 6 * H + 4 * S * H) + sizeof(int) * S;
}

static size_t dien_bwd_smem(int H, int G) {
  const int S = DIEN_THREADS / G;
  return sizeof(float) * (size_t) (6 * H * dien_pitch(H) + 6 * H + 6 * H * H + 6 * H + 2 * S * H + 6 * S * H + S * H) +
         sizeof(int) * S;
}

template <typename K>
static int dien_smem_attr(K kernel, size_t smem, const char* name) {
  if (smem <= 48 * 1024) return B2_OK;
  cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) smem);
  if (e != cudaSuccess) return b2_fail(B2_E_CUDA, "%s: shared memory %zu: %s", name, smem, cudaGetErrorString(e));
  return B2_OK;
}

extern "C" B2_API int b2_gru_fwd(const float* x, int64_t ld_x, const uint8_t* mask, const float* W_ih,
                                 const float* b_ih, const float* W_hh, const float* b_hh, const float* att, int cell,
                                 int64_t batch, int L, int H, float* h_seq, float* h_last, void* stream) {
  if (int rc = dien_check(batch, L, H)) return rc;
  B2_REQUIRE(x && mask && W_ih && b_ih && W_hh && b_hh && h_seq, "NULL pointer");
  if (int rc = dien_cell_check(cell, att)) return rc;
  B2_REQUIRE(ld_x >= (int64_t) L * H, "DIEN: ld_x %lld < L H = %lld", (long long) ld_x, (long long) L * H);
  if (batch == 0) return B2_OK;
  const int G = dien_group(H), S = DIEN_THREADS / G;
  const size_t smem = dien_fwd_smem(H, G);
  if (int rc = dien_smem_attr(dien_gru_fwd_kernel, smem, "b2_gru_fwd")) return rc;
  B2_LAUNCH(dien_gru_fwd_kernel, (unsigned) b2_ceil_div(batch, S), DIEN_THREADS, smem, (cudaStream_t) stream, x, ld_x,
            mask, W_ih, b_ih, W_hh, b_hh, att, cell, batch, L, H, G, h_seq, h_last);
  B2_CUDA_LAUNCH_CHECK("b2_gru_fwd");
  return B2_OK;
}

extern "C" B2_API int b2_gru_bwd(const float* x, int64_t ld_x, const uint8_t* mask, const float* W_ih,
                                 const float* b_ih, const float* W_hh, const float* b_hh, const float* att, int cell,
                                 int64_t batch, int L, int H, const float* h_seq, const float* dh_seq,
                                 const float* dh_last, float* dx, int accumulate, float* da, float* dW_ih, float* db_ih,
                                 float* dW_hh, float* db_hh, void* stream) {
  if (int rc = dien_check(batch, L, H)) return rc;
  B2_REQUIRE(x && mask && W_ih && b_ih && W_hh && b_hh && h_seq && dx && dW_ih && db_ih && dW_hh && db_hh,
             "NULL pointer");
  if (int rc = dien_cell_check(cell, att)) return rc;
  B2_REQUIRE(cell == B2_DIEN_GRU || da, "DIEN: AUGRU and AGRU write da (NULL pointer)");
  B2_REQUIRE(ld_x >= (int64_t) L * H, "DIEN: ld_x %lld < L H = %lld", (long long) ld_x, (long long) L * H);
  if (batch == 0) return B2_OK;
  const int G = dien_group(H), S = DIEN_THREADS / G;
  const size_t smem = dien_bwd_smem(H, G);
  if (int rc = dien_smem_attr(dien_gru_bwd_kernel, smem, "b2_gru_bwd")) return rc;
  B2_LAUNCH(dien_gru_bwd_kernel, (unsigned) b2_ceil_div(batch, S), DIEN_THREADS, smem, (cudaStream_t) stream, x, ld_x,
            mask, W_ih, b_ih, W_hh, b_hh, att, cell, batch, L, H, G, h_seq, dh_seq, dh_last, dx, accumulate,
            cell == B2_DIEN_GRU ? nullptr : da, dW_ih, db_ih, dW_hh, db_hh);
  B2_CUDA_LAUNCH_CHECK("b2_gru_bwd");
  return B2_OK;
}

extern "C" B2_API int b2_dien_scores_fwd(const float* h_seq, const float* t, int64_t ld_t, const float* W,
                                         const uint8_t* mask, int64_t batch, int L, int H, float* q, float* s,
                                         void* stream) {
  if (int rc = dien_check(batch, L, H)) return rc;
  B2_REQUIRE(h_seq && t && mask && q && s, "NULL pointer");
  B2_REQUIRE(ld_t >= H, "DIEN: ld_t %lld < H %d", (long long) ld_t, H);
  if (batch == 0) return B2_OK;
  const int G = dien_group(H), S = DIEN_THREADS / G;
  B2_LAUNCH(dien_scores_fwd_kernel, (unsigned) b2_ceil_div(batch, S), DIEN_THREADS, 2 * S * H * sizeof(float),
            (cudaStream_t) stream, h_seq, t, ld_t, W, mask, batch, L, H, G, q, s);
  B2_CUDA_LAUNCH_CHECK("b2_dien_scores_fwd");
  return B2_OK;
}

extern "C" B2_API int b2_dien_scores_bwd(const float* h_seq, const float* t, int64_t ld_t, const float* W,
                                         const uint8_t* mask, const float* q, const float* ds, int64_t batch, int L,
                                         int H, float* dh_seq, int accumulate, float* dq, float* dt, void* stream) {
  if (int rc = dien_check(batch, L, H)) return rc;
  B2_REQUIRE(h_seq && t && mask && q && ds && dh_seq && dq && dt, "NULL pointer");
  B2_REQUIRE(ld_t >= H, "DIEN: ld_t %lld < H %d", (long long) ld_t, H);
  if (batch == 0) return B2_OK;
  const int G = dien_group(H), S = DIEN_THREADS / G;
  B2_LAUNCH(dien_scores_bwd_kernel, (unsigned) b2_ceil_div(batch, S), DIEN_THREADS, S * H * sizeof(float),
            (cudaStream_t) stream, h_seq, W, mask, q, ds, batch, L, H, G, dh_seq, accumulate, dq, dt);
  B2_CUDA_LAUNCH_CHECK("b2_dien_scores_bwd");
  return B2_OK;
}

extern "C" B2_API int b2_dien_sum_pool_fwd(const float* x, const float* t, int64_t ld_t, int64_t batch, int L, int H,
                                           float* out, int64_t ld_out, void* stream) {
  if (int rc = dien_check(batch, L, H)) return rc;
  B2_REQUIRE(x && t && out, "NULL pointer");
  B2_REQUIRE(ld_t >= H && ld_out >= 2 * H, "DIEN: ld_t %lld < H or ld_out %lld < 2 H (H = %d)", (long long) ld_t,
             (long long) ld_out, H);
  if (batch == 0) return B2_OK;
  const int G = dien_group(H), S = DIEN_THREADS / G;
  B2_LAUNCH(dien_sum_pool_fwd_kernel, (unsigned) b2_ceil_div(batch, S), DIEN_THREADS, 0, (cudaStream_t) stream, x, t,
            ld_t, batch, L, H, G, out, ld_out);
  B2_CUDA_LAUNCH_CHECK("b2_dien_sum_pool_fwd");
  return B2_OK;
}

extern "C" B2_API int b2_dien_sum_pool_bwd(const float* x, const float* t, int64_t ld_t, const float* g, int64_t ld_g,
                                           int64_t batch, int L, int H, float* dx, float* dt, int accumulate,
                                           void* stream) {
  if (int rc = dien_check(batch, L, H)) return rc;
  B2_REQUIRE(x && t && g && dx && dt, "NULL pointer");
  B2_REQUIRE(ld_t >= H && ld_g >= 2 * H, "DIEN: ld_t %lld < H or ld_g %lld < 2 H (H = %d)", (long long) ld_t,
             (long long) ld_g, H);
  if (batch == 0) return B2_OK;
  const int G = dien_group(H), S = DIEN_THREADS / G;
  B2_LAUNCH(dien_sum_pool_bwd_kernel, (unsigned) b2_ceil_div(batch, S), DIEN_THREADS, 0, (cudaStream_t) stream, x, t,
            ld_t, g, ld_g, batch, L, H, G, dx, dt, accumulate);
  B2_CUDA_LAUNCH_CHECK("b2_dien_sum_pool_bwd");
  return B2_OK;
}

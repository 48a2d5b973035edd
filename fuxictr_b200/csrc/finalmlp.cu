// finalmlp.cu — FinalMLP's feature-selection gates and its two-stream interaction aggregation, sm_90a.
//
// Gate (FeatureSelection): f_s = e * (2 g_s) for the two streams s = 1, 2, in one pass over the flattened
// embedding e (B, d).  A gate is one broadcast row (1, d), when it has no context features, or one row per sample.
// The backward writes de = df1 (2 g1) + df2 (2 g2) and dg_s = 2 (df_s e): per row, or for a broadcast gate its
// column sum over the batch (rk_cta_colsum, one float atomic per column and CTA).
//
// Aggregation (InteractionAggregation, output_dim 1): out = w_x.x + b_x + w_y.y + b_y + sum_h x_h^T W_h y_h.  Around
// one GEMM Q = x W_aug^T + [w_y, 0] (W_aug: the block diagonal of the W_h^T, then w_x) this file holds the pack of
// W_aug, the row kernels out = y.Q[:dy] + Q[dy] + b_x + b_y and back, and the unpack of the W_aug gradient.  Layouts:
// include/fuxictr_b200.h "FinalMLP".
#include "row_common.cuh"

// f1 = e * (2 g1), f2 = e * (2 g2) (+ their GEMM-operand copies); a gate row is g_s + row * ldg_s (ldg_s 0: broadcast)
template <int VW>
__global__ void __launch_bounds__(RK_THREADS)
fs_gate_fwd_kernel(const float* __restrict__ e, const float* __restrict__ g1, const float* __restrict__ g2,
                   int64_t ldg1, int64_t ldg2, int64_t batch, int d, int tx_n, float* __restrict__ f1,
                   float* __restrict__ f2, void* f1_aux, void* f2_aux, int aux_dtype, int64_t ld_aux) {
  const int tx = threadIdx.x % tx_n, ty = threadIdx.x / tx_n, ty_n = blockDim.x / tx_n;
  const int c = (blockIdx.y * tx_n + tx) * VW;
  b2_pdl_wait();
  if (c < d) {
    for (int64_t row = (int64_t) blockIdx.x * ty_n + ty; row < batch; row += (int64_t) gridDim.x * ty_n) {
      float x[VW], a[VW], b[VW];
      rk_load<VW>(e + row * d + c, x);
      rk_load<VW>(g1 + row * ldg1 + c, a);
      rk_load<VW>(g2 + row * ldg2 + c, b);
#pragma unroll
      for (int k = 0; k < VW; ++k) {
        a[k] = x[k] * (2.f * a[k]);
        b[k] = x[k] * (2.f * b[k]);
      }
      rk_store<VW>(f1 + row * d + c, a);
      rk_store<VW>(f2 + row * d + c, b);
      if (f1_aux) {
        rk_store_aux<VW>(f1_aux, aux_dtype, row * ld_aux + c, a);
        rk_store_aux<VW>(f2_aux, aux_dtype, row * ld_aux + c, b);
      }
    }
  }
  b2_pdl_trigger();
}

// de = df1 (2 g1) + df2 (2 g2); dg_s = 2 (df_s e), per row (ldg_s = d, "=") or summed over the rows (ldg_s = 0, "+=")
template <int VW>
__global__ void __launch_bounds__(RK_THREADS)
fs_gate_bwd_kernel(const float* __restrict__ e, const float* __restrict__ g1, const float* __restrict__ g2,
                   int64_t ldg1, int64_t ldg2, const float* __restrict__ df1, const float* __restrict__ df2,
                   int64_t batch, int d, int tx_n, float* __restrict__ de, float* __restrict__ dg1,
                   float* __restrict__ dg2) {
  __shared__ float red[RK_THREADS * VW];
  const int tx = threadIdx.x % tx_n, ty = threadIdx.x / tx_n, ty_n = blockDim.x / tx_n;
  const int c = (blockIdx.y * tx_n + tx) * VW;
  float acc1[VW], acc2[VW];
#pragma unroll
  for (int k = 0; k < VW; ++k) acc1[k] = acc2[k] = 0.f;
  b2_pdl_wait();
  if (c < d) {
    for (int64_t row = (int64_t) blockIdx.x * ty_n + ty; row < batch; row += (int64_t) gridDim.x * ty_n) {
      float x[VW], a[VW], b[VW], u[VW], v[VW];
      rk_load<VW>(e + row * d + c, x);
      rk_load<VW>(g1 + row * ldg1 + c, a);
      rk_load<VW>(g2 + row * ldg2 + c, b);
      rk_load<VW>(df1 + row * d + c, u);
      rk_load<VW>(df2 + row * d + c, v);
#pragma unroll
      for (int k = 0; k < VW; ++k) {
        a[k] = u[k] * (2.f * a[k]) + v[k] * (2.f * b[k]);     // de
        u[k] = 2.f * (u[k] * x[k]);                            // dg1
        v[k] = 2.f * (v[k] * x[k]);                            // dg2
      }
      rk_store<VW>(de + row * d + c, a);
      if (ldg1) rk_store<VW>(dg1 + row * d + c, u);
      if (ldg2) rk_store<VW>(dg2 + row * d + c, v);
#pragma unroll
      for (int k = 0; k < VW; ++k) {
        acc1[k] += u[k];
        acc2[k] += v[k];
      }
    }
  }
  b2_pdl_trigger();
  if (ldg1 == 0) {
    rk_cta_colsum<VW>(red, tx, tx_n, ty_n, acc1);
    if (ty == 0 && c < d)
#pragma unroll
      for (int k = 0; k < VW; ++k)
        if (acc1[k] != 0.f) b2_red_add(dg1 + c + k, acc1[k]);
    __syncthreads();                                   // red is reused below
  }
  if (ldg2 == 0) {
    rk_cta_colsum<VW>(red, tx, tx_n, ty_n, acc2);
    if (ty == 0 && c < d)
#pragma unroll
      for (int k = 0; k < VW; ++k)
        if (acc2[k] != 0.f) b2_red_add(dg2 + c + k, acc2[k]);
  }
}

// W_aug (n_aug, dx): row r < dy is head h = r / hy's W_h column r % hy over that head's x columns, zero elsewhere;
// row dy is w_x; the rest are zero.  bias_aug (n_aug) = [w_y, 0 ...].  ("=")
__global__ void __launch_bounds__(256)
agg_pack_kernel(const float* __restrict__ w_xy, const float* __restrict__ w_x, const float* __restrict__ w_y, int dx,
                int dy, int hx, int hy, int n_aug, float* __restrict__ W_aug, float* __restrict__ bias_aug) {
  b2_pdl_wait();
  const int64_t n = (int64_t) n_aug * dx;
  for (int64_t t = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; t < n + n_aug; t += (int64_t) gridDim.x * blockDim.x) {
    if (t >= n) {
      const int r = (int) (t - n);
      bias_aug[r] = r < dy ? __ldg(w_y + r) : 0.f;
      continue;
    }
    const int r = (int) (t / dx), c = (int) (t % dx);
    float v = 0.f;
    if (r < dy) {
      if (c / hx == r / hy) v = __ldg(w_xy + (int64_t) c * hy + r % hy);    // W_h[c - h hx, r - h hy]
    } else if (r == dy) {
      v = __ldg(w_x + c);
    }
    W_aug[t] = v;
  }
  b2_pdl_trigger();
}

// gw_xy = the diagonal blocks of dW_aug, gw_x = its row dy  ("=")
__global__ void __launch_bounds__(256)
agg_unpack_kernel(const float* __restrict__ dW, int dx, int dy, int hx, int hy, float* __restrict__ gw_xy,
                  float* __restrict__ gw_x) {
  b2_pdl_wait();
  const int64_t n = (int64_t) dx * hy;
  for (int64_t t = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; t < n + dx; t += (int64_t) gridDim.x * blockDim.x) {
    if (t >= n) {
      const int c = (int) (t - n);
      gw_x[c] = __ldg(dW + (int64_t) dy * dx + c);
      continue;
    }
    const int c = (int) (t / hy), j = (int) (t % hy);     // w_xy[c hy + j] = W_h[c - h hx, j], h = c / hx
    gw_xy[t] = __ldg(dW + (int64_t) ((c / hx) * hy + j) * dx + c);
  }
  b2_pdl_trigger();
}

// out_b = sum_{j < dy} y_bj Q_bj + Q_b,dy + b_x + b_y: one warp per row
template <int VW>
__global__ void __launch_bounds__(256)
agg_fwd_kernel(const float* __restrict__ Q, const float* __restrict__ y, const float* __restrict__ bx,
               const float* __restrict__ by, int64_t batch, int dy, int n_aug, float* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const int64_t warps = (int64_t) gridDim.x * (blockDim.x >> 5);
  b2_pdl_wait();
  const float bias = __ldg(bx) + __ldg(by);
  for (int64_t row = (int64_t) blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); row < batch; row += warps) {
    const float* q = Q + row * n_aug;
    const float* yr = y + row * dy;
    float s = 0.f;
    for (int c = lane * VW; c < dy; c += 32 * VW) {
      float a[VW], b[VW];
      rk_load<VW>(yr + c, a);
      rk_load<VW>(q + c, b);
#pragma unroll
      for (int k = 0; k < VW; ++k) s = fmaf(a[k], b[k], s);
    }
    s = b2_warp_sum(s);
    if (lane == 0) out[row] = s + __ldg(q + dy) + bias;
  }
  b2_pdl_trigger();
}

// dy = g Q[:, :dy]; ys = [g y | g | 0] (+ its GEMM-operand copy); gw_y += sum_rows g y, gb_x, gb_y += sum_rows g
template <int VW>
__global__ void __launch_bounds__(RK_THREADS)
agg_bwd_kernel(const float* __restrict__ Q, const float* __restrict__ y, const float* __restrict__ g, int64_t batch,
               int dy, int n_aug, int tx_n, float* __restrict__ gy, float* __restrict__ ys, void* ys_aux,
               int aux_dtype, int64_t ld_aux, float* __restrict__ gw_y, float* __restrict__ gb_x,
               float* __restrict__ gb_y) {
  __shared__ float red[RK_THREADS * VW];
  const int tx = threadIdx.x % tx_n, ty = threadIdx.x / tx_n, ty_n = blockDim.x / tx_n;
  const int c = (blockIdx.y * tx_n + tx) * VW;
  float acc[VW];
#pragma unroll
  for (int k = 0; k < VW; ++k) acc[k] = 0.f;
  b2_pdl_wait();
  if (c < n_aug) {
    for (int64_t row = (int64_t) blockIdx.x * ty_n + ty; row < batch; row += (int64_t) gridDim.x * ty_n) {
      const float gr = __ldg(g + row);
      float s[VW];
      if (c < dy) {       // VW divides dy: a slot lies wholly left of column dy or wholly right of it
        float a[VW], q[VW];
        rk_load<VW>(y + row * dy + c, a);
        rk_load<VW>(Q + row * n_aug + c, q);
#pragma unroll
        for (int k = 0; k < VW; ++k) {
          s[k] = gr * a[k];
          q[k] = gr * q[k];
        }
        rk_store<VW>(gy + row * dy + c, q);
      } else {
#pragma unroll
        for (int k = 0; k < VW; ++k) s[k] = c + k == dy ? gr : 0.f;
      }
      rk_store<VW>(ys + row * n_aug + c, s);
      if (ys_aux) rk_store_aux<VW>(ys_aux, aux_dtype, row * ld_aux + c, s);
#pragma unroll
      for (int k = 0; k < VW; ++k) acc[k] += s[k];
    }
  }
  b2_pdl_trigger();
  rk_cta_colsum<VW>(red, tx, tx_n, ty_n, acc);
  if (ty == 0 && c < n_aug) {
#pragma unroll
    for (int k = 0; k < VW; ++k) {
      if (acc[k] == 0.f) continue;
      if (c + k < dy) {
        b2_red_add(gw_y + c + k, acc[k]);
      } else if (c + k == dy) {
        b2_red_add(gb_x, acc[k]);
        b2_red_add(gb_y, acc[k]);
      }
    }
  }
}

// ---------------------------------------------------------------------------------
// Host side
// ---------------------------------------------------------------------------------
static int fm_check(int64_t batch, int d) {
  B2_REQUIRE(d >= 1, "width d = %d < 1", d);
  B2_REQUIRE(batch >= 0, "negative batch");
  B2_REQUIRE(batch * (int64_t) d < ((int64_t) 1 << 31), "batch * d = %lld >= 2^31", (long long) (batch * (int64_t) d));
  return B2_OK;
}

static int agg_check(int64_t batch, int dx, int dy, int heads) {
  B2_REQUIRE(dx >= 1 && dy >= 1, "widths dx = %d, dy = %d must be >= 1", dx, dy);
  B2_REQUIRE(heads >= 1 && dx % heads == 0 && dy % heads == 0, "num_heads = %d must divide dx = %d and dy = %d",
             heads, dx, dy);
  if (int rc = fm_check(batch, dx)) return rc;
  return fm_check(batch, B2_AGG_COLS(dy));
}

static int fs_launch_blocks(int64_t n) {
  const int64_t blocks = b2_ceil_div(n, 256), cap = (int64_t) B2_NUM_SMS * 8;
  return (int) (blocks < 1 ? 1 : (blocks > cap ? cap : blocks));
}

extern "C" B2_API int b2_fs_gate_fwd(const float* e, const float* g1, const float* g2, int per_row1, int per_row2,
                                     int64_t batch, int d, float* f1, float* f2, void* f1_aux, void* f2_aux,
                                     int aux_dtype, int64_t ld_aux, void* stream) {
  B2_REQUIRE(e && g1 && g2 && f1 && f2, "NULL pointer");
  B2_REQUIRE((f1_aux == nullptr) == (f2_aux == nullptr), "f1_aux and f2_aux: both or neither");
  if (int rc = fm_check(batch, d)) return rc;
  if (int rc = rk_check_aux(f1_aux, aux_dtype, ld_aux, d)) return rc;
  if (batch == 0) return B2_OK;
  const int64_t ldg1 = per_row1 ? d : 0, ldg2 = per_row2 ? d : 0;
  const void* ptrs[] = {e, g1, g2, f1, f2};
  if (rk_vec(d, ptrs, 5, f1_aux, aux_dtype, ld_aux) && rk_vec(d, ptrs, 0, f2_aux, aux_dtype, ld_aux)) {
    const rk_grid p = rk_plan(batch, d, 4, 8);
    B2_LAUNCH(fs_gate_fwd_kernel<4>, p.grid, p.threads, 0, (cudaStream_t) stream, e, g1, g2, ldg1, ldg2, batch, d,
              p.tx_n, f1, f2, f1_aux, f2_aux, aux_dtype, ld_aux);
  } else {
    const rk_grid p = rk_plan(batch, d, 1, 8);
    B2_LAUNCH(fs_gate_fwd_kernel<1>, p.grid, p.threads, 0, (cudaStream_t) stream, e, g1, g2, ldg1, ldg2, batch, d,
              p.tx_n, f1, f2, f1_aux, f2_aux, aux_dtype, ld_aux);
  }
  B2_CUDA_LAUNCH_CHECK("b2_fs_gate_fwd");
  return B2_OK;
}

extern "C" B2_API int b2_fs_gate_bwd(const float* e, const float* g1, const float* g2, int per_row1, int per_row2,
                                     const float* df1, const float* df2, int64_t batch, int d, float* de, float* dg1,
                                     float* dg2, void* stream) {
  B2_REQUIRE(e && g1 && g2 && df1 && df2 && de && dg1 && dg2, "NULL pointer");
  if (int rc = fm_check(batch, d)) return rc;
  if (batch == 0) return B2_OK;
  const int64_t ldg1 = per_row1 ? d : 0, ldg2 = per_row2 ? d : 0;
  const void* ptrs[] = {e, g1, g2, df1, df2, de, dg1, dg2};
  if (rk_vec(d, ptrs, 8, nullptr, 0, 0)) {
    const rk_grid p = rk_plan(batch, d, 4, 4);
    B2_LAUNCH(fs_gate_bwd_kernel<4>, p.grid, p.threads, 0, (cudaStream_t) stream, e, g1, g2, ldg1, ldg2, df1, df2,
              batch, d, p.tx_n, de, dg1, dg2);
  } else {
    const rk_grid p = rk_plan(batch, d, 1, 4);
    B2_LAUNCH(fs_gate_bwd_kernel<1>, p.grid, p.threads, 0, (cudaStream_t) stream, e, g1, g2, ldg1, ldg2, df1, df2,
              batch, d, p.tx_n, de, dg1, dg2);
  }
  B2_CUDA_LAUNCH_CHECK("b2_fs_gate_bwd");
  return B2_OK;
}

extern "C" B2_API int b2_agg_pack(const float* w_xy, const float* w_x, const float* w_y, int dx, int dy, int heads,
                                  float* W_aug, float* bias_aug, void* stream) {
  B2_REQUIRE(w_xy && w_x && w_y && W_aug && bias_aug, "NULL pointer");
  if (int rc = agg_check(0, dx, dy, heads)) return rc;
  const int n_aug = B2_AGG_COLS(dy);
  B2_REQUIRE((int64_t) n_aug * dx < ((int64_t) 1 << 31), "W_aug (%d, %d) has 2^31 elements or more", n_aug, dx);
  B2_LAUNCH(agg_pack_kernel, fs_launch_blocks((int64_t) n_aug * dx + n_aug), 256, 0, (cudaStream_t) stream, w_xy, w_x,
            w_y, dx, dy, dx / heads, dy / heads, n_aug, W_aug, bias_aug);
  B2_CUDA_LAUNCH_CHECK("b2_agg_pack");
  return B2_OK;
}

extern "C" B2_API int b2_agg_fwd(const float* Q, const float* y, const float* b_x, const float* b_y, int64_t batch,
                                 int dy, float* out, void* stream) {
  B2_REQUIRE(Q && y && b_x && b_y && out, "NULL pointer");
  if (int rc = agg_check(batch, 1, dy, 1)) return rc;
  if (batch == 0) return B2_OK;
  const int64_t blocks = b2_ceil_div(batch, 8), cap = (int64_t) B2_NUM_SMS * 8;
  const int grid = (int) (blocks > cap ? cap : blocks);
  if (dy % 4 == 0 && rk_al16(Q) && rk_al16(y)) {
    B2_LAUNCH(agg_fwd_kernel<4>, grid, 256, 0, (cudaStream_t) stream, Q, y, b_x, b_y, batch, dy, B2_AGG_COLS(dy), out);
  } else {
    B2_LAUNCH(agg_fwd_kernel<1>, grid, 256, 0, (cudaStream_t) stream, Q, y, b_x, b_y, batch, dy, B2_AGG_COLS(dy), out);
  }
  B2_CUDA_LAUNCH_CHECK("b2_agg_fwd");
  return B2_OK;
}

extern "C" B2_API int b2_agg_bwd(const float* Q, const float* y, const float* g, int64_t batch, int dy, float* gy,
                                 float* ys, void* ys_aux, int aux_dtype, int64_t ld_aux, float* gw_y, float* gb_x,
                                 float* gb_y, void* stream) {
  B2_REQUIRE(Q && y && g && gy && ys && gw_y && gb_x && gb_y, "NULL pointer");
  if (int rc = agg_check(batch, 1, dy, 1)) return rc;
  const int n_aug = B2_AGG_COLS(dy);
  if (int rc = rk_check_aux(ys_aux, aux_dtype, ld_aux, n_aug)) return rc;
  if (batch == 0) return B2_OK;
  const void* ptrs[] = {Q, y, gy, ys};
  if (rk_vec(dy, ptrs, 4, ys_aux, aux_dtype, ld_aux)) {
    const rk_grid p = rk_plan(batch, n_aug, 4, 4);
    B2_LAUNCH(agg_bwd_kernel<4>, p.grid, p.threads, 0, (cudaStream_t) stream, Q, y, g, batch, dy, n_aug, p.tx_n, gy,
              ys, ys_aux, aux_dtype, ld_aux, gw_y, gb_x, gb_y);
  } else {
    const rk_grid p = rk_plan(batch, n_aug, 1, 4);
    B2_LAUNCH(agg_bwd_kernel<1>, p.grid, p.threads, 0, (cudaStream_t) stream, Q, y, g, batch, dy, n_aug, p.tx_n, gy,
              ys, ys_aux, aux_dtype, ld_aux, gw_y, gb_x, gb_y);
  }
  B2_CUDA_LAUNCH_CHECK("b2_agg_bwd");
  return B2_OK;
}

extern "C" B2_API int b2_agg_unpack(const float* dW_aug, int dx, int dy, int heads, float* gw_xy, float* gw_x,
                                    void* stream) {
  B2_REQUIRE(dW_aug && gw_xy && gw_x, "NULL pointer");
  if (int rc = agg_check(0, dx, dy, heads)) return rc;
  B2_LAUNCH(agg_unpack_kernel, fs_launch_blocks((int64_t) dx * (dy / heads) + dx), 256, 0, (cudaStream_t) stream,
            dW_aug, dx, dy, dx / heads, dy / heads, gw_xy, gw_x);
  B2_CUDA_LAUNCH_CHECK("b2_agg_unpack");
  return B2_OK;
}

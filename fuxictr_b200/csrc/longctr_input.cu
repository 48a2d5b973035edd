// longctr_input.cu — the LongCTR input triple (model_zoo/LongCTR/longctr_dataloader.py, BatchCollator) built on the
// device from an HBM-resident store, sm_90a.
//
// Per sample b (one row of the batch matrix): u = user_index, t = item_index, n = min(seq_len, len(history of u)).
// The collator pads full_seq[u][:seq_len] with keras pad_sequences(maxlen = L, value = 0, padding = truncating = p):
// the k = min(n, L) kept items are the last k of the n (p = "pre", right-aligned) or the first k (p = "post",
// left-aligned).  Slot L is t.  Every item column c holds item_info row id (positional: padding slots copy row 0),
// and mask = id > 0 by value.  One CTA column per sample, threads over the L + 1 slots: every store is coalesced, the
// three batch values of a row are one broadcast load per warp, and the history is read in slot order.
#include "b2_common.cuh"

#define LONGCTR_THREADS 256

template <typename T>
__global__ void __launch_bounds__(LONGCTR_THREADS)
longctr_collate_kernel(const T* __restrict__ batch, int64_t row_stride, int col_user, int col_item, int col_seq_len,
                       const int64_t* __restrict__ offsets, const int32_t* __restrict__ hist,
                       const int32_t* __restrict__ item_info, int C, int64_t rows, int L, int post,
                       float* __restrict__ mask, int64_t* __restrict__ items) {
  b2_pdl_wait();
  const int l = blockIdx.y * blockDim.x + threadIdx.x;
  if (l > L) return;
  const int64_t b = blockIdx.x;
  const T* row = batch + b * row_stride;
  int64_t id;
  if (l == L) {
    id = (int64_t) row[col_item];
  } else {
    const int64_t u = (int64_t) row[col_user];
    const int64_t o = offsets[u];
    const int64_t n = min((int64_t) row[col_seq_len], offsets[u + 1] - o);
    const int k = (int) min(n, (int64_t) L);
    const int s = post ? l : l - (L - k);        // position among the k kept items
    id = (s >= 0 && s < k) ? (int64_t) hist[o + (post ? 0 : n - k) + s] : 0;
    mask[b * L + l] = id > 0 ? 1.f : 0.f;
  }
  const int32_t* r = item_info + id * C;
  const int64_t plane = rows * (int64_t) (L + 1);
  int64_t* out = items + b * (L + 1) + l;
  for (int c = 0; c < C; ++c) out[c * plane] = (int64_t) r[c];
}

extern "C" B2_API int b2_longctr_collate(const void* batch, int batch_dtype, int64_t rows, int64_t row_stride,
                                        int col_user, int col_item, int col_seq_len, const int64_t* offsets,
                                        const int32_t* hist, int64_t num_users, const int32_t* item_info,
                                        int64_t num_items, int num_cols, int L, int padding, float* mask,
                                        int64_t* items, void* stream) {
  B2_REQUIRE(batch && offsets && hist && item_info && items && (mask || L == 0), "NULL pointer");
  B2_REQUIRE(batch_dtype == B2_I64 || batch_dtype == B2_I32,
             "LongCTR collate: the batch matrix must be int64 or int32 (dtype code %d)", batch_dtype);
  B2_REQUIRE(padding == B2_LONGCTR_PAD_PRE || padding == B2_LONGCTR_PAD_POST,
             "LongCTR collate: padding must be B2_LONGCTR_PAD_PRE or B2_LONGCTR_PAD_POST, got %d", padding);
  B2_REQUIRE(rows >= 0 && rows < ((int64_t) 1 << 31), "LongCTR collate: %lld rows outside [0, 2^31)",
             (long long) rows);
  B2_REQUIRE(L >= 0 && L <= B2_LONGCTR_MAX_LEN, "LongCTR collate: L = %d outside [0, %d]", L, B2_LONGCTR_MAX_LEN);
  B2_REQUIRE(num_cols >= 1 && num_cols <= B2_LONGCTR_MAX_COLS, "LongCTR collate: %d item columns outside [1, %d]",
             num_cols, B2_LONGCTR_MAX_COLS);
  B2_REQUIRE(row_stride >= 1 && col_user >= 0 && col_item >= 0 && col_seq_len >= 0 && col_user < row_stride &&
                 col_item < row_stride && col_seq_len < row_stride,
             "LongCTR collate: columns (%d, %d, %d) outside a row of stride %lld", col_user, col_item, col_seq_len,
             (long long) row_stride);
  B2_REQUIRE(num_users >= 1 && num_items >= 1, "LongCTR collate: empty store (%lld users, %lld items)",
             (long long) num_users, (long long) num_items);
  if (rows == 0) return B2_OK;
  const int threads = (int) std::min<int64_t>(b2_ceil_div(L + 1, 32) * 32, LONGCTR_THREADS);
  const dim3 grid((unsigned) rows, (unsigned) b2_ceil_div(L + 1, threads));
  const int post = padding == B2_LONGCTR_PAD_POST;
  cudaStream_t st = (cudaStream_t) stream;
  if (batch_dtype == B2_I64)
    B2_LAUNCH(longctr_collate_kernel<int64_t>, grid, threads, 0, st, (const int64_t*) batch, row_stride, col_user,
              col_item, col_seq_len, offsets, hist, item_info, num_cols, rows, L, post, mask, items);
  else
    B2_LAUNCH(longctr_collate_kernel<int32_t>, grid, threads, 0, st, (const int32_t*) batch, row_stride, col_user,
              col_item, col_seq_len, offsets, hist, item_info, num_cols, rows, L, post, mask, items);
  B2_CUDA_LAUNCH_CHECK("b2_longctr_collate");
  return B2_OK;
}

// metrics.cu — device-resident evaluation metrics (SURVEY.md 8f row 3), sm_90a.
//
// BaseModel.evaluate (fuxictr/pytorch/models/rank_model.py:350-381) copies y_pred / y_true to the
// host after EVERY batch, grows Python lists, and hands float64 arrays to sklearn's log_loss and
// roc_auc_score (fuxictr/metrics.py:45-48).  Here predictions stay in HBM; at the end of the epoch
//   b2_logloss_sum : sum_i -[y log p + (1-y) log(1-p)]  in fp64 with sklearn's clip to [eps, 1-eps]
//   b2_auc         : the EXACT tie-aware Mann-Whitney statistic in integers — partition the scores
//                    into negatives / positives as order-preserving u32 keys, LSD radix sort of the
//                    negatives (4 x 8-bit digits, stable), then per positive lower+upper bound
// and one 40-byte D2H returns {n_neg, n_pos, n_nan, n_badlabel, 2U}; AUC = 2U / (2 n_pos n_neg).
// All three are HBM/L2-bound integer work (keys are 4 B; the sorted negatives of a Criteo-size
// validation split, ~14 MB, stay L2-resident for the searches).
#include "b2_common.cuh"

namespace {
constexpr int RS_THREADS = 256;               // one chunk = 256 keys
constexpr int RS_WARPS = RS_THREADS / 32;
constexpr int RS_MAX_BLOCKS = B2_NUM_SMS * 4;
constexpr int RS_DIGITS = 256;

// order-preserving map float -> u32 (ascending); -0.0 and +0.0 tie as they do for sklearn
__device__ __forceinline__ uint32_t score_key(float s) {
  uint32_t u = (s == 0.f) ? 0u : __float_as_uint(s);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

__device__ __forceinline__ unsigned long long warp_sum_u64(unsigned long long v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double warp_sum_f64(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// ---- log loss ----------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
logloss_kernel(const float* __restrict__ y_pred, const float* __restrict__ y_true, int64_t n,
               double* __restrict__ sum) {
  __shared__ double red[8];
  const double eps = 2.220446049250313e-16;   // np.finfo(np.float64).eps: evaluate() widens to float64
  double acc = 0.0;
  for (int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t) gridDim.x * blockDim.x) {
    const double p = (double) y_pred[i];
    const double y = (double) y_true[i];
    // sklearn: y_prob = [1-p, p], clipped column-wise; loss = -(xlogy(1-y, .) + xlogy(y, .))
    const double p1 = fmin(fmax(p, eps), 1.0 - eps);
    const double p0 = fmin(fmax(1.0 - p, eps), 1.0 - eps);
    if (y != 0.0) acc -= y * log(p1);
    if (y != 1.0) acc -= (1.0 - y) * log(p0);
  }
  acc = warp_sum_f64(acc);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x < 32) {
    double t = threadIdx.x < 8 ? red[threadIdx.x] : 0.0;
    t = warp_sum_f64(t);
    if (threadIdx.x == 0 && t != 0.0) atomicAdd(sum, t);
  }
}

// ---- partition into negative / positive key lists ----------------------------------------------
// res[0] = n_neg, res[1] = n_pos, res[2] = n_nan, res[3] = n_badlabel.  Negatives fill keys[0..),
// positives fill keys[n-1 ..) downwards.  Order inside a list is irrelevant.
__global__ void __launch_bounds__(256)
auc_partition_kernel(const float* __restrict__ y_pred, const float* __restrict__ y_true, int64_t n,
                     uint32_t* __restrict__ keys, unsigned long long* __restrict__ res) {
  const int lane = threadIdx.x & 31;
  const unsigned lt = (1u << lane) - 1u;
  for (int64_t base = (int64_t) blockIdx.x * blockDim.x; base < n; base += (int64_t) gridDim.x * blockDim.x) {
    const int64_t i = base + threadIdx.x;      // trip count is uniform across the block
    const bool on = i < n;
    const float s = on ? y_pred[i] : 0.f;
    const float y = on ? y_true[i] : 0.f;
    const bool pos = on && y == 1.f;
    const bool neg = on && y == 0.f;
    const unsigned mp = __ballot_sync(0xffffffffu, pos);
    const unsigned mn = __ballot_sync(0xffffffffu, neg);
    const unsigned mnan = __ballot_sync(0xffffffffu, on && s != s);
    const unsigned mbad = __ballot_sync(0xffffffffu, on && !pos && !neg);
    unsigned long long bn = 0, bp = 0;
    if (lane == 0) {
      if (mn) bn = atomicAdd(&res[0], (unsigned long long) __popc(mn));
      if (mp) bp = atomicAdd(&res[1], (unsigned long long) __popc(mp));
      if (mnan) atomicAdd(&res[2], (unsigned long long) __popc(mnan));
      if (mbad) atomicAdd(&res[3], (unsigned long long) __popc(mbad));
    }
    bn = __shfl_sync(0xffffffffu, bn, 0);
    bp = __shfl_sync(0xffffffffu, bp, 0);
    const uint32_t key = score_key(s);
    if (neg) keys[bn + __popc(mn & lt)] = key;
    if (pos) keys[n - 1 - (int64_t) (bp + __popc(mp & lt))] = key;
  }
}

// ---- stable LSD radix sort of keys[0, *count) --------------------------------------------------
__device__ __forceinline__ int64_t rs_per_block(int64_t n, int nblocks) {
  const int64_t t = (n + nblocks - 1) / nblocks;
  return (t + RS_THREADS - 1) / RS_THREADS * RS_THREADS;
}

__global__ void set_count_kernel(unsigned long long* count, unsigned long long n) { *count = n; }

// counts[digit * gridDim.x + block] = number of keys of this block's tile with that digit
__global__ void __launch_bounds__(RS_THREADS)
rs_hist_kernel(const uint32_t* __restrict__ keys, const unsigned long long* __restrict__ count, int shift,
               uint32_t* __restrict__ counts) {
  __shared__ uint32_t h[RS_DIGITS];
  h[threadIdx.x] = 0;
  __syncthreads();
  const int64_t n = (int64_t) *count;
  const int64_t per = rs_per_block(n, gridDim.x);
  const int64_t lo = (int64_t) blockIdx.x * per;
  const int64_t hi = min(lo + per, n);
  const int lane = threadIdx.x & 31;
  for (int64_t c = lo; c < hi; c += RS_THREADS) {   // uniform across the block
    const int64_t i = c + threadIdx.x;
    const bool on = i < hi;
    const uint32_t d = on ? ((keys[i] >> shift) & 255u) : 0xffffffffu;
    const unsigned peers = __match_any_sync(0xffffffffu, d);
    if (on && (peers & ((1u << lane) - 1u)) == 0) atomicAdd(&h[d], (uint32_t) __popc(peers));
  }
  __syncthreads();
  counts[(int64_t) threadIdx.x * gridDim.x + blockIdx.x] = h[threadIdx.x];
}

// in-place exclusive prefix sum over `len` u32 entries, one block of 1024 threads
__global__ void __launch_bounds__(1024)
rs_scan_kernel(uint32_t* __restrict__ counts, int len) {
  __shared__ uint32_t part[1024];
  const int per = (len + 1023) / 1024;
  const int lo = min(threadIdx.x * per, len), hi = min(lo + per, len);
  uint32_t s = 0;
  for (int i = lo; i < hi; ++i) s += counts[i];
  part[threadIdx.x] = s;
  __syncthreads();
  for (int off = 1; off < 1024; off <<= 1) {      // Hillis-Steele inclusive scan
    const uint32_t add = threadIdx.x >= off ? part[threadIdx.x - off] : 0u;
    __syncthreads();
    part[threadIdx.x] += add;
    __syncthreads();
  }
  uint32_t run = part[threadIdx.x] - s;            // exclusive prefix of this thread's segment
  for (int i = lo; i < hi; ++i) {
    const uint32_t c = counts[i];
    counts[i] = run;
    run += c;
  }
}

// offsets = exclusive scan of the histogram (digit-major, then block): keys keep their order inside
// a digit => stable
__global__ void __launch_bounds__(RS_THREADS)
rs_scatter_kernel(const uint32_t* __restrict__ in, uint32_t* __restrict__ out,
                  const unsigned long long* __restrict__ count, int shift, const uint32_t* __restrict__ offsets) {
  __shared__ uint32_t next[RS_DIGITS];               // next output slot of each digit for this block
  __shared__ uint32_t whist[RS_WARPS][RS_DIGITS];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  next[threadIdx.x] = offsets[(int64_t) threadIdx.x * gridDim.x + blockIdx.x];
  const int64_t n = (int64_t) *count;
  const int64_t per = rs_per_block(n, gridDim.x);
  const int64_t lo = (int64_t) blockIdx.x * per;
  const int64_t hi = min(lo + per, n);
  for (int64_t c = lo; c < hi; c += RS_THREADS) {    // uniform across the block
#pragma unroll
    for (int w = 0; w < RS_WARPS; ++w) whist[w][threadIdx.x] = 0;
    __syncthreads();
    const int64_t i = c + threadIdx.x;
    const bool on = i < hi;
    const uint32_t key = on ? in[i] : 0u;
    const uint32_t d = on ? ((key >> shift) & 255u) : 0xffffffffu;
    const unsigned peers = __match_any_sync(0xffffffffu, d);
    const int rank = __popc(peers & ((1u << lane) - 1u));
    if (on && rank == 0) whist[warp][d] = (uint32_t) __popc(peers);
    __syncthreads();
    {
      uint32_t run = next[threadIdx.x];              // thread t owns digit t
#pragma unroll
      for (int w = 0; w < RS_WARPS; ++w) {
        const uint32_t cnt = whist[w][threadIdx.x];
        whist[w][threadIdx.x] = run;
        run += cnt;
      }
      next[threadIdx.x] = run;
    }
    __syncthreads();
    if (on) out[whist[warp][d] + rank] = key;
    __syncthreads();
  }
}

// ---- Mann-Whitney numerator -----------------------------------------------------------------------
// res[4] += sum over positives of (#neg < s) + (#neg <= s)   == 2 * [#(neg<pos) + 0.5 #(neg==pos)]
__global__ void __launch_bounds__(256)
auc_count_kernel(const uint32_t* __restrict__ keys, int64_t n, unsigned long long* __restrict__ res) {
  __shared__ unsigned long long red[8];
  const int64_t nneg = (int64_t) res[0], npos = (int64_t) res[1];
  unsigned long long acc = 0;
  for (int64_t j = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; j < npos; j += (int64_t) gridDim.x * blockDim.x) {
    const uint32_t k = keys[n - 1 - j];
    int64_t lo = 0, hi = nneg;                    // lower bound: first index with key >= k
    while (lo < hi) {
      const int64_t mid = (lo + hi) >> 1;
      if (keys[mid] < k) lo = mid + 1; else hi = mid;
    }
    const int64_t lb = lo;
    hi = nneg;                                    // upper bound: first index with key > k (>= lb)
    while (lo < hi) {
      const int64_t mid = (lo + hi) >> 1;
      if (keys[mid] <= k) lo = mid + 1; else hi = mid;
    }
    acc += (unsigned long long) (lb + lo);
  }
  acc = warp_sum_u64(acc);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x < 32) {
    unsigned long long t = threadIdx.x < 8 ? red[threadIdx.x] : 0ull;
    t = warp_sum_u64(t);
    if (threadIdx.x == 0 && t != 0ull) atomicAdd(&res[4], t);
  }
}

int sort_blocks(int64_t n) {
  int64_t b = b2_ceil_div(n, (int64_t) RS_THREADS * 8);
  if (b > RS_MAX_BLOCKS) b = RS_MAX_BLOCKS;
  return (int) (b < 1 ? 1 : b);
}
int stream_grid(int64_t n) {
  int64_t b = b2_ceil_div(n, 256);
  if (b > (int64_t) B2_NUM_SMS * 8) b = (int64_t) B2_NUM_SMS * 8;
  return (int) (b < 1 ? 1 : b);
}

// sorts a[0, *count); tmp is the ping-pong buffer; 4 passes end in `a`
int radix_sort(uint32_t* a, uint32_t* tmp, int64_t n_max, const unsigned long long* count, uint32_t* counts,
               cudaStream_t st) {
  const int g = sort_blocks(n_max);
  uint32_t* src = a;
  uint32_t* dst = tmp;
  for (int shift = 0; shift < 32; shift += 8) {
    rs_hist_kernel<<<g, RS_THREADS, 0, st>>>(src, count, shift, counts);
    rs_scan_kernel<<<1, 1024, 0, st>>>(counts, RS_DIGITS * g);
    rs_scatter_kernel<<<g, RS_THREADS, 0, st>>>(src, dst, count, shift, counts);
    uint32_t* t = src; src = dst; dst = t;
  }
  B2_CUDA_LAUNCH_CHECK("radix_sort");
  return B2_OK;
}

// workspace layout (bytes): [keys n*4][tmp n*4][counts 256*G*4][count 8], each 256-byte aligned
struct AucWs { size_t keys, tmp, counts, count, total; };
AucWs auc_layout(int64_t n) {
  auto up = [](size_t x) { return (x + 255) / 256 * 256; };
  AucWs w;
  w.keys = 0;
  w.tmp = up((size_t) n * 4);
  w.counts = w.tmp + up((size_t) n * 4);
  w.count = w.counts + up((size_t) RS_DIGITS * sort_blocks(n) * 4);
  w.total = w.count + 256;
  return w;
}
}  // namespace

extern "C" B2_API int b2_logloss_sum(const float* y_pred, const float* y_true, int64_t n, double* sum, void* stream) {
  B2_REQUIRE(n >= 0, "negative n");
  if (n == 0) return B2_OK;
  B2_REQUIRE(y_pred && y_true && sum, "NULL argument");
  logloss_kernel<<<stream_grid(n), 256, 0, (cudaStream_t) stream>>>(y_pred, y_true, n, sum);
  B2_CUDA_LAUNCH_CHECK("b2_logloss_sum");
  return B2_OK;
}

extern "C" B2_API int b2_auc_workspace_bytes(int64_t n, int64_t* bytes) {
  B2_REQUIRE(bytes != nullptr, "NULL argument");
  B2_REQUIRE(n >= 1 && n < ((int64_t) 1 << 31), "n=%lld outside [1, 2^31)", (long long) n);
  *bytes = (int64_t) auc_layout(n).total;
  return B2_OK;
}

extern "C" B2_API int b2_sort_u32(uint32_t* keys, int64_t n, void* workspace, int64_t workspace_bytes, void* stream) {
  B2_REQUIRE(n >= 0 && n < ((int64_t) 1 << 31), "n=%lld outside [0, 2^31)", (long long) n);
  if (n == 0) return B2_OK;
  B2_REQUIRE(keys && workspace, "NULL argument");
  const AucWs w = auc_layout(n);
  B2_REQUIRE(workspace_bytes >= (int64_t) w.total, "workspace of %lld bytes < %lld needed (b2_auc_workspace_bytes)",
             (long long) workspace_bytes, (long long) w.total);
  B2_REQUIRE((reinterpret_cast<uintptr_t>(workspace) & 255) == 0, "workspace must be 256-byte aligned");
  char* ws = static_cast<char*>(workspace);
  cudaStream_t st = (cudaStream_t) stream;
  unsigned long long* count = reinterpret_cast<unsigned long long*>(ws + w.count);
  set_count_kernel<<<1, 1, 0, st>>>(count, (unsigned long long) n);
  return radix_sort(keys, reinterpret_cast<uint32_t*>(ws + w.tmp), n, count, reinterpret_cast<uint32_t*>(ws + w.counts), st);
}

extern "C" B2_API int b2_auc(const float* y_pred, const float* y_true, int64_t n, void* workspace,
                             int64_t workspace_bytes, uint64_t* result, void* stream) {
  B2_REQUIRE(n >= 1 && n < ((int64_t) 1 << 31), "n=%lld outside [1, 2^31)", (long long) n);
  B2_REQUIRE(y_pred && y_true && workspace && result, "NULL argument");
  const AucWs w = auc_layout(n);
  B2_REQUIRE(workspace_bytes >= (int64_t) w.total, "workspace of %lld bytes < %lld needed (b2_auc_workspace_bytes)",
             (long long) workspace_bytes, (long long) w.total);
  B2_REQUIRE((reinterpret_cast<uintptr_t>(workspace) & 255) == 0, "workspace must be 256-byte aligned");
  B2_REQUIRE((reinterpret_cast<uintptr_t>(result) & 7) == 0, "result must be 8-byte aligned");
  char* ws = static_cast<char*>(workspace);
  cudaStream_t st = (cudaStream_t) stream;
  uint32_t* keys = reinterpret_cast<uint32_t*>(ws + w.keys);
  unsigned long long* res = reinterpret_cast<unsigned long long*>(result);
  if (cudaMemsetAsync(res, 0, 5 * sizeof(unsigned long long), st) != cudaSuccess)
    return b2_fail(B2_E_CUDA, "b2_auc: memset failed: %s", cudaGetErrorString(cudaGetLastError()));
  auc_partition_kernel<<<stream_grid(n), 256, 0, st>>>(y_pred, y_true, n, keys, res);
  B2_CUDA_LAUNCH_CHECK("b2_auc partition");
  int rc = radix_sort(keys, reinterpret_cast<uint32_t*>(ws + w.tmp), n, res /* res[0] = n_neg */,
                      reinterpret_cast<uint32_t*>(ws + w.counts), st);
  if (rc != B2_OK) return rc;
  auc_count_kernel<<<stream_grid(n), 256, 0, st>>>(keys, n, res);
  B2_CUDA_LAUNCH_CHECK("b2_auc count");
  return B2_OK;
}

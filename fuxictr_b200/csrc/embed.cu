// embed.cu — fused multi-field embedding gather / scatter-add and the D=1
// LogisticRegression gather-reduce, sm_90a.
//
// Reference semantics (reczoo/FuxiCTR v2.3.10):
//   FeatureEmbeddingDict.forward   fuxictr/pytorch/layers/embeddings/feature_embedding.py:261-297
//   FeatureEmbeddingDict.dict2tensor                                  feature_embedding.py:230-259
//   MaskedAveragePooling / MaskedSumPooling        fuxictr/pytorch/layers/pooling.py:33-49, 62-73
//   LogisticRegression.forward      fuxictr/pytorch/layers/blocks/logistic_regression.py:46-59
//
// HBM-bound integer/byte work: no tensor cores.  A work item is one table row
// (one (sample, field[, position]) triple); LPR = 2^k lanes own one row and move
// it with 16-byte accesses, so a warp reads 32/LPR independent rows per
// instruction and writes a contiguous span of the stacked/concatenated output.
// Field descriptors travel as a __grid_constant__ launch parameter (no H2D
// copy, CUDA-graph friendly) and are staged once per CTA in shared memory.
#include "embed_common.cuh"
#include <stdlib.h>

// ---------------------------------------------------------------------------------
// Forward, fast path: no pooled field, every row fits one pass of its LPR lanes.
// ---------------------------------------------------------------------------------
template <int VEC>
__device__ __forceinline__ typename VecT<VEC>::type b2_ld_row(const typename VecT<VEC>::type* p, int mode) {
  return __ldg(p);
}
// mode 0: plain read-only load; 1: L1::no_allocate (one-touch); 2: read-only load with the L2::64B
// prefetch-size hint — a D=16 row is exactly one 64-byte sector pair.  Not the default (its gain on the
// H100 is not measured), kept selectable through B2_GATHER_STREAM=2.
template <>
__device__ __forceinline__ float4 b2_ld_row<4>(const float4* p, int mode) {
  if (mode == 2) {
    float4 r;
    asm volatile("ld.global.nc.L2::64B.v4.f32 {%0,%1,%2,%3}, [%4];"
                 : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w)
                 : "l"(p));
    return r;
  }
  return mode == 1 ? b2_ldg_stream(p) : __ldg(p);
}
template <int VEC>
__device__ __forceinline__ void b2_st_row(typename VecT<VEC>::type* p, const typename VecT<VEC>::type& v, int mode) {
  *p = v;
}
template <>
__device__ __forceinline__ void b2_st_row<4>(float4* p, const float4& v, int mode) {
  if (mode == 1) b2_stg_stream(p, v); else *p = v;
}

// HOT > 0: the first `hot_rows` rows of every table (FuxiCTR's tokenizer numbers ids by descending
// frequency, so small ids are the hot ones; Zipf-like data sends 20-40 % of the lookups there) are staged
// once per CTA in shared memory and served from it instead of L2.
template <typename IdxT, int VEC, int UNROLL, bool HOT>
__global__ void __launch_bounds__(256)
gather_fast_kernel(const __grid_constant__ B2FieldPack pack, int64_t batch, int lpr_log2,
                   int32_t* __restrict__ status, int stream, int hot_rows, int hot_dim) {
  using V = typename VecT<VEC>::type;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const SmemFields sf = b2_stage_fields(pack, smem_raw);
  const int nslots = pack.nslots, nfields = pack.nfields;
  float* hot = nullptr;
  if (HOT) {   // [field][row][hot_dim] fp32, rows beyond a table's vocabulary are never addressed
    hot = reinterpret_cast<float*>(smem_raw + ((pack_smem_bytes(pack.nfields) + 15) & ~(size_t) 15));
    const int per_row = hot_dim / VEC;
    const int total = nfields * hot_rows * per_row;
    for (int i = threadIdx.x; i < total; i += blockDim.x) {
      const int fi = i / (hot_rows * per_row);
      const int rem = i - fi * (hot_rows * per_row);
      const int r = rem / per_row, c = (rem - r * per_row) * VEC;
      V v = b2_vzero<VEC>();
      if (r < sf.f[fi].vocab)
        v = __ldg(reinterpret_cast<const V*>(reinterpret_cast<const float*>(sf.f[fi].table) + (int64_t) r * hot_dim + c));
      *reinterpret_cast<V*>(hot + ((int64_t) fi * hot_rows + r) * hot_dim + c) = v;
    }
    __syncthreads();
  }
  const bool all_len1 = pack.all_len1 != 0;
  const int sub = threadIdx.x & ((1 << lpr_log2) - 1);
  const int e = sub * VEC;  // first element this lane moves
  const int64_t nitems = batch * (int64_t) nslots;
  const int64_t ngroups = ((int64_t) gridDim.x * blockDim.x) >> lpr_log2;
  const int64_t group = ((int64_t) blockIdx.x * blockDim.x + threadIdx.x) >> lpr_log2;
  const bool small = nitems < (int64_t) 0x7fffffff;

  for (int64_t base = group; base < nitems; base += ngroups * UNROLL) {
    const V* src[UNROLL];
    V* dst[UNROLL];
    bool live[UNROLL];
    bool in_smem[UNROLL];
    // Phase 1: all index loads in flight together.
#pragma unroll
    for (int u = 0; u < UNROLL; ++u) {
      const int64_t item = base + (int64_t) u * ngroups;
      live[u] = false;
      in_smem[u] = false;
      src[u] = nullptr;
      dst[u] = nullptr;
      if (item < nitems) {
        int64_t b;
        int slot;
        if (small) {
          const uint32_t it = (uint32_t) item;
          const uint32_t bq = it / (uint32_t) nslots;
          b = bq;
          slot = (int) (it - bq * (uint32_t) nslots);
        } else {
          b = item / nslots;
          slot = (int) (item - b * nslots);
        }
        const int fi = all_len1 ? slot : b2_slot_field(sf.slot_start, nfields, slot);
        const b2_field& fd = sf.f[fi];
        const int l = slot - sf.slot_start[fi];
        const int64_t row = b2_load_index<IdxT>(fd.idx, b * fd.idx_stride + l);
        const bool lane_on = e < fd.dim;
        if (lane_on) {
          dst[u] = reinterpret_cast<V*>(reinterpret_cast<float*>(fd.out) + b * fd.out_stride +
                                        (int64_t) l * fd.dim + e);
          if (HOT && row >= 0 && row < hot_rows && row < fd.vocab) {
            src[u] = reinterpret_cast<const V*>(hot + ((int64_t) fi * hot_rows + row) * hot_dim + e);
            live[u] = in_smem[u] = true;
          } else if (row >= 0 && row < fd.vocab) {
            src[u] = reinterpret_cast<const V*>(reinterpret_cast<const float*>(fd.table) +
                                                row * fd.dim + e);
            live[u] = true;
          } else if (status != nullptr && sub == 0) {
            atomicMax(status, fi + 1);  // reference raises IndexError; we flag and zero-fill
          }
        }
      }
    }
    // Phase 2: all row loads in flight together.
    V val[UNROLL];
#pragma unroll
    for (int u = 0; u < UNROLL; ++u) {
      val[u] = b2_vzero<VEC>();
      if (live[u]) val[u] = (HOT && in_smem[u]) ? *src[u] : b2_ld_row<VEC>(src[u], stream);
    }
    // Phase 3: coalesced stores of the stacked/concatenated tensor.
#pragma unroll
    for (int u = 0; u < UNROLL; ++u)
      if (dst[u] != nullptr) b2_st_row<VEC>(dst[u], val[u], stream);
  }
}

// ---------------------------------------------------------------------------------
// Forward, general path: pooled sequence fields and rows longer than one pass.
// One group of LPR lanes per (sample, slot); a pooled field is a single slot whose
// group walks the L positions and reduces in registers (fp32, position order —
// the same order torch.sum(dim=1) uses for a short inner loop).
// ---------------------------------------------------------------------------------
template <typename IdxT, int VEC>
__global__ void __launch_bounds__(256)
gather_general_kernel(const __grid_constant__ B2FieldPack pack, int64_t batch, int lpr_log2,
                      float* __restrict__ mean_count, int32_t* __restrict__ status) {
  using V = typename VecT<VEC>::type;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const SmemFields sf = b2_stage_fields(pack, smem_raw);
  const int nslots = pack.nslots, nfields = pack.nfields;
  const int LPR = 1 << lpr_log2;
  const int lane = threadIdx.x & 31;
  const int sub = lane & (LPR - 1);
  const unsigned gmask = (LPR == 32) ? 0xffffffffu : (((1u << LPR) - 1u) << (lane & ~(LPR - 1)));
  const int64_t nitems = batch * (int64_t) nslots;
  const int64_t ngroups = ((int64_t) gridDim.x * blockDim.x) >> lpr_log2;
  const int64_t group = ((int64_t) blockIdx.x * blockDim.x + threadIdx.x) >> lpr_log2;

  for (int64_t item = group; item < nitems; item += ngroups) {
    const int64_t b = item / nslots;
    const int slot = (int) (item - b * nslots);
    const int fi = b2_slot_field(sf.slot_start, nfields, slot);
    const b2_field fd = sf.f[fi];
    const float* table = reinterpret_cast<const float*>(fd.table);
    float* out = reinterpret_cast<float*>(fd.out) + b * fd.out_stride;
    const bool pooled = (fd.seq_len > 1 && fd.pool != B2_POOL_NONE);
    if (!pooled) {
      const int l = slot - sf.slot_start[fi];
      const int64_t row = b2_load_index<IdxT>(fd.idx, b * fd.idx_stride + l);
      const bool ok = row >= 0 && row < fd.vocab;
      if (!ok && status != nullptr && sub == 0) atomicMax(status, fi + 1);
      for (int e = sub * VEC; e < fd.dim; e += LPR * VEC) {
        V v = b2_vzero<VEC>();
        if (ok) v = __ldg(reinterpret_cast<const V*>(table + row * fd.dim + e));
        *reinterpret_cast<V*>(out + (int64_t) l * fd.dim + e) = v;
      }
    } else {
      // MaskedSumPooling: sum over positions (pooling.py:73).
      // MaskedAveragePooling: sum / (count(rows whose vector sum != 0) + 1e-12) (pooling.py:45-49).
      float count = 0.f;
      if (fd.pool == B2_POOL_MEAN) {
        for (int l = 0; l < fd.seq_len; ++l) {
          const int64_t row = b2_load_index<IdxT>(fd.idx, b * fd.idx_stride + l);
          const bool ok = row >= 0 && row < fd.vocab;
          float part = 0.f;
          if (ok)
            for (int e = sub * VEC; e < fd.dim; e += LPR * VEC)
              part += b2_vsum(__ldg(reinterpret_cast<const V*>(table + row * fd.dim + e)));
          for (int o = LPR >> 1; o > 0; o >>= 1) part += __shfl_xor_sync(gmask, part, o);
          count += (part != 0.f) ? 1.f : 0.f;
        }
        if (mean_count != nullptr && sub == 0) mean_count[(int64_t) fi * batch + b] = count;
      }
      for (int e = sub * VEC; e < fd.dim; e += LPR * VEC) {
        V acc = b2_vzero<VEC>();
        for (int l = 0; l < fd.seq_len; ++l) {
          const int64_t row = b2_load_index<IdxT>(fd.idx, b * fd.idx_stride + l);
          const bool ok = row >= 0 && row < fd.vocab;
          if (!ok && status != nullptr && sub == 0 && e == 0) atomicMax(status, fi + 1);
          if (ok) b2_vadd(acc, __ldg(reinterpret_cast<const V*>(table + row * fd.dim + e)));
        }
        if (fd.pool == B2_POOL_MEAN) acc = b2_vdiv(acc, count + 1e-12f);
        *reinterpret_cast<V*>(out + e) = acc;
      }
    }
  }
}

// ---------------------------------------------------------------------------------
// Backward: dense-gradient scatter-add with warp-level aggregation.
// Before issuing its vector `red`, each LPR-lane group looks (match.any on the
// destination row address) for other groups of the same warp that target the
// same row; the lowest such group sums the duplicates through shuffles and
// issues ONE reduction.  Hot Zipf rows therefore cost one L2 atomic per warp
// instead of one per occurrence.
// ---------------------------------------------------------------------------------
template <typename IdxT, int VEC>
__global__ void __launch_bounds__(256)
scatter_bwd_kernel(const __grid_constant__ B2FieldPack pack, int64_t batch, int lpr_log2,
                   const float* __restrict__ mean_count) {
  using V = typename VecT<VEC>::type;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const SmemFields sf = b2_stage_fields(pack, smem_raw);
  const int nfields = pack.nfields;
  // In the backward every (field, position) is its own slot — pooled fields fan the
  // same incoming gradient out to all L rows.  slot_start here counts seq_len per field.
  const int nslots = pack.nslots;
  const int LPR = 1 << lpr_log2;
  const int lane = threadIdx.x & 31;
  const int sub = lane & (LPR - 1);
  const int my_group = lane >> lpr_log2;
  const int groups_per_warp = 32 >> lpr_log2;
  const int64_t nitems = batch * (int64_t) nslots;
  const int64_t ngroups = ((int64_t) gridDim.x * blockDim.x) >> lpr_log2;
  const int64_t group = ((int64_t) blockIdx.x * blockDim.x + threadIdx.x) >> lpr_log2;
  // Warp-uniform trip count so the shuffles below are executed by all 32 lanes.
  const int64_t warp_first = group - my_group;

  for (int64_t wbase = warp_first; wbase < nitems; wbase += ngroups) {
    const int64_t item = wbase + my_group;
    float* drow = nullptr;        // destination row (gradient table), null = nothing to add
    const float* grow = nullptr;  // incoming gradient row
    int dim = 0;
    float scale = 1.f;
    if (item < nitems) {
      const int64_t b = item / nslots;
      const int slot = (int) (item - b * nslots);
      const int fi = pack.all_len1 ? slot : b2_slot_field(sf.slot_start, nfields, slot);
      const b2_field& fd = sf.f[fi];
      const int l = slot - sf.slot_start[fi];
      const int64_t row = b2_load_index<IdxT>(fd.idx, b * fd.idx_stride + l);
      if (row >= 0 && row < fd.vocab && row != (int64_t) fd.padding_idx) {
        dim = fd.dim;
        drow = reinterpret_cast<float*>(const_cast<void*>(fd.table)) + row * fd.dim;
        const bool pooled = (fd.seq_len > 1 && fd.pool != B2_POOL_NONE);
        grow = reinterpret_cast<const float*>(fd.out) + b * fd.out_stride +
               (pooled ? 0 : (int64_t) l * fd.dim);
        if (pooled && fd.pool == B2_POOL_MEAN)
          scale = 1.f / (mean_count[(int64_t) fi * batch + b] + 1e-12f);
      }
    }
    // Peers: lanes of the warp aiming at the same destination row.
    const unsigned peers = __match_any_sync(0xffffffffu, (unsigned long long) drow);
    // Bit g of gset = group g targets my row (take each group's sub-lane 0 bit).
    unsigned gset = 0;
    for (int g = 0; g < groups_per_warp; ++g) gset |= ((peers >> (g << lpr_log2)) & 1u) << g;
    const bool leader = (drow != nullptr) && ((gset & ((1u << my_group) - 1u)) == 0u);
    const bool has_dups = (drow != nullptr) && (gset != (1u << my_group));
    const unsigned any_dups = __ballot_sync(0xffffffffu, has_dups);
    const int max_dim = __reduce_max_sync(0xffffffffu, dim);

    for (int e0 = 0; e0 < max_dim; e0 += LPR * VEC) {
      const int e = e0 + sub * VEC;
      V v = b2_vzero<VEC>();
      if (grow != nullptr && e < dim) {
        v = *reinterpret_cast<const V*>(grow + e);
        if (scale != 1.f) v = b2_vscale(v, scale);
      }
      if (any_dups != 0u) {
        // Sum duplicates into the leader: walk the groups, pull lane (g*LPR+sub)'s value.
        V acc = v;
        for (int g = 0; g < groups_per_warp; ++g) {
          const int srcl = (g << lpr_log2) + sub;
          V o;
          if constexpr (VEC == 4) {
            o.x = __shfl_sync(0xffffffffu, v.x, srcl);
            o.y = __shfl_sync(0xffffffffu, v.y, srcl);
            o.z = __shfl_sync(0xffffffffu, v.z, srcl);
            o.w = __shfl_sync(0xffffffffu, v.w, srcl);
          } else if constexpr (VEC == 2) {
            o.x = __shfl_sync(0xffffffffu, v.x, srcl);
            o.y = __shfl_sync(0xffffffffu, v.y, srcl);
          } else {
            o = __shfl_sync(0xffffffffu, v, srcl);
          }
          if (g != my_group && ((gset >> g) & 1u)) b2_vadd(acc, o);
        }
        v = acc;
      }
      if (leader && e < dim) b2_vred(drow + e, v);
    }
  }
}

// ---------------------------------------------------------------------------------
// LogisticRegression: out[b] = sum_slots w_f[idx] (+ bias).  One warp per sample,
// lanes stride over the (field, position) slots, shuffle-reduce.
// ---------------------------------------------------------------------------------
template <typename IdxT>
__global__ void __launch_bounds__(256)
lr_fwd_kernel(const __grid_constant__ B2FieldPack pack, int64_t batch,
              const float* __restrict__ bias, float* __restrict__ out,
              int32_t* __restrict__ status) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const SmemFields sf = b2_stage_fields(pack, smem_raw);
  const int nslots = pack.nslots, nfields = pack.nfields;
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t) blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t) gridDim.x * blockDim.x) >> 5;
  const float bv = (bias != nullptr) ? __ldg(bias) : 0.f;
  for (int64_t b = warp; b < batch; b += nwarps) {
    float acc = 0.f;
    for (int slot = lane; slot < nslots; slot += 32) {
      const int fi = pack.all_len1 ? slot : b2_slot_field(sf.slot_start, nfields, slot);
      const b2_field& fd = sf.f[fi];
      const int l = slot - sf.slot_start[fi];
      const int64_t row = b2_load_index<IdxT>(fd.idx, b * fd.idx_stride + l);
      if (row >= 0 && row < fd.vocab) acc += __ldg(reinterpret_cast<const float*>(fd.table) + row);
      else if (status != nullptr) atomicMax(status, fi + 1);
    }
    acc = b2_warp_sum(acc);
    if (lane == 0) out[b] = acc + bv;
  }
}

template <typename IdxT>
__global__ void __launch_bounds__(256)
lr_bwd_kernel(const __grid_constant__ B2FieldPack pack, int64_t batch,
              const float* __restrict__ gout, float* __restrict__ gbias) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const SmemFields sf = b2_stage_fields(pack, smem_raw);
  __shared__ float red[32];
  const int nslots = pack.nslots, nfields = pack.nfields;
  const int64_t nitems = batch * (int64_t) nslots;
  const int64_t nthreads = (int64_t) gridDim.x * blockDim.x;
  float gb = 0.f;
  for (int64_t item = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; item < nitems;
       item += nthreads) {
    const int64_t b = item / nslots;
    const int slot = (int) (item - b * nslots);
    const int fi = pack.all_len1 ? slot : b2_slot_field(sf.slot_start, nfields, slot);
    const b2_field& fd = sf.f[fi];
    const int l = slot - sf.slot_start[fi];
    const float g = __ldg(gout + b);
    if (slot == 0) gb += g;
    const int64_t row = b2_load_index<IdxT>(fd.idx, b * fd.idx_stride + l);
    if (row >= 0 && row < fd.vocab && row != (int64_t) fd.padding_idx)
      b2_red_add(reinterpret_cast<float*>(const_cast<void*>(fd.table)) + row, g);
  }
  if (gbias != nullptr) {
    const float t = b2_block_sum(gb, red);
    if (threadIdx.x == 0 && t != 0.f) b2_red_add(gbias, t);
  }
}

// ---------------------------------------------------------------------------------
// Host side
// ---------------------------------------------------------------------------------
template <typename IdxT>
static int launch_gather(const B2FieldPack& pack, int64_t batch, int vec, int max_dim,
                         bool any_pooled, float* mean_count, int32_t* status, int hot_rows, cudaStream_t st) {
  const int block = 256;
  size_t smem = pack_smem_bytes(pack.nfields);
  int lpr_log2 = next_pow2_log2((max_dim + vec - 1) / vec);
  if (lpr_log2 > 5) lpr_log2 = 5;
  const bool one_pass = ((1 << lpr_log2) * vec) >= max_dim;
  const int64_t nitems = batch * (int64_t) pack.nslots;
  if (!any_pooled && one_pass) {
    // Large launches unroll deeper: 8 independent 16-byte row loads per lane in flight
    // (tools/debug_gather.py on 10 GB of tables, B=524288: 3.31 TB/s at 4, 3.77 TB/s at 8).
    static const int env_unroll = getenv("B2_GATHER_UNROLL") ? atoi(getenv("B2_GATHER_UNROLL")) : 0;
    static const int env_stream = getenv("B2_GATHER_STREAM") ? atoi(getenv("B2_GATHER_STREAM")) : -1;
    const bool big = nitems >= (int64_t) 1 << 20;
    const int unroll = env_unroll ? env_unroll : (big ? 8 : 4);
    const int stream = env_stream > 0 ? env_stream : 0;  // load flavour (b2_ld_row); measured (10 GB tables, B=524288): 3.77 TB/s plain vs 3.65 TB/s streaming
    // hot-row staging: one common dim, every field one slot, a staging area of at most 44 KB per CTA
    bool same_dim = pack.all_len1 != 0;
    for (int i = 0; i < pack.nfields && same_dim; ++i) same_dim = pack.f[i].dim == max_dim;
    const size_t hot_bytes = (size_t) pack.nfields * hot_rows * max_dim * sizeof(float);
    if (hot_rows > 0 && same_dim && vec == 4 && unroll == 8 && (max_dim % 4) == 0 && hot_bytes <= 44 * 1024) {
      const size_t hsmem = ((smem + 15) & ~(size_t) 15) + hot_bytes;
      const int grid = grid_for(b2_ceil_div(nitems, 8) << lpr_log2, block);
      gather_fast_kernel<IdxT, 4, 8, true><<<grid, block, hsmem, st>>>(pack, batch, lpr_log2, status, stream, hot_rows, max_dim);
      B2_CUDA_LAUNCH_CHECK("b2_embed_gather_fwd");
      return B2_OK;
    }
    if (unroll == 8) {
      const int grid = grid_for(b2_ceil_div(nitems, 8) << lpr_log2, block);
      if (vec == 4) gather_fast_kernel<IdxT, 4, 8, false><<<grid, block, smem, st>>>(pack, batch, lpr_log2, status, stream, 0, 0);
      else if (vec == 2) gather_fast_kernel<IdxT, 2, 8, false><<<grid, block, smem, st>>>(pack, batch, lpr_log2, status, stream, 0, 0);
      else gather_fast_kernel<IdxT, 1, 8, false><<<grid, block, smem, st>>>(pack, batch, lpr_log2, status, stream, 0, 0);
    } else {
      const int grid = grid_for(b2_ceil_div(nitems, 4) << lpr_log2, block);
      if (vec == 4) gather_fast_kernel<IdxT, 4, 4, false><<<grid, block, smem, st>>>(pack, batch, lpr_log2, status, stream, 0, 0);
      else if (vec == 2) gather_fast_kernel<IdxT, 2, 4, false><<<grid, block, smem, st>>>(pack, batch, lpr_log2, status, stream, 0, 0);
      else gather_fast_kernel<IdxT, 1, 4, false><<<grid, block, smem, st>>>(pack, batch, lpr_log2, status, stream, 0, 0);
    }
  } else {
    const int grid = grid_for(nitems << lpr_log2, block);
    if (vec == 4) gather_general_kernel<IdxT, 4><<<grid, block, smem, st>>>(pack, batch, lpr_log2, mean_count, status);
    else if (vec == 2) gather_general_kernel<IdxT, 2><<<grid, block, smem, st>>>(pack, batch, lpr_log2, mean_count, status);
    else gather_general_kernel<IdxT, 1><<<grid, block, smem, st>>>(pack, batch, lpr_log2, mean_count, status);
  }
  B2_CUDA_LAUNCH_CHECK("b2_embed_gather_fwd");
  return B2_OK;
}

template <typename IdxT>
static int launch_scatter(const B2FieldPack& pack, int64_t batch, int vec, int max_dim,
                          const float* mean_count, cudaStream_t st) {
  const int block = 256;
  const size_t smem = pack_smem_bytes(pack.nfields);
  int lpr_log2 = next_pow2_log2((max_dim + vec - 1) / vec);
  if (lpr_log2 > 5) lpr_log2 = 5;
  const int64_t nitems = batch * (int64_t) pack.nslots;
  const int grid = grid_for(nitems << lpr_log2, block);
  if (vec == 4) scatter_bwd_kernel<IdxT, 4><<<grid, block, smem, st>>>(pack, batch, lpr_log2, mean_count);
  else if (vec == 2) scatter_bwd_kernel<IdxT, 2><<<grid, block, smem, st>>>(pack, batch, lpr_log2, mean_count);
  else scatter_bwd_kernel<IdxT, 1><<<grid, block, smem, st>>>(pack, batch, lpr_log2, mean_count);
  B2_CUDA_LAUNCH_CHECK("b2_embed_scatter_bwd");
  return B2_OK;
}

extern "C" B2_API int b2_embed_gather_fwd(const b2_field* fields, int nfields, int64_t batch,
                                   int idx_dtype, int elem_dtype, float* mean_count,
                                   int32_t* status, void* stream) {
  return b2_embed_gather_hot_fwd(fields, nfields, batch, idx_dtype, elem_dtype, mean_count, status, 0, stream);
}

extern "C" B2_API int b2_embed_gather_hot_fwd(const b2_field* fields, int nfields, int64_t batch,
                                       int idx_dtype, int elem_dtype, float* mean_count,
                                       int32_t* status, int hot_rows, void* stream) {
  B2_REQUIRE(hot_rows >= 0, "negative hot_rows");
  B2_REQUIRE(elem_dtype == B2_F32, "elem_dtype %d unsupported (only B2_F32)", elem_dtype);
  B2_REQUIRE(batch >= 0, "negative batch");
  if (batch == 0) return B2_OK;
  static thread_local B2FieldPack pack;
  int vec, max_dim;
  bool any_pooled;
  int rc = build_pack(pack, fields, nfields, false, true, &vec, &max_dim, &any_pooled);
  if (rc != B2_OK) return rc;
  for (int i = 0; i < nfields; ++i)
    if (fields[i].seq_len > 1 && fields[i].pool == B2_POOL_MEAN)
      B2_REQUIRE(mean_count != nullptr, "field %d: POOL_MEAN needs mean_count", i);
  cudaStream_t st = (cudaStream_t) stream;
  switch (idx_dtype) {
    case B2_F64: return launch_gather<double>(pack, batch, vec, max_dim, any_pooled, mean_count, status, hot_rows, st);
    case B2_I64: return launch_gather<int64_t>(pack, batch, vec, max_dim, any_pooled, mean_count, status, hot_rows, st);
    case B2_I32: return launch_gather<int32_t>(pack, batch, vec, max_dim, any_pooled, mean_count, status, hot_rows, st);
    default: return b2_fail(B2_E_INVALID, "idx_dtype %d unsupported", idx_dtype);
  }
}

extern "C" B2_API int b2_embed_scatter_bwd(const b2_field* fields, int nfields, int64_t batch,
                                    int idx_dtype, int elem_dtype, const float* mean_count,
                                    void* stream) {
  B2_REQUIRE(elem_dtype == B2_F32, "elem_dtype %d unsupported (only B2_F32)", elem_dtype);
  B2_REQUIRE(batch >= 0, "negative batch");
  if (batch == 0) return B2_OK;
  static thread_local B2FieldPack pack;
  int vec, max_dim;
  bool any_pooled;
  int rc = build_pack(pack, fields, nfields, true, true, &vec, &max_dim, &any_pooled);
  if (rc != B2_OK) return rc;
  for (int i = 0; i < nfields; ++i)
    if (fields[i].seq_len > 1 && fields[i].pool == B2_POOL_MEAN)
      B2_REQUIRE(mean_count != nullptr, "field %d: POOL_MEAN needs mean_count", i);
  cudaStream_t st = (cudaStream_t) stream;
  switch (idx_dtype) {
    case B2_F64: return launch_scatter<double>(pack, batch, vec, max_dim, mean_count, st);
    case B2_I64: return launch_scatter<int64_t>(pack, batch, vec, max_dim, mean_count, st);
    case B2_I32: return launch_scatter<int32_t>(pack, batch, vec, max_dim, mean_count, st);
    default: return b2_fail(B2_E_INVALID, "idx_dtype %d unsupported", idx_dtype);
  }
}

template <typename IdxT>
static int launch_lr_fwd(const B2FieldPack& pack, int64_t batch, const float* bias, float* out,
                         int32_t* status, cudaStream_t st) {
  const int block = 256;
  const int grid = grid_for(batch * 32, block);
  lr_fwd_kernel<IdxT><<<grid, block, pack_smem_bytes(pack.nfields), st>>>(pack, batch, bias, out, status);
  B2_CUDA_LAUNCH_CHECK("b2_lr_fwd");
  return B2_OK;
}
template <typename IdxT>
static int launch_lr_bwd(const B2FieldPack& pack, int64_t batch, const float* gout, float* gbias,
                         cudaStream_t st) {
  const int block = 256;
  const int grid = grid_for(batch * (int64_t) pack.nslots, block);
  lr_bwd_kernel<IdxT><<<grid, block, pack_smem_bytes(pack.nfields), st>>>(pack, batch, gout, gbias);
  B2_CUDA_LAUNCH_CHECK("b2_lr_bwd");
  return B2_OK;
}

extern "C" B2_API int b2_lr_fwd(const b2_field* fields, int nfields, int64_t batch, int idx_dtype,
                         const float* bias, float* out, int32_t* status, void* stream) {
  B2_REQUIRE(out != nullptr, "out is NULL");
  B2_REQUIRE(batch >= 0, "negative batch");
  if (batch == 0) return B2_OK;
  static thread_local B2FieldPack pack;
  int rc = build_pack(pack, fields, nfields, true, false, nullptr, nullptr, nullptr);
  if (rc != B2_OK) return rc;
  cudaStream_t st = (cudaStream_t) stream;
  switch (idx_dtype) {
    case B2_F64: return launch_lr_fwd<double>(pack, batch, bias, out, status, st);
    case B2_I64: return launch_lr_fwd<int64_t>(pack, batch, bias, out, status, st);
    case B2_I32: return launch_lr_fwd<int32_t>(pack, batch, bias, out, status, st);
    default: return b2_fail(B2_E_INVALID, "idx_dtype %d unsupported", idx_dtype);
  }
}

extern "C" B2_API int b2_lr_bwd(const b2_field* fields, int nfields, int64_t batch, int idx_dtype,
                         const float* gout, float* gbias, void* stream) {
  B2_REQUIRE(gout != nullptr, "gout is NULL");
  B2_REQUIRE(batch >= 0, "negative batch");
  if (batch == 0) return B2_OK;
  static thread_local B2FieldPack pack;
  int rc = build_pack(pack, fields, nfields, true, false, nullptr, nullptr, nullptr);
  if (rc != B2_OK) return rc;
  cudaStream_t st = (cudaStream_t) stream;
  switch (idx_dtype) {
    case B2_F64: return launch_lr_bwd<double>(pack, batch, gout, gbias, st);
    case B2_I64: return launch_lr_bwd<int64_t>(pack, batch, gout, gbias, st);
    case B2_I32: return launch_lr_bwd<int32_t>(pack, batch, gout, gbias, st);
    default: return b2_fail(B2_E_INVALID, "idx_dtype %d unsupported", idx_dtype);
  }
}

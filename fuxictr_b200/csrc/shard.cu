// shard.cu — row-sharded embedding tables across the GPUs of one NVSwitch box: the lookup and
// its exchange are ONE kernel over peer memory (no NCCL all-to-all, no variable-size splits).
//
// Layout (SURVEY.md 8e): row `r` of every table lives on rank r % world at local row r / world.
// Every rank exposes, in NVLink peer-mapped ("symmetric") memory,
//     ids   (B_local, W)  the batch matrix the collator produced (indices of ITS samples)
//     emb   (B_local, F*D) the embedding rows of ITS samples      — written by the row owners
//     lrw   (B_local, F)   the D=1 LogisticRegression weights      — written by the row owners
//     gemb  (B_local, F*D), glogit (B_local)  gradients of ITS samples — read by the row owners
// Forward  `shard_push_kernel`: each rank walks the ids of ALL ranks (P2P loads, 8 B per item),
//   and for the rows it owns gathers the local table row and stores it STRAIGHT into the
//   requesting rank's `emb`/`lrw` (P2P stores, 16 B per lane).  Each (sample, field) slot has
//   exactly one owner, so the stores never collide and exactly (world-1)/world of B*F*D*4 bytes
//   cross NVLink — the volume of an ideal all-to-all, with the gather fused into the transfer.
// While pushing, the owner appends every (requester, sample, field, local row) it served to a local
//   list (warp-aggregated append): ~B_local*F entries, its exact share of the global batch.
// Backward `shard_pull_kernel`: the owner walks THAT LIST (not world*B*F candidates, and no second
//   pass over the peers' id matrices), pulls each gradient row from the requesting rank's `gemb`
//   (P2P loads) and scatter-adds it (warp-aggregated `red.global.add.v4.f32`) into its local
//   dense-gradient shard.
// `shard_publish_ids_kernel`: one launch stores this rank's ids, narrowed to int32, and the padding rows it owns
//   into its slot on every peer.
// Replaces, for sharded tables, FeatureEmbedding/LogisticRegression lookups and their autograd
// (fuxictr/pytorch/layers/embeddings/feature_embedding.py:261-297,
//  fuxictr/pytorch/layers/blocks/logistic_regression.py:55-58); the reference has no multi-GPU path.
// Cross-rank ordering (ids visible -> push -> pushes landed -> ... ) is the caller's barrier.
#include "embed_common.cuh"
#include "lazy_replay.cuh"

namespace {
struct PeerPtrs {
  const void* ids[16];
  float* emb[16];
  float* lrw[16];
  const float* gemb[16];
  const float* glogit[16];
};

struct BcastDst { void* p[16]; };

// flags packed next to the field index in an owned-list entry
#define B2_OWN_EMB (1 << 17)
#define B2_OWN_LR (1 << 16)

#define B2_OWN_ZERO (1 << 18)    // out-of-range id: the slot is defined as a zero row, no gradient
#define B2_OWN_PAD (1 << 19)     // padding id: the requester copies the published padding row, no gradient

constexpr int SERVE_U = 4;       // list entries a lane group serves at once (loads in flight)

// Candidates are (requester, sample, SLOT): a categorical field is one slot, an unpooled sequence of
// length L is L consecutive slots (slot_start of the pack), S = nslots slots per sample.  Slot s of
// sample b takes its id from column idx_stride + (s - slot_start[f]) and lands at b*S*D + s*D of the
// requester's emb; rem = b*S + s is what an owned-list entry keeps in .y.
// Two phases per 256-item chunk.  SCAN: one thread per candidate reads the id and keeps it only when this
// rank owns the row — the (world-1)/world candidates that belong to other ranks cost one coalesced 4-byte
// load each.  With pad_rows, a padding id is served by the REQUESTER itself from the padding rows their
// owners published before the push (b2_shard_publish_ids): no rank serves other ranks' padding slots.
// SERVE: the block walks the compacted list in shared memory with dim/4 lanes per entry (gather the table
// row, 16-byte P2P stores into the requester's slot), and appends the entries that will receive a gradient
// to the rank's owned-row list with ONE global atomic per chunk (a per-warp atomic on the one counter
// serialises ~1e5 times per launch at 8 ranks).
// LAZY: the tables are lazily evaluated (b2_lazy_ctx); ALL_LEN1: every field is one slot (no slot ->
// field search) — separate instantiations, so that the plain categorical push keeps its register budget
// (and occupancy).
// RAGGED (the evaluation lookup, b2_shard_lookup): requester p has rows_all[p] <= batch_local samples this
// round, so the candidates of samples b >= rows_all[p] are skipped; it runs without an owned list and lazy
// context, and the training instantiations (RAGGED = false) never read rows_all.
template <typename IdxT, bool LAZY, bool ALL_LEN1, bool RAGGED>
__global__ void __launch_bounds__(256)
shard_push_kernel(const __grid_constant__ B2FieldPack emb, const __grid_constant__ B2FieldPack lr,
                  const __grid_constant__ PeerPtrs peers, const __grid_constant__ b2_lazy_ctx lz,
                  int64_t batch_local, int64_t ids_stride,
                  int dim, int lpr_log2, int has_lr, int world, int rank,
                  int32_t* __restrict__ status, int4* __restrict__ owned, int32_t* __restrict__ owned_count,
                  int32_t owned_cap, const float* __restrict__ pad_rows, const int32_t* __restrict__ rows_all) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const SmemFields sf = b2_stage_fields(emb, smem_raw);
  SmemFields lf;
  lf.f = nullptr;
  lf.slot_start = nullptr;
  const size_t pack_bytes = (pack_smem_bytes(emb.nfields) + 15) & ~(size_t) 15;
  if (has_lr) lf = b2_stage_fields(lr, smem_raw + pack_bytes);
  int4* list = reinterpret_cast<int4*>(smem_raw + 2 * pack_bytes);      // 256 entries
  __shared__ int s_front, s_back, s_gbase;
  const int F = emb.nfields;
  const int S = ALL_LEN1 ? F : emb.nslots;
  const int LPR = 1 << lpr_log2;
  const int lane = threadIdx.x & 31;
  const int sub = threadIdx.x & (LPR - 1);
  const int e = sub * 4;
  const int64_t per_rank = batch_local * (int64_t) S;
  const int64_t nitems = per_rank * world;
  const int done = LAZY ? (int) *lz.step_dev : 0;   // lazy tables: steps completed so far
  const int gstride = 256 >> lpr_log2;               // lane groups per block
  for (int64_t base = (int64_t) blockIdx.x * 256; base < nitems; base += (int64_t) gridDim.x * 256) {
    if (threadIdx.x == 0) { s_front = 0; s_back = 0; }
    __syncthreads();
    // ---- scan
    const int64_t item = base + threadIdx.x;
    int4 entry = make_int4(0, 0, 0, 0);
    int kind = 0;                       // 1: goes on the owned list (front), 2: served only (back)
    if (item < nitems && (!RAGGED || (item % per_rank) / S < (int64_t) __ldg(rows_all + item / per_rank))) {
      const int p = (int) (item / per_rank);           // requesting rank
      const int64_t rem = item - (int64_t) p * per_rank;
      const int64_t b = rem / S;
      const int slot = (int) (rem - b * S);
      const int f = ALL_LEN1 ? slot : b2_slot_field(sf.slot_start, F, slot);
      const b2_field& fd = sf.f[f];
      // fd.idx_stride carries the COLUMN of this field inside the batch matrix (a sequence's columns are
      // consecutive: position k of it is column idx_stride + k)
      const int64_t col = ALL_LEN1 ? fd.idx_stride : fd.idx_stride + (slot - sf.slot_start[f]);
      const int64_t row = b2_load_index<IdxT>(peers.ids[p], b * ids_stride + col);
      if (row < 0 || row >= fd.vocab) {
        if (status != nullptr && p == rank) atomicMax(status, f + 1);
        if ((row < 0 ? 0 : (int) (row % world)) == rank) {  // keep the slot defined: zero row
          entry = make_int4(p, (int) rem, 0, f | B2_OWN_ZERO);
          kind = 2;
        }
      } else if (pad_rows != nullptr && row == (int64_t) fd.padding_idx) {   // my own padding slot
        if (p == rank) {
          entry = make_int4(p, (int) rem, f, f | B2_OWN_PAD);
          kind = 2;
        }
      } else if ((int) (row % world) == rank) {          // my row
        int flags = (row != (int64_t) fd.padding_idx) ? B2_OWN_EMB : 0;     // padding rows get no gradient
        if (has_lr && row != (int64_t) lf.f[f].padding_idx) flags |= B2_OWN_LR;
        entry = make_int4(p, (int) rem, (int) (row / world), f | flags);
        kind = (flags != 0 && owned != nullptr) ? 1 : 2;
      }
    }
    // block compaction: list entries from the front, serve-only entries from the back
    const unsigned m1 = __ballot_sync(0xffffffffu, kind == 1), m2 = __ballot_sync(0xffffffffu, kind == 2);
    int b1 = 0, b2 = 0;
    if (lane == 0) {
      if (m1 != 0u) b1 = atomicAdd(&s_front, __popc(m1));
      if (m2 != 0u) b2 = atomicAdd(&s_back, __popc(m2));
    }
    b1 = __shfl_sync(0xffffffffu, b1, 0);
    b2 = __shfl_sync(0xffffffffu, b2, 0);
    const unsigned below = (1u << lane) - 1u;
    if (kind == 1) list[b1 + __popc(m1 & below)] = entry;
    if (kind == 2) list[255 - (b2 + __popc(m2 & below))] = entry;
    __syncthreads();
    const int nfront = s_front, nback = s_back;
    if (threadIdx.x == 0 && nfront > 0) s_gbase = atomicAdd(owned_count, nfront);
    // ---- serve: SERVE_U entries per lane group at once, all row loads (and for lazy tables all
    // last_step and moment loads) in flight; a stale row is brought up to date in registers before
    // it is stored (lazy_replay.cuh), an out-of-range id stores a zero row
    const int nserve = nfront + nback;
    for (int k0 = threadIdx.x >> lpr_log2; k0 < nserve; k0 += SERVE_U * gstride) {
      int4 it[SERVE_U];
      int f[SERVE_U];
      int64_t lrow[SERVE_U];
      bool on_e[SERVE_U], on_l[SERVE_U];
      float4 v[SERVE_U];
      float w[SERVE_U];
#pragma unroll
      for (int u = 0; u < SERVE_U; ++u) {
        const int k = k0 + u * gstride;
        it[u] = (k < nserve) ? list[k < nfront ? k : 255 - (k - nfront)] : make_int4(-1, 0, 0, B2_OWN_ZERO);
        f[u] = it[u].w & 0xffff;
        lrow[u] = it[u].z;
        // a padding entry reads row f of the published padding rows (its .z holds f): bit-exact, any value,
        // and never replayed (a padding row has no gradient, so Adam leaves it unchanged)
        const bool pad = (it[u].w & B2_OWN_PAD) != 0;
        const bool row_ok = !(it[u].w & (B2_OWN_ZERO | B2_OWN_PAD));
        on_e[u] = row_ok && e < dim;
        on_l[u] = row_ok && has_lr && sub == 0;
        v[u] = make_float4(0.f, 0.f, 0.f, 0.f);
        w[u] = 0.f;
        if ((row_ok || pad) && e < dim) {
          const float* t = pad ? pad_rows : reinterpret_cast<const float*>(sf.f[f[u]].table);
          v[u] = __ldg(reinterpret_cast<const float4*>(t + lrow[u] * dim + e));
        }
        if ((row_ok || pad) && has_lr && sub == 0) {
          const float* t = pad ? pad_rows + (int64_t) F * dim : reinterpret_cast<const float*>(lf.f[f[u]].table);
          w[u] = __ldg(t + lrow[u]);
        }
      }
      if (LAZY) b2_lazy_replay<SERVE_U>(lz, done, sf, lf, dim, e, f, lrow, on_e, on_l, v, w);
#pragma unroll
      for (int u = 0; u < SERVE_U; ++u) {
        const int p = it[u].x;
        if (p < 0) continue;
        const int64_t bf = it[u].y;
        if (e < dim) *reinterpret_cast<float4*>(peers.emb[p] + bf * dim + e) = v[u];   // P2P store
        if (has_lr && sub == 0) peers.lrw[p][bf] = w[u];
      }
    }
    __syncthreads();
    if (threadIdx.x < nfront) {
      const int pos = s_gbase + threadIdx.x;
      if (pos < owned_cap) owned[pos] = list[threadIdx.x];
    }
    __syncthreads();
  }
}

__global__ void __launch_bounds__(256)
shard_pull_kernel(const __grid_constant__ B2FieldPack emb, const __grid_constant__ B2FieldPack lr,
                  const __grid_constant__ PeerPtrs peers, const __grid_constant__ b2_lazy_ctx lz, int lazy,
                  int dim, int lpr_log2, int has_lr, float scale,
                  const int4* __restrict__ owned, const int32_t* __restrict__ owned_count, int32_t owned_cap,
                  const b2_touch tch) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const SmemFields sf = b2_stage_fields(emb, smem_raw);
  SmemFields lf;
  lf.f = nullptr;
  lf.slot_start = nullptr;
  if (has_lr) lf = b2_stage_fields(lr, smem_raw + ((pack_smem_bytes(emb.nfields) + 15) & ~(size_t) 15));
  const int S = emb.nslots;     // an entry's .y is sample * S + slot
  const int LPR = 1 << lpr_log2;
  const int lane = threadIdx.x & 31;
  const int sub = lane & (LPR - 1);
  const int my_group = lane >> lpr_log2;
  const int groups_per_warp = 32 >> lpr_log2;
  const int e = sub * 4;
  const int64_t nitems = min(*owned_count, owned_cap);
  const int64_t ngroups = ((int64_t) gridDim.x * blockDim.x) >> lpr_log2;
  const int64_t group = ((int64_t) blockIdx.x * blockDim.x + threadIdx.x) >> lpr_log2;
  const int64_t warp_first = group - my_group;
  const int tmark = lazy ? (int) *lz.step_dev + 1 : 0;   // the optimizer step these gradients feed
  for (int64_t wbase = warp_first; wbase < nitems; wbase += ngroups) {
    const int64_t item = wbase + my_group;
    float* drow = nullptr;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    int enq_e = -1, enq_l = -1;   // local rows (global over this rank's lazy tables) this lane enqueues
    if (item < nitems) {
      const int4 it = __ldg(owned + item);
      const int p = it.x, f = it.w & 0xffff;
      const int64_t bf = it.y, lrow = it.z;
      const b2_field& fd = sf.f[f];
      if ((it.w & B2_OWN_EMB) && fd.table != nullptr) {
        drow = reinterpret_cast<float*>(const_cast<void*>(fd.table)) + lrow * dim;
        // several requesters may send gradients for this row: the first of them this step enqueues it
        if (lazy && sub == 0) {
          const int grow = (int) (lz.grow_emb[f] + lrow);
          if (b2_lazy_claim(lz, grow, tmark)) enq_e = grow;
        }
        if (e < dim) {
          v = *reinterpret_cast<const float4*>(peers.gemb[p] + bf * dim + e);  // P2P load
          v.x *= scale; v.y *= scale; v.z *= scale; v.w *= scale;
        }
      }
      if (has_lr && sub == 0 && (it.w & B2_OWN_LR)) {
        const b2_field& ld = lf.f[f];
        if (ld.table != nullptr) {
          float* dst = reinterpret_cast<float*>(const_cast<void*>(ld.table)) + lrow;
          b2_red_add(dst, peers.glogit[p][bf / S] * scale);
          b2_touch_mark(tch, dst, true);
          if (lazy) {
            const int grow = (int) (lz.grow_lr[f] + lrow);
            if (b2_lazy_claim(lz, grow, tmark)) enq_l = grow;
          }
        }
      }
    }
    if (lazy) b2_lazy_append(lz, enq_e, enq_l, lane);
    const unsigned peers_mask = __match_any_sync(0xffffffffu, (unsigned long long) drow);
    unsigned gset = 0;
    for (int g = 0; g < groups_per_warp; ++g) gset |= ((peers_mask >> (g << lpr_log2)) & 1u) << g;
    const bool leader = (drow != nullptr) && ((gset & ((1u << my_group) - 1u)) == 0u);
    const bool has_dups = (drow != nullptr) && (gset != (1u << my_group));
    if (__ballot_sync(0xffffffffu, has_dups) != 0u) {
      float4 acc = v;
      for (int g = 0; g < groups_per_warp; ++g) {
        const int srcl = (g << lpr_log2) + sub;
        float4 o;
        o.x = __shfl_sync(0xffffffffu, v.x, srcl);
        o.y = __shfl_sync(0xffffffffu, v.y, srcl);
        o.z = __shfl_sync(0xffffffffu, v.z, srcl);
        o.w = __shfl_sync(0xffffffffu, v.w, srcl);
        if (g != my_group && ((gset >> g) & 1u)) { acc.x += o.x; acc.y += o.y; acc.z += o.z; acc.w += o.w; }
      }
      v = acc;
    }
    if (leader && e < dim) {
      b2_red_add_v4(drow + e, v);
      b2_touch_mark(tch, drow + e, e == 0);
    }
  }
}

// The id exchange, compressed: the batch matrix arrives as float64 (the reference's collator), the owners
// only need the row numbers — one launch truncates like `.long()`, narrows to int32 (vocabularies < 2^31)
// and stores the result into this rank's slot on every peer: 4 bytes per id over NVLink instead of 8.
template <typename IdxT>
__device__ __forceinline__ void bcast_ids(const void* __restrict__ src, int64_t n, const BcastDst& dst, int world) {
  const int64_t tid = (int64_t) blockIdx.x * blockDim.x + threadIdx.x, nth = (int64_t) gridDim.x * blockDim.x;
  const int64_t n4 = n >> 2;
  for (int64_t i = tid; i < n4; i += nth) {
    int4 v;
    v.x = (int) b2_load_index<IdxT>(src, 4 * i + 0);
    v.y = (int) b2_load_index<IdxT>(src, 4 * i + 1);
    v.z = (int) b2_load_index<IdxT>(src, 4 * i + 2);
    v.w = (int) b2_load_index<IdxT>(src, 4 * i + 3);
    for (int p = 0; p < world; ++p) reinterpret_cast<int4*>(dst.p[p])[i] = v;
  }
  for (int64_t i = (n4 << 2) + tid; i < n; i += nth) {
    const int v = (int) b2_load_index<IdxT>(src, i);
    for (int p = 0; p < world; ++p) reinterpret_cast<int32_t*>(dst.p[p])[i] = v;
  }
}

// Padding rows this rank owns (NULL: another rank publishes that field's row), and every rank's pad buffer.
struct PadSrc {
  const float* e[B2_MAX_FIELDS];
  const float* l[B2_MAX_FIELDS];
};
struct PadDst { float* p[16]; };

// The id exchange, plus the padding rows: the owner of each field's padding row stores it (and its LR weight)
// into every rank's pad buffer, (F, D) rows then F weights, so that every rank fills its own padding slots in
// the push.  The push that reads them comes after the barrier that follows this launch.
template <typename IdxT>
__device__ __forceinline__ void publish_ids_pad(const void* __restrict__ src, int64_t n, const BcastDst& dst,
                                                int world, const PadSrc& ps, const PadDst& pd, int nfields, int dim) {
  bcast_ids<IdxT>(src, n, dst, world);
  const int64_t tid = (int64_t) blockIdx.x * blockDim.x + threadIdx.x, nth = (int64_t) gridDim.x * blockDim.x;
  const int64_t nemb = (int64_t) nfields * dim, npad = nemb + nfields;
  for (int64_t i = tid; i < npad; i += nth) {
    const float* s;
    if (i < nemb) {
      const int f = (int) (i / dim);
      s = ps.e[f] != nullptr ? ps.e[f] + (i - (int64_t) f * dim) : nullptr;
    } else {
      s = ps.l[i - nemb];
    }
    if (s == nullptr) continue;
    const float v = *s;
    for (int p = 0; p < world; ++p) pd.p[p][i] = v;
  }
}

template <typename IdxT>
__global__ void __launch_bounds__(256)
shard_publish_ids_kernel(const void* __restrict__ src, int64_t n, const __grid_constant__ BcastDst dst, int world,
                         const __grid_constant__ PadSrc ps, const __grid_constant__ PadDst pd, int nfields, int dim) {
  publish_ids_pad<IdxT>(src, n, dst, world, ps, pd, nfields, dim);
}

struct RowsDst { int32_t* p[16]; };

// The evaluation round's exchange: the first `rows` rows of the batch matrix (n = rows * width ids), the padding
// rows, and the row count itself into word `rank` of every peer's rows_all — the bound of the lookup that follows
// the barrier.
template <typename IdxT>
__global__ void __launch_bounds__(256)
shard_publish_rows_kernel(const void* __restrict__ src, int64_t n, const __grid_constant__ BcastDst dst, int world,
                          const __grid_constant__ PadSrc ps, const __grid_constant__ PadDst pd, int nfields, int dim,
                          const __grid_constant__ RowsDst rd, int rank, int32_t rows) {
  publish_ids_pad<IdxT>(src, n, dst, world, ps, pd, nfields, dim);
  if (blockIdx.x == 0 && (int) threadIdx.x < world) rd.p[threadIdx.x][rank] = rows;
}

// After the push: logit[b] = [0.5*sum_d((sum_f e)^2 - sum_f e^2)] + [sum_f lrw[b,f] + bias]; sums[b,:] = sum_f e.
__global__ void __launch_bounds__(256)
front_reduce_kernel(const float* __restrict__ emb, const float* __restrict__ lrw,
                    const float* __restrict__ bias, int64_t batch, int F, int dim, int lpr_log2,
                    int want_fm, float* __restrict__ logit, float* __restrict__ sums) {
  const int LPR = 1 << lpr_log2;
  const int rows_per_pass = 32 >> lpr_log2;
  const int lane = threadIdx.x & 31;
  const int sub = lane & (LPR - 1), rg = lane >> lpr_log2;
  const int e = sub * 4;
  const bool lane_on = e < dim;
  const int64_t warp = ((int64_t) blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t) gridDim.x * blockDim.x) >> 5;
  const float bv = (bias != nullptr) ? __ldg(bias) : 0.f;
  const int64_t FD = (int64_t) F * dim;
  for (int64_t b = warp; b < batch; b += nwarps) {
    float4 s = make_float4(0.f, 0.f, 0.f, 0.f), q = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int f = rg; f < F; f += rows_per_pass) {
      if (lane_on) {
        const float4 v = *reinterpret_cast<const float4*>(emb + b * FD + (int64_t) f * dim + e);
        s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
        q.x = fmaf(v.x, v.x, q.x); q.y = fmaf(v.y, v.y, q.y); q.z = fmaf(v.z, v.z, q.z); q.w = fmaf(v.w, v.w, q.w);
      }
    }
    for (int o = LPR; o < 32; o <<= 1) {
      s.x += __shfl_xor_sync(0xffffffffu, s.x, o); s.y += __shfl_xor_sync(0xffffffffu, s.y, o);
      s.z += __shfl_xor_sync(0xffffffffu, s.z, o); s.w += __shfl_xor_sync(0xffffffffu, s.w, o);
      q.x += __shfl_xor_sync(0xffffffffu, q.x, o); q.y += __shfl_xor_sync(0xffffffffu, q.y, o);
      q.z += __shfl_xor_sync(0xffffffffu, q.z, o); q.w += __shfl_xor_sync(0xffffffffu, q.w, o);
    }
    if (sums != nullptr && rg == 0 && lane_on) *reinterpret_cast<float4*>(sums + b * dim + e) = s;
    float total = 0.f;
    if (want_fm) {
      float t = ((s.x * s.x - q.x) + (s.y * s.y - q.y) + (s.z * s.z - q.z) + (s.w * s.w - q.w)) * 0.5f;
      if (!lane_on) t = 0.f;
      for (int o = 1; o < LPR; o <<= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
      total = t;
    }
    float lrsum = 0.f;
    if (lrw != nullptr)
      for (int f = lane; f < F; f += 32) lrsum += lrw[b * F + f];
    lrsum = b2_warp_sum(lrsum);
    if (lane == 0) logit[b] = total + (lrsum + bv);
  }
}

// Before the pull: gemb[b,f,:] = gx[b,f,:] + gl[b] * (sums[b,:] - emb[b,f,:])   (second term if want_fm)
__global__ void __launch_bounds__(256)
front_gprep_kernel(const float* __restrict__ gx, const float* __restrict__ emb,
                   const float* __restrict__ sums, const float* __restrict__ glogit, int64_t batch,
                   int F, int dim, int want_fm, float* __restrict__ gemb, float* __restrict__ glogit_out,
                   float* __restrict__ gbias) {
  __shared__ float red[32];
  const int64_t n4 = batch * (int64_t) F * dim / 4;
  const int d4 = dim / 4;
  if (glogit_out != nullptr || gbias != nullptr) {
    // publish the logit gradient where the row owners can read it (LR tables); its sum is the LR bias gradient
    float acc = 0.f;
    for (int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; i < batch; i += (int64_t) gridDim.x * blockDim.x) {
      const float g = __ldg(glogit + i);
      if (glogit_out != nullptr) glogit_out[i] = g;
      acc += g;
    }
    if (gbias != nullptr) {
      const float t = b2_block_sum(acc, red);
      if (threadIdx.x == 0 && t != 0.f) b2_red_add(gbias, t);
    }
  }
  for (int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; i < n4;
       i += (int64_t) gridDim.x * blockDim.x) {
    const int64_t bf = i / d4;
    const int c = (int) (i - bf * d4);
    const int64_t b = bf / F;
    float4 g = (gx != nullptr) ? *reinterpret_cast<const float4*>(gx + i * 4) : make_float4(0.f, 0.f, 0.f, 0.f);
    if (want_fm) {
      const float gl = __ldg(glogit + b);
      const float4 ev = *reinterpret_cast<const float4*>(emb + i * 4);
      const float4 sv = *reinterpret_cast<const float4*>(sums + b * dim + c * 4);
      g.x = fmaf(gl, sv.x - ev.x, g.x); g.y = fmaf(gl, sv.y - ev.y, g.y);
      g.z = fmaf(gl, sv.z - ev.z, g.z); g.w = fmaf(gl, sv.w - ev.w, g.w);
    }
    *reinterpret_cast<float4*>(gemb + i * 4) = g;
  }
}

// One slot per categorical field, seq_len consecutive slots per unpooled sequence (the slots of `fields`,
// the LR pack takes the embedding pack's layout: LR tables exist only when every field is one slot).
void fill_pack_cols(B2FieldPack& pack, const b2_field* fields, int nfields) {
  int slots = 0;
  for (int i = 0; i < nfields; ++i) {
    pack.f[i] = fields[i];
    pack.slot_start[i] = slots;
    slots += fields[i].seq_len;
  }
  pack.slot_start[nfields] = slots;
  pack.nfields = nfields;
  pack.nslots = slots;
  pack.all_len1 = (slots == nfields) ? 1 : 0;
  pack.pad_ = 0;
}

int64_t count_slots(const b2_field* emb, int nfields) {
  int64_t s = 0;
  for (int i = 0; i < nfields; ++i) s += emb[i].seq_len;
  return s;
}

int check_shard_args(const b2_field* emb, const b2_field* lr, int nfields, int world, int rank) {
  B2_REQUIRE(emb != nullptr, "emb fields is NULL");
  B2_REQUIRE(nfields >= 1 && nfields <= B2_MAX_FIELDS, "nfields=%d outside [1,%d]", nfields, B2_MAX_FIELDS);
  B2_REQUIRE(world >= 1 && world <= 16 && rank >= 0 && rank < world, "bad world/rank %d/%d", world, rank);
  const int dim = emb[0].dim;
  B2_REQUIRE(dim >= 4 && dim <= 128 && dim % 4 == 0, "sharded front needs emb dim %% 4 == 0 and <= 128 (got %d)", dim);
  for (int i = 0; i < nfields; ++i) {
    B2_REQUIRE(emb[i].dim == dim, "field %d: one common dim", i);
    B2_REQUIRE(emb[i].seq_len >= 1 && (emb[i].seq_len == 1 || emb[i].pool == B2_POOL_NONE),
               "field %d: a sequence (seq_len %d) needs pool == B2_POOL_NONE (no pooling across owners)", i,
               emb[i].seq_len);
    B2_REQUIRE(lr == nullptr || emb[i].seq_len == 1, "field %d: LR tables need one slot per field", i);
  }
  B2_REQUIRE(count_slots(emb, nfields) <= (1 << 30), "more than 2^30 slots per sample");
  return B2_OK;
}

template <typename IdxT, bool LAZY, bool RAGGED, typename... Args>
void launch_push_len(bool all_len1, int grid, size_t smem, cudaStream_t st, Args... args) {
  if (all_len1) shard_push_kernel<IdxT, LAZY, true, RAGGED><<<grid, 256, smem, st>>>(args...);
  else shard_push_kernel<IdxT, LAZY, false, RAGGED><<<grid, 256, smem, st>>>(args...);
}

template <typename IdxT, typename... Args>
int launch_push(bool lazy, bool all_len1, int grid, size_t smem, cudaStream_t st, Args... args) {
  const int32_t* no_rows = nullptr;      // the training push serves full batches
  if (lazy) launch_push_len<IdxT, true, false>(all_len1, grid, smem, st, args..., no_rows);
  else launch_push_len<IdxT, false, false>(all_len1, grid, smem, st, args..., no_rows);
  return B2_OK;
}

// The publish launches' destinations and the padding rows this rank owns (both publish entry points).
int publish_setup(int32_t* const* peer_dst, const b2_field* emb_fields, const b2_field* lr_fields, int nfields,
                  int world, int rank, float* const* peer_pad, BcastDst& d, PadDst& pd, PadSrc& ps) {
  int rc = check_shard_args(emb_fields, lr_fields, nfields, world, rank);
  if (rc != B2_OK) return rc;
  for (int i = 0; i < 16; ++i) { d.p[i] = nullptr; pd.p[i] = nullptr; }
  for (int i = 0; i < world; ++i) {
    B2_REQUIRE(peer_dst[i] != nullptr && ((uintptr_t) peer_dst[i] % 16) == 0, "peer_dst[%d] NULL or misaligned", i);
    B2_REQUIRE(peer_pad[i] != nullptr && ((uintptr_t) peer_pad[i] % 16) == 0, "peer_pad[%d] NULL or misaligned", i);
    d.p[i] = peer_dst[i];
    pd.p[i] = peer_pad[i];
  }
  const int dim = emb_fields[0].dim;
  for (int f = 0; f < nfields; ++f) {
    ps.e[f] = nullptr;
    ps.l[f] = nullptr;
    const int64_t pad = emb_fields[f].padding_idx;
    if (pad < 0 || pad >= emb_fields[f].vocab || (int) (pad % world) != rank) continue;     // not mine
    if (emb_fields[f].table != nullptr) ps.e[f] = reinterpret_cast<const float*>(emb_fields[f].table) + (pad / world) * dim;
    if (lr_fields != nullptr) {
      B2_REQUIRE(lr_fields[f].padding_idx == pad, "field %d: the LR and embedding tables need one padding row", f);
      if (lr_fields[f].table != nullptr) ps.l[f] = reinterpret_cast<const float*>(lr_fields[f].table) + pad / world;
    }
  }
  return B2_OK;
}

int check_lazy(const b2_lazy_ctx* lz) {
  if (lz == nullptr) return B2_OK;
  B2_REQUIRE(lz->last_step && lz->sched && lz->step_dev && lz->mark && lz->worklist && lz->counter,
             "lazy context: NULL last_step / sched / step_dev / mark / worklist / counter");
  B2_REQUIRE(lz->worklist_capacity >= 1, "lazy context: worklist_capacity %d", lz->worklist_capacity);
  return B2_OK;
}

// What a shard_push_kernel launch needs beyond the caller's own arguments.
struct PushLaunch {
  const B2FieldPack* epack;
  const B2FieldPack* lpack;
  PeerPtrs pp;
  int dim, lpr_log2, has_lr, grid;
  size_t smem;
};

// The host side shared by the training push and the evaluation lookup (both launch shard_push_kernel): the
// checks of the fields, the peer pointer arrays and the padding rows, then the field packs, the peer buffers, the
// shared memory (both packs and the 256-entry list) and a grid over every candidate of a full batch.
int push_setup(const b2_field* emb_fields, const b2_field* lr_fields, int nfields, int64_t batch_local, int world,
               int rank, const void* const* peer_ids, float* const* peer_emb, float* const* peer_lrw,
               const float* pad_rows, PushLaunch& pl) {
  int rc = check_shard_args(emb_fields, lr_fields, nfields, world, rank);
  if (rc != B2_OK) return rc;
  B2_REQUIRE(peer_ids && peer_emb && (lr_fields == nullptr || peer_lrw != nullptr), "NULL peer pointer array");
  B2_REQUIRE(pad_rows == nullptr || ((uintptr_t) pad_rows % 16) == 0, "pad_rows must be 16-byte aligned");
  if (pad_rows != nullptr && lr_fields != nullptr)
    for (int i = 0; i < nfields; ++i)
      B2_REQUIRE(lr_fields[i].padding_idx == emb_fields[i].padding_idx,
                 "field %d: the LR and embedding tables need one padding row", i);
  const int64_t nslots = count_slots(emb_fields, nfields);
  B2_REQUIRE(batch_local * nslots < (1ll << 31), "batch_local * slots must fit 31 bits");
  static thread_local B2FieldPack epack, lpack;
  fill_pack_cols(epack, emb_fields, nfields);
  pl.has_lr = lr_fields != nullptr;
  if (pl.has_lr) fill_pack_cols(lpack, lr_fields, nfields); else lpack.nfields = 0;
  pl.epack = &epack;
  pl.lpack = &lpack;
  for (int i = 0; i < world; ++i) {
    pl.pp.ids[i] = peer_ids[i];
    pl.pp.emb[i] = peer_emb[i];
    pl.pp.lrw[i] = pl.has_lr ? peer_lrw[i] : nullptr;
    pl.pp.gemb[i] = nullptr;
    pl.pp.glogit[i] = nullptr;
  }
  pl.dim = emb_fields[0].dim;
  pl.lpr_log2 = next_pow2_log2((pl.dim + 3) / 4);
  pl.smem = 2 * ((pack_smem_bytes(nfields) + 15) & ~(size_t) 15) + 256 * sizeof(int4);
  pl.grid = grid_for(batch_local * nslots * world, 256);
  return B2_OK;
}
}  // namespace

extern "C" B2_API int b2_shard_push(const b2_field* emb_fields, const b2_field* lr_fields, int nfields,
                                    int64_t batch_local, int world, int rank, const void* const* peer_ids,
                                    int idx_dtype, int64_t ids_stride, float* const* peer_emb,
                                    float* const* peer_lrw, int32_t* status, int32_t* owned,
                                    int32_t* owned_count, int32_t owned_capacity, const b2_lazy_ctx* lazy,
                                    const float* pad_rows, void* stream) {
  PushLaunch pl;
  int rc = push_setup(emb_fields, lr_fields, nfields, batch_local, world, rank, peer_ids, peer_emb, peer_lrw,
                      pad_rows, pl);
  if (rc != B2_OK) return rc;
  rc = check_lazy(lazy);
  if (rc != B2_OK) return rc;
  B2_REQUIRE(owned == nullptr || (owned_count != nullptr && owned_capacity >= 1), "owned list needs a counter and a capacity");
  B2_REQUIRE(owned == nullptr || ((uintptr_t) owned % 16) == 0, "owned list must be 16-byte aligned");
  cudaStream_t st = (cudaStream_t) stream;
  if (owned != nullptr) {
    cudaError_t e = cudaMemsetAsync(owned_count, 0, sizeof(int32_t), st);
    if (e != cudaSuccess) return b2_fail(B2_E_CUDA, "b2_shard_push: memset: %s", cudaGetErrorString(e));
  }
  if (batch_local <= 0) return B2_OK;
  int4* ow = reinterpret_cast<int4*>(owned);
  static thread_local b2_lazy_ctx lz_none;
  const b2_lazy_ctx& lz = lazy ? *lazy : lz_none;
  const bool len1 = pl.epack->all_len1 != 0;
  switch (idx_dtype) {
    case B2_F64: rc = launch_push<double>(lazy != nullptr, len1, pl.grid, pl.smem, st, *pl.epack, *pl.lpack, pl.pp, lz, batch_local, ids_stride, pl.dim, pl.lpr_log2, pl.has_lr, world, rank, status, ow, owned_count, owned_capacity, pad_rows); break;
    case B2_I64: rc = launch_push<int64_t>(lazy != nullptr, len1, pl.grid, pl.smem, st, *pl.epack, *pl.lpack, pl.pp, lz, batch_local, ids_stride, pl.dim, pl.lpr_log2, pl.has_lr, world, rank, status, ow, owned_count, owned_capacity, pad_rows); break;
    case B2_I32: rc = launch_push<int32_t>(lazy != nullptr, len1, pl.grid, pl.smem, st, *pl.epack, *pl.lpack, pl.pp, lz, batch_local, ids_stride, pl.dim, pl.lpr_log2, pl.has_lr, world, rank, status, ow, owned_count, owned_capacity, pad_rows); break;
    default: return b2_fail(B2_E_INVALID, "idx_dtype %d unsupported", idx_dtype);
  }
  B2_CUDA_LAUNCH_CHECK("b2_shard_push");
  return B2_OK;
}

extern "C" B2_API int b2_shard_pull(const b2_field* emb_fields, const b2_field* lr_fields, int nfields,
                                    int64_t batch_local, int world, int rank, const float* const* peer_gemb,
                                    const float* const* peer_glogit, float scale, const int32_t* owned,
                                    const int32_t* owned_count, int32_t owned_capacity, const b2_lazy_ctx* lazy,
                                    const b2_touch* touch, void* stream) {
  int rc = check_shard_args(emb_fields, lr_fields, nfields, world, rank);
  if (rc != B2_OK) return rc;
  rc = check_lazy(lazy);
  if (rc != B2_OK) return rc;
  b2_touch tch;
  rc = b2_touch_arg(touch, tch);
  if (rc != B2_OK) return rc;
  B2_REQUIRE(peer_gemb && (lr_fields == nullptr || peer_glogit != nullptr), "NULL peer pointer array");
  B2_REQUIRE(owned && owned_count && owned_capacity >= 1 && ((uintptr_t) owned % 16) == 0, "bad owned list");
  if (batch_local <= 0) return B2_OK;
  static thread_local B2FieldPack epack, lpack;
  fill_pack_cols(epack, emb_fields, nfields);
  const int has_lr = lr_fields != nullptr;
  if (has_lr) fill_pack_cols(lpack, lr_fields, nfields); else lpack.nfields = 0;
  PeerPtrs pp;
  for (int i = 0; i < world; ++i) {
    pp.ids[i] = nullptr;
    pp.emb[i] = nullptr;
    pp.lrw[i] = nullptr;
    pp.gemb[i] = peer_gemb[i];
    pp.glogit[i] = has_lr ? peer_glogit[i] : nullptr;
  }
  const int dim = emb_fields[0].dim;
  const int lpr_log2 = next_pow2_log2((dim + 3) / 4);
  const size_t smem = ((pack_smem_bytes(nfields) + 15) & ~(size_t) 15) + pack_smem_bytes(nfields) + 16;
  // the list holds ~batch_local * slots entries on a balanced batch (this rank's share of the global batch)
  int64_t expect = batch_local * (int64_t) epack.nslots * 2;
  if (expect > owned_capacity) expect = owned_capacity;
  const int grid = grid_for(expect << lpr_log2, 256);
  static thread_local b2_lazy_ctx lz_none;
  const b2_lazy_ctx& lz = lazy ? *lazy : lz_none;
  shard_pull_kernel<<<grid, 256, smem, (cudaStream_t) stream>>>(epack, lpack, pp, lz, lazy ? 1 : 0, dim, lpr_log2,
                                                               has_lr, scale, reinterpret_cast<const int4*>(owned),
                                                               owned_count, owned_capacity, tch);
  B2_CUDA_LAUNCH_CHECK("b2_shard_pull");
  return B2_OK;
}

extern "C" B2_API int b2_shard_publish_ids(const void* src, int idx_dtype, int64_t count, int32_t* const* peer_dst,
                                           const b2_field* emb_fields, const b2_field* lr_fields, int nfields,
                                           int world, int rank, float* const* peer_pad, void* stream) {
  B2_REQUIRE(src && peer_dst && peer_pad && count >= 0, "bad argument");
  BcastDst d;
  PadDst pd;
  static thread_local PadSrc ps;
  int rc = publish_setup(peer_dst, emb_fields, lr_fields, nfields, world, rank, peer_pad, d, pd, ps);
  if (rc != B2_OK) return rc;
  const int dim = emb_fields[0].dim;
  const int64_t npad = (int64_t) nfields * (dim + 1);
  const int grid = grid_for((count >> 2) > npad ? (count >> 2) : npad, 256);
  cudaStream_t st = (cudaStream_t) stream;
  switch (idx_dtype) {
    case B2_F64: shard_publish_ids_kernel<double><<<grid, 256, 0, st>>>(src, count, d, world, ps, pd, nfields, dim); break;
    case B2_I64: shard_publish_ids_kernel<int64_t><<<grid, 256, 0, st>>>(src, count, d, world, ps, pd, nfields, dim); break;
    case B2_I32: shard_publish_ids_kernel<int32_t><<<grid, 256, 0, st>>>(src, count, d, world, ps, pd, nfields, dim); break;
    default: return b2_fail(B2_E_INVALID, "idx_dtype %d unsupported", idx_dtype);
  }
  B2_CUDA_LAUNCH_CHECK("b2_shard_publish_ids");
  return B2_OK;
}

extern "C" B2_API int b2_shard_publish_rows(const void* src, int idx_dtype, int64_t rows, int64_t width,
                                            int64_t capacity_rows, int32_t* const* peer_dst,
                                            const b2_field* emb_fields, const b2_field* lr_fields, int nfields,
                                            int world, int rank, float* const* peer_pad, int32_t* const* peer_rows,
                                            void* stream) {
  B2_REQUIRE(peer_dst && peer_pad && peer_rows, "NULL peer pointer array");
  B2_REQUIRE(capacity_rows >= 0 && capacity_rows < (1ll << 31), "capacity_rows %lld outside [0, 2^31)",
             (long long) capacity_rows);
  B2_REQUIRE(rows >= 0 && rows <= capacity_rows, "rows %lld outside [0, capacity_rows = %lld]", (long long) rows,
             (long long) capacity_rows);
  B2_REQUIRE(width >= 1, "width %lld < 1", (long long) width);
  B2_REQUIRE(src != nullptr || rows == 0, "src is NULL");
  BcastDst d;
  PadDst pd;
  RowsDst rd;
  static thread_local PadSrc ps;
  int rc = publish_setup(peer_dst, emb_fields, lr_fields, nfields, world, rank, peer_pad, d, pd, ps);
  if (rc != B2_OK) return rc;
  for (int i = 0; i < 16; ++i) rd.p[i] = nullptr;
  for (int i = 0; i < world; ++i) {
    B2_REQUIRE(peer_rows[i] != nullptr && ((uintptr_t) peer_rows[i] % 4) == 0, "peer_rows[%d] NULL or misaligned", i);
    rd.p[i] = peer_rows[i];
  }
  const int dim = emb_fields[0].dim;
  const int64_t count = rows * width;
  const int64_t npad = (int64_t) nfields * (dim + 1);
  const int grid = grid_for((count >> 2) > npad ? (count >> 2) : npad, 256);
  cudaStream_t st = (cudaStream_t) stream;
  const int32_t r32 = (int32_t) rows;
  switch (idx_dtype) {
    case B2_F64: shard_publish_rows_kernel<double><<<grid, 256, 0, st>>>(src, count, d, world, ps, pd, nfields, dim, rd, rank, r32); break;
    case B2_I64: shard_publish_rows_kernel<int64_t><<<grid, 256, 0, st>>>(src, count, d, world, ps, pd, nfields, dim, rd, rank, r32); break;
    case B2_I32: shard_publish_rows_kernel<int32_t><<<grid, 256, 0, st>>>(src, count, d, world, ps, pd, nfields, dim, rd, rank, r32); break;
    default: return b2_fail(B2_E_INVALID, "idx_dtype %d unsupported", idx_dtype);
  }
  B2_CUDA_LAUNCH_CHECK("b2_shard_publish_rows");
  return B2_OK;
}

extern "C" B2_API int b2_shard_lookup(const b2_field* emb_fields, const b2_field* lr_fields, int nfields,
                                      int64_t batch_local, int world, int rank, const int32_t* const* peer_ids,
                                      int64_t ids_stride, float* const* peer_emb, float* const* peer_lrw,
                                      const int32_t* rows_all, int32_t* status, const float* pad_rows, void* stream) {
  B2_REQUIRE(rows_all != nullptr, "rows_all is NULL");
  B2_REQUIRE(batch_local >= 0, "batch_local %lld < 0", (long long) batch_local);
  B2_REQUIRE(ids_stride >= 1, "ids_stride %lld < 1", (long long) ids_stride);
  PushLaunch pl;
  int rc = push_setup(emb_fields, lr_fields, nfields, batch_local, world, rank,
                      reinterpret_cast<const void* const*>(peer_ids), peer_emb, peer_lrw, pad_rows, pl);
  if (rc != B2_OK) return rc;
  for (int i = 0; i < world; ++i)
    B2_REQUIRE(peer_ids[i] && peer_emb[i] && (lr_fields == nullptr || peer_lrw[i]), "peer %d: NULL buffer", i);
  if (batch_local == 0) return B2_OK;
  // the grid covers every candidate of a full round; the samples past rows_all[p] drop out in the scan
  static thread_local b2_lazy_ctx lz_none;
  launch_push_len<int32_t, false, true>(pl.epack->all_len1 != 0, pl.grid, pl.smem, (cudaStream_t) stream, *pl.epack,
                                        *pl.lpack, pl.pp, lz_none, batch_local, ids_stride, pl.dim, pl.lpr_log2,
                                        pl.has_lr, world, rank, status, (int4*) nullptr, (int32_t*) nullptr,
                                        (int32_t) 0, pad_rows, rows_all);
  B2_CUDA_LAUNCH_CHECK("b2_shard_lookup");
  return B2_OK;
}

extern "C" B2_API int b2_front_reduce(const float* emb, const float* lrw, const float* bias, int64_t batch,
                                      int nfields, int dim, int want_fm, float* logit, float* sums,
                                      void* stream) {
  B2_REQUIRE(emb && logit, "NULL pointer");
  B2_REQUIRE(dim >= 4 && dim <= 128 && dim % 4 == 0 && nfields >= 1, "bad dim/nfields");
  B2_REQUIRE(!want_fm || sums != nullptr, "want_fm needs sums");
  if (batch <= 0) return B2_OK;
  const int lpr_log2 = next_pow2_log2((dim + 3) / 4);
  const int grid = grid_for(batch * 32, 256);
  front_reduce_kernel<<<grid, 256, 0, (cudaStream_t) stream>>>(emb, lrw, bias, batch, nfields, dim, lpr_log2,
                                                              want_fm, logit, sums);
  B2_CUDA_LAUNCH_CHECK("b2_front_reduce");
  return B2_OK;
}

extern "C" B2_API int b2_front_gprep(const float* gx, const float* emb, const float* sums, const float* glogit,
                                     int64_t batch, int nfields, int dim, int want_fm, float* gemb,
                                     float* glogit_out, float* gbias, int gbias_is_zero, void* stream) {
  B2_REQUIRE(gemb != nullptr, "NULL output");
  B2_REQUIRE((glogit_out == nullptr && gbias == nullptr) || glogit != nullptr, "glogit_out / gbias need glogit");
  if (gbias != nullptr && !gbias_is_zero) {
    cudaError_t e = cudaMemsetAsync(gbias, 0, sizeof(float), (cudaStream_t) stream);
    if (e != cudaSuccess) return b2_fail(B2_E_CUDA, "b2_front_gprep: memset: %s", cudaGetErrorString(e));
  }
  B2_REQUIRE(dim >= 4 && dim % 4 == 0 && nfields >= 1, "bad dim/nfields");
  B2_REQUIRE(!want_fm || (emb && sums && glogit), "want_fm needs emb, sums, glogit");
  if (batch <= 0) return B2_OK;
  const int64_t n4 = batch * (int64_t) nfields * dim / 4;
  const int grid = grid_for(n4, 256);
  front_gprep_kernel<<<grid, 256, 0, (cudaStream_t) stream>>>(gx, emb, sums, glogit, batch, nfields, dim, want_fm, gemb,
                                                             glogit_out, gbias);
  B2_CUDA_LAUNCH_CHECK("b2_front_gprep");
  return B2_OK;
}

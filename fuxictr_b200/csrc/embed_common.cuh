// embed_common.cuh — launch pack, shared-memory staging and vector helpers shared by the
// embedding kernels (embed.cu, fused_front.cu).
#pragma once
#include "b2_common.cuh"

struct B2FieldPack {
  b2_field f[B2_MAX_FIELDS];
  int32_t slot_start[B2_MAX_FIELDS + 1];  // prefix sum of slots per field
  int32_t nfields;
  int32_t nslots;
  int32_t all_len1;  // every field has exactly one slot
  int32_t pad_;
};

// Shared-memory image of the pack, trimmed to nfields.
struct SmemFields {
  b2_field* f;
  int32_t* slot_start;
};

__device__ __forceinline__ SmemFields b2_stage_fields(const B2FieldPack& pack, unsigned char* smem) {
  SmemFields s;
  s.f = reinterpret_cast<b2_field*>(smem);
  s.slot_start = reinterpret_cast<int32_t*>(smem + sizeof(b2_field) * pack.nfields);
  const int nwords = (int) (sizeof(b2_field) / 4) * pack.nfields;
  const uint32_t* src = reinterpret_cast<const uint32_t*>(&pack.f[0]);
  uint32_t* dst = reinterpret_cast<uint32_t*>(smem);
  for (int i = threadIdx.x; i < nwords; i += blockDim.x) dst[i] = src[i];
  for (int i = threadIdx.x; i <= pack.nfields; i += blockDim.x) s.slot_start[i] = pack.slot_start[i];
  __syncthreads();
  return s;
}

// slot -> field by binary search over the prefix sums (<= 7 steps).
__device__ __forceinline__ int b2_slot_field(const int32_t* slot_start, int nfields, int slot) {
  int lo = 0, hi = nfields;  // invariant: slot_start[lo] <= slot < slot_start[hi]
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (slot_start[mid] <= slot) lo = mid; else hi = mid;
  }
  return lo;
}

template <int VEC> struct VecT;
template <> struct VecT<4> { using type = float4; };
template <> struct VecT<2> { using type = float2; };
template <> struct VecT<1> { using type = float; };

template <int VEC>
__device__ __forceinline__ typename VecT<VEC>::type b2_vzero();
template <> __device__ __forceinline__ float4 b2_vzero<4>() { return make_float4(0.f, 0.f, 0.f, 0.f); }
template <> __device__ __forceinline__ float2 b2_vzero<2>() { return make_float2(0.f, 0.f); }
template <> __device__ __forceinline__ float b2_vzero<1>() { return 0.f; }

__device__ __forceinline__ void b2_vadd(float4& a, const float4& b) { a.x += b.x; a.y += b.y; a.z += b.z; a.w += b.w; }
__device__ __forceinline__ void b2_vadd(float2& a, const float2& b) { a.x += b.x; a.y += b.y; }
__device__ __forceinline__ void b2_vadd(float& a, const float& b) { a += b; }
__device__ __forceinline__ float b2_vsum(const float4& a) { return (a.x + a.y) + (a.z + a.w); }
__device__ __forceinline__ float b2_vsum(const float2& a) { return a.x + a.y; }
__device__ __forceinline__ float b2_vsum(const float& a) { return a; }
__device__ __forceinline__ float4 b2_vscale(const float4& a, float s) { return make_float4(a.x * s, a.y * s, a.z * s, a.w * s); }
__device__ __forceinline__ float2 b2_vscale(const float2& a, float s) { return make_float2(a.x * s, a.y * s); }
__device__ __forceinline__ float b2_vscale(const float& a, float s) { return a * s; }
__device__ __forceinline__ float4 b2_vdiv(const float4& a, float s) { return make_float4(a.x / s, a.y / s, a.z / s, a.w / s); }
__device__ __forceinline__ float2 b2_vdiv(const float2& a, float s) { return make_float2(a.x / s, a.y / s); }
__device__ __forceinline__ float b2_vdiv(const float& a, float s) { return a / s; }

__device__ __forceinline__ void b2_vred(float* p, const float4& v) { b2_red_add_v4(p, v); }
__device__ __forceinline__ void b2_vred(float* p, const float2& v) { b2_red_add_v2(p, v.x, v.y); }
__device__ __forceinline__ void b2_vred(float* p, const float& v) { b2_red_add(p, v); }


// ---------------------------------------------------------------------------------
// Host-side helpers
// ---------------------------------------------------------------------------------
static inline int next_pow2_log2(int v) {
  int l = 0;
  while ((1 << l) < v) ++l;
  return l;
}

// Builds the launch pack; `bwd_slots` = one slot per (field, position) even for pooled fields.
static inline int build_pack(B2FieldPack& pack, const b2_field* fields, int nfields, bool bwd_slots,
                      bool need_out, int* vec_out, int* max_dim_out, bool* any_pooled_out) {
  B2_REQUIRE(fields != nullptr, "fields is NULL");
  B2_REQUIRE(nfields >= 1 && nfields <= B2_MAX_FIELDS, "nfields=%d outside [1,%d]", nfields,
             B2_MAX_FIELDS);
  int vec = 4, max_dim = 1;
  bool any_pooled = false;
  int slots = 0;
  for (int i = 0; i < nfields; ++i) {
    const b2_field& f = fields[i];
    B2_REQUIRE(f.table != nullptr && f.idx != nullptr, "field %d: NULL table or idx", i);
    B2_REQUIRE(!need_out || f.out != nullptr, "field %d: NULL out", i);
    B2_REQUIRE(f.dim >= 1 && f.seq_len >= 1 && f.vocab >= 1, "field %d: bad dim/seq_len/vocab", i);
    B2_REQUIRE(f.pool >= B2_POOL_NONE && f.pool <= B2_POOL_MEAN, "field %d: bad pool mode", i);
    const bool pooled = f.seq_len > 1 && f.pool != B2_POOL_NONE;
    any_pooled |= pooled;
    pack.f[i] = f;
    pack.slot_start[i] = slots;
    slots += (pooled && !bwd_slots) ? 1 : f.seq_len;
    if (f.dim > max_dim) max_dim = f.dim;
    if (need_out) {
      // widest vector every row start of this field is aligned to
      int v = 4;
      while (v > 1 && ((f.dim % v) != 0 || (f.out_stride % v) != 0 ||
                       ((uintptr_t) f.table % (v * 4)) != 0 || ((uintptr_t) f.out % (v * 4)) != 0))
        v >>= 1;
      if (v < vec) vec = v;
    }
  }
  pack.slot_start[nfields] = slots;
  pack.nfields = nfields;
  pack.nslots = slots;
  pack.all_len1 = (slots == nfields) ? 1 : 0;
  pack.pad_ = 0;
  if (vec_out) *vec_out = vec;
  if (max_dim_out) *max_dim_out = max_dim;
  if (any_pooled_out) *any_pooled_out = any_pooled;
  return B2_OK;
}

__host__ __device__ static inline size_t pack_smem_bytes(int nfields) {
  return sizeof(b2_field) * nfields + sizeof(int32_t) * (nfields + 1);
}

// Grid sized in whole waves of B2_NUM_SMS (132) SMs x 8 resident 256-thread CTAs, capped by the work.
static inline int grid_for(int64_t nthreads_needed, int block) {
  int64_t blocks = b2_ceil_div(nthreads_needed, block);
  const int64_t wave = (int64_t) B2_NUM_SMS * 8;
  if (blocks > wave) blocks = wave;
  if (blocks < 1) blocks = 1;
  return (int) blocks;
}

// The touched-granule descriptor a backward launch takes by value (b2_touch); NULL = one that marks nothing.
static inline int b2_touch_arg(const b2_touch* touch, b2_touch& out) {
  out = b2_touch{nullptr, nullptr, 0};
  if (touch == nullptr || touch->flags == nullptr || touch->n <= 0) return B2_OK;
  B2_REQUIRE(touch->base != nullptr && ((uintptr_t) touch->base % 16) == 0, "touch: base must be 16-byte aligned");
  out = *touch;
  return B2_OK;
}


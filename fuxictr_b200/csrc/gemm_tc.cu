// gemm_tc.cu — TMA-fed wgmma (Hopper tensor core) GEMM with register accumulators and a fused
// epilogue, sm_90a.  The dense contraction behind MLP_Block
// (fuxictr/pytorch/layers/blocks/mlp_block.py:74-85), CrossNetV2's d x d Linear
// (fuxictr/pytorch/layers/interactions/cross_net.py:126-129) and CIN's 1x1 Conv1d
// (fuxictr/pytorch/layers/interactions/compressed_interaction_net.py:72).
//
//   C[m, n] = epi( sum_k A(m, k) * B(n, k) )
// Each operand is either K-major (memory (rows, K), K contiguous) or MN-major (memory (K, rows),
// rows contiguous).  TMA copies both exactly as they lie in memory, so the dgrad (dX = dZ W) and wgrad
// (dW = dZ^T X) contractions of a Linear layer need no transpose pass in HBM.
//
// Arithmetic: wgmma .tf32 on fp32 operands, fp32 accumulation in registers.
//   precision 1 ("tf32"):   one pass on big(x) = x with the 13 low mantissa bits cleared, ~1e-3 relative.
//   precision 3 ("tf32x3"): error-compensated 3xTF32: with x = big(x) + small(x),
//        A.B ~= A_big.B_big + A_big.B_small + A_small.B_big
//     where small = rna_tf32(x - big(x)) — fp32-class accuracy (the 1e-5 parity bar) on tensor cores.  The
//     main product of every k-block is accumulated from zero and added to the running sum in fp32
//     round-to-nearest, so the error does not grow with the length of the contraction.
//   bf16 operands (elem_dtype B2_BF16): wgmma .bf16, 64-element k-blocks, fp32 accumulation.
//
// Structure (one CTA per 128 x BN output tile and K split; 384 threads):
//   warpgroup 0    thread 0 issues cp.async.bulk.tensor loads of the raw operand tiles into a 3-stage
//                  mbarrier ring; the whole warpgroup converts each raw tile (either major, fp32 or bf16)
//                  into the K-major 128B-swizzled tiles wgmma reads — big and small parts for 3xTF32 —
//                  in a second 3-stage ring.  wgmma reads tf32 operands from shared memory only in K-major
//                  form, so this pass is what lets MN-major operands stay as they lie in HBM.
//   warpgroups 1-2 64 rows each: wgmma m64nBNk8 (tf32) / k16 (bf16) from the converted tiles, then the fused
//                  epilogue straight from the accumulator registers (each quad of lanes writes 32 contiguous
//                  bytes of one output row).
// Kernels of a step are chained with programmatic dependent launch (prologue under the predecessor's tail).
// Every mbarrier wait is bounded: a pipeline bug traps with a message instead of hanging the GPU.
#include "b2_common.cuh"
#include <string.h>
#include <cstdlib>
#include <cuda.h>  // CUtensorMap + enums only; cuTensorMapEncodeTiled is resolved at run time

namespace tc {
constexpr int BM = 128;          // two consumer warpgroups x wgmma M = 64
constexpr int NTHREADS = 384;    // converter warpgroup + two wgmma warpgroups
constexpr int RSTAGES = 3;       // raw TMA tiles in flight
constexpr int CSTAGES = 3;       // converted tiles in flight

struct Params {
  CUtensorMap map_a;
  CUtensorMap map_b;
  float* c;
  float* c_small;         // optional: tf32_small(C) (or the bf16 copy of C) for the consumer's operand
  float* c_pre;           // optional: acc + bias BEFORE mul/add/act (CrossNetV2 saves it for its backward)
  int64_t ldc;
  const float* bias;
  const float* mul;
  const float* add;
  const float* ybwd;      // optional (M, N) ld = ldc: C = act_bwd'(ybwd) * (...)   (activation backward)
  float* colsum;          // optional (N): += column sums of C (bias gradient)
  int M, N, K, act, act_bwd, beta, kb_per_split;
  int a_mn, b_mn;         // operand is MN-major (memory (K, rows))
  int esz;                // operand element bytes: 4 = fp32 (tf32 passes), 2 = bf16
  int64_t ld_aux;         // leading dimension of c_small
  int tiles_m, tiles_n, splits;
};

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return (uint32_t) __cvta_generic_to_shared(p);
}
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
      "selp.u32 %0, 1, 0, p;\n"
      "}\n"
      : "=r"(ok)
      : "r"(bar), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded wait: ~2 s at 2 GHz, then report and trap (never hang the device).
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity, int which) {
  if (mbar_try_wait(bar, parity)) return;
  const long long t0 = clock64();
  while (!mbar_try_wait(bar, parity)) {
    if (clock64() - t0 > 4000000000LL) {
      printf("b2 tc_gemm: mbarrier wait timed out (role %d, block %d,%d,%d)\n", which, blockIdx.x,
             blockIdx.y, blockIdx.z);
      __trap();
    }
  }
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* map, uint32_t bar,
                                            int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
      ::"r"(dst), "l"(reinterpret_cast<uint64_t>(map)), "r"(c0), "r"(c1), "r"(bar)
      : "memory");
}
// wgmma shared-memory matrix descriptor of a K-major, 128B-swizzled tile: rows 128 B apart, 8-row swizzle
// atoms 1024 B apart (SBO); the leading byte offset is unused for swizzled K-major layouts.
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t addr) {
  uint64_t d = 0;
  d |= (uint64_t) ((addr & 0x3FFFFu) >> 4);  // start address  [0,14)
  d |= (uint64_t) 1 << 16;                   // leading byte offset [16,30)
  d |= (uint64_t) (1024 >> 4) << 32;         // stride byte offset [32,46)
  d |= (uint64_t) 1 << 62;                   // layout: SWIZZLE_128B
  return d;
}
// Byte offset of 16-byte chunk `c` (0..7) of row `r` in a K-major 128B-swizzled tile (1024-byte aligned base).
__device__ __forceinline__ uint32_t swz(int r, int c) { return (uint32_t) (r * 128 + ((c ^ (r & 7)) << 4)); }
__device__ __forceinline__ float tf32_small(float v) { return b2_tf32_small(v); }
__device__ __forceinline__ float tf32_big(float v) { return __uint_as_float(__float_as_uint(v) & 0xffffe000u); }
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait0() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }

// wgmma.mma_async m64nNk8 (tf32) / m64nNk16 (bf16), both operands from shared memory, fp32 accumulators
// d[] in the wgmma fragment layout; scale_d == 0 overwrites the accumulators.
__device__ __forceinline__ void wgmma_tf32(float (&d)[16], uint64_t a, uint64_t b, uint32_t scale_d) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %18, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(a), "l"(b), "r"(scale_d));
}
__device__ __forceinline__ void wgmma_tf32(float (&d)[32], uint64_t a, uint64_t b, uint32_t scale_d) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(a), "l"(b), "r"(scale_d));
}
__device__ __forceinline__ void wgmma_tf32(float (&d)[64], uint64_t a, uint64_t b, uint32_t scale_d) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(a), "l"(b), "r"(scale_d));
}
__device__ __forceinline__ void wgmma_bf16(float (&d)[16], uint64_t a, uint64_t b, uint32_t scale_d) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %18, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, 0, 0;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(a), "l"(b), "r"(scale_d));
}
__device__ __forceinline__ void wgmma_bf16(float (&d)[32], uint64_t a, uint64_t b, uint32_t scale_d) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(a), "l"(b), "r"(scale_d));
}
__device__ __forceinline__ void wgmma_bf16(float (&d)[64], uint64_t a, uint64_t b, uint32_t scale_d) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 0;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(a), "l"(b), "r"(scale_d));
}

// 16 bytes of K-major fp32 operand -> the converted tile: big part (13 low mantissa bits cleared) and, for
// 3xTF32, the small part at the same offset in the small tile.
template <bool X3>
__device__ __forceinline__ void store_split(uint8_t* dst, uint32_t small_off, uint32_t off, const float4& v) {
  *reinterpret_cast<float4*>(dst + off) = make_float4(tf32_big(v.x), tf32_big(v.y), tf32_big(v.z), tf32_big(v.w));
  if (X3)
    *reinterpret_cast<float4*>(dst + small_off + off) =
        make_float4(tf32_small(v.x), tf32_small(v.y), tf32_small(v.z), tf32_small(v.w));
}

// One operand's k-block as TMA wrote it -> K-major 128B-swizzled tile of `rows` rows, by the 128 threads of
// the converter warpgroup.  Raw layouts: K-major (rows, 128 B of k); MN-major (k, rows): 32 fp32 or 64 bf16
// k-rows of `rows` elements, transposed here in registers (4 x 4 fp32 or 8 x 8 bf16 per thread).
template <bool X3>
__device__ __forceinline__ void convert_tile(const uint8_t* src, uint8_t* dst, uint32_t small_off, int rows, int mn,
                                             int esz, int ct) {
  if (esz == 2) {
    if (!mn) {
      for (int q = ct; q < rows * 8; q += 128)
        *reinterpret_cast<uint4*>(dst + swz(q >> 3, q & 7)) = *reinterpret_cast<const uint4*>(src + 16 * q);
    } else {
      for (int b = ct; b < rows; b += 128) {
        const int kq = b & 7, r0 = (b >> 3) * 8;
        uint4 v[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] = *reinterpret_cast<const uint4*>(src + ((8 * kq + j) * rows + r0) * 2);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          uint32_t w[4];
#pragma unroll
          for (int j = 0; j < 8; j += 2) {
            const uint32_t lo = reinterpret_cast<const uint16_t*>(&v[j])[i];
            const uint32_t hi = reinterpret_cast<const uint16_t*>(&v[j + 1])[i];
            w[j >> 1] = lo | (hi << 16);
          }
          *reinterpret_cast<uint4*>(dst + swz(r0 + i, kq)) = make_uint4(w[0], w[1], w[2], w[3]);
        }
      }
    }
    return;
  }
  if (!mn) {
    for (int q = ct; q < rows * 8; q += 128)
      store_split<X3>(dst, small_off, swz(q >> 3, q & 7), *reinterpret_cast<const float4*>(src + 16 * q));
  } else {
    for (int b = ct; b < 2 * rows; b += 128) {
      const int kq = b & 7, r0 = (b >> 3) * 4;
      float4 v[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) v[j] = *reinterpret_cast<const float4*>(src + ((4 * kq + j) * rows + r0) * 4);
      store_split<X3>(dst, small_off, swz(r0 + 0, kq), make_float4(v[0].x, v[1].x, v[2].x, v[3].x));
      store_split<X3>(dst, small_off, swz(r0 + 1, kq), make_float4(v[0].y, v[1].y, v[2].y, v[3].y));
      store_split<X3>(dst, small_off, swz(r0 + 2, kq), make_float4(v[0].z, v[1].z, v[2].z, v[3].z));
      store_split<X3>(dst, small_off, swz(r0 + 3, kq), make_float4(v[0].w, v[1].w, v[2].w, v[3].w));
    }
  }
}

// One output element (m, n) of the fused epilogue, t = accumulator + bias; returns what enters the column sum.
__device__ __forceinline__ float epilogue_elem(const Params& p, int m, int n, float t) {
  const int64_t o = (int64_t) m * p.ldc + n;
  if (p.splits > 1) {          // split-K: partial sums of a plain linear output (C was zeroed by the host)
    b2_red_add(p.c + o, t);
    return 0.f;
  }
  if (p.c_pre != nullptr) p.c_pre[o] = t;
  if (p.mul != nullptr) t *= __ldg(p.mul + o);
  if (p.add != nullptr) t += __ldg(p.add + o);
  if (p.act == B2_ACT_RELU) t = fmaxf(t, 0.f);
  else if (p.act == B2_ACT_SIGMOID) t = 1.f / (1.f + expf(-t));
  if (p.ybwd != nullptr) {     // activation backward of the PRODUCER of this gradient, fused
    const float yv = __ldg(p.ybwd + o);
    if (p.act_bwd == B2_ACT_RELU) t = (yv > 0.f) ? t : 0.f;
    else if (p.act_bwd == B2_ACT_SIGMOID) t = t * ((1.f - yv) * yv);
  }
  if (p.beta) t += p.c[o];
  p.c[o] = t;
  if (p.c_small != nullptr) {
    const int64_t oa = (int64_t) m * p.ld_aux + n;
    if (p.esz == 4) p.c_small[oa] = tf32_small(t);   // the consumer's 3xTF32 small part, produced where C is
    else reinterpret_cast<__nv_bfloat16*>(p.c_small)[oa] = __float2bfloat16_rn(t);   // bf16 mode operand
  }
  return t;
}

template <int BN, bool X3>
__global__ void __launch_bounds__(NTHREADS, 1)
gemm_tc_kernel(const __grid_constant__ Params p) {
  constexpr int NR = BN / 2;                            // accumulators per thread: 64 x BN per warpgroup
  constexpr uint32_t TILE_BYTES = (BM + BN) * 128;      // one k-block of A and B (raw, or converted big part)
  constexpr uint32_t CONV_BYTES = (X3 ? 2 : 1) * TILE_BYTES;
  extern __shared__ uint8_t smem_raw[];
  // 128B-swizzled tiles need 1024-byte aligned bases: align by hand (1 KB of slack is requested).
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t* raw0 = smem;
  uint8_t* conv0 = smem + RSTAGES * TILE_BYTES;
  uint64_t* bars = reinterpret_cast<uint64_t*>(conv0 + CSTAGES * CONV_BYTES);
  const uint32_t rfull0 = smem_u32(bars), cfull0 = smem_u32(bars + RSTAGES),
                 cempty0 = smem_u32(bars + RSTAGES + CSTAGES);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int bke = 128 / p.esz;                      // k elements per k-block: one 128-byte swizzle row
  const int num_kb_total = (p.K + bke - 1) / bke;
  const int tiles_mn = p.tiles_m * p.tiles_n;
  const int z = blockIdx.x / tiles_mn, rr = blockIdx.x - z * tiles_mn;
  const int m0 = (rr / p.tiles_n) * BM, n0 = (rr % p.tiles_n) * BN;
  const int kb_begin = z * p.kb_per_split;
  const int nkb = min(num_kb_total, kb_begin + p.kb_per_split) - kb_begin;

  if (threadIdx.x == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&p.map_a)) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&p.map_b)) : "memory");
    for (int s = 0; s < RSTAGES; ++s) mbar_init(rfull0 + 8 * s, 1);
    for (int s = 0; s < CSTAGES; ++s) {
      mbar_init(cfull0 + 8 * s, 4);      // one arrival per converter warp
      mbar_init(cempty0 + 8 * s, 8);     // one arrival per consumer warp
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  __syncthreads();
  // PDL: everything above touched only shared memory and the kernel parameters; from here on the
  // predecessor's outputs are read.  Let the successor begin ITS prologue once every CTA got this far.
  b2_pdl_trigger();
  b2_pdl_wait();

  if (warp < 4) {
    // ---------------- warpgroup 0: TMA (thread 0) and operand conversion ----------------
    const int ct = threadIdx.x;
    auto load = [&](int i) {
      const int s = i % RSTAGES, kb = kb_begin + i;
      const uint32_t dst = smem_u32(raw0 + s * TILE_BYTES), bar = rfull0 + 8 * s;
      mbar_expect_tx(bar, TILE_BYTES);   // out-of-range parts of a box arrive zero-filled and count in full
      if (p.a_mn) tma_load_2d(dst, &p.map_a, bar, m0, kb * bke);
      else tma_load_2d(dst, &p.map_a, bar, kb * bke, m0);
      if (p.b_mn) tma_load_2d(dst + BM * 128, &p.map_b, bar, n0, kb * bke);
      else tma_load_2d(dst + BM * 128, &p.map_b, bar, kb * bke, n0);
    };
    if (ct == 0)
      for (int i = 0; i < RSTAGES && i < nkb; ++i) load(i);
    for (int i = 0; i < nkb; ++i) {
      const int rs = i % RSTAGES, cs = i % CSTAGES;
      mbar_wait(rfull0 + 8 * rs, (uint32_t) (i / RSTAGES) & 1u, 0);
      mbar_wait(cempty0 + 8 * cs, ((uint32_t) (i / CSTAGES) & 1u) ^ 1u, 1);
      const uint8_t* src = raw0 + rs * TILE_BYTES;
      uint8_t* dst = conv0 + cs * CONV_BYTES;
      convert_tile<X3>(src, dst, TILE_BYTES, BM, p.a_mn, p.esz, ct);
      convert_tile<X3>(src + BM * 128, dst + BM * 128, TILE_BYTES, BN, p.b_mn, p.esz, ct);
      // generic-proxy stores -> visible to wgmma (async proxy) before the consumers are told
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
      __syncwarp();
      if (lane == 0) mbar_arrive(cfull0 + 8 * cs);
      asm volatile("bar.sync 1, 128;" ::: "memory");   // every converter thread is done with raw stage rs
      if (ct == 0 && i + RSTAGES < nkb) load(i + RSTAGES);
    }
  } else {
    // ---------------- warpgroups 1-2: wgmma on rows 64 g .. 64 g + 63 of the tile, then the epilogue ----------
    const int g = (warp >> 2) - 1;
    float acc[NR];
    float part[X3 ? NR : 1], corr[X3 ? NR : 1];
#pragma unroll
    for (int r = 0; r < NR; ++r) acc[r] = 0.f;
#pragma unroll
    for (int r = 0; r < (X3 ? NR : 1); ++r) { part[r] = 0.f; corr[r] = 0.f; }
    for (int i = 0; i < nkb; ++i) {
      const int cs = i % CSTAGES;
      mbar_wait(cfull0 + 8 * cs, (uint32_t) (i / CSTAGES) & 1u, 2);
      const uint32_t base = smem_u32(conv0 + cs * CONV_BYTES);
      // one instruction consumes 32 bytes of K per row (8 tf32 / 16 bf16): +2 in the (addr >> 4) field
      const uint64_t ad = make_smem_desc(base + g * 64 * 128), bd = make_smem_desc(base + BM * 128);
      wgmma_fence();
      if constexpr (X3) {
        const uint64_t asd = ad + (TILE_BYTES >> 4), bsd = bd + (TILE_BYTES >> 4);
#pragma unroll
        for (int k = 0; k < 4; ++k) wgmma_tf32(part, ad + 2 * k, bd + 2 * k, k > 0 ? 1u : 0u);   // A_big . B_big
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          wgmma_tf32(corr, ad + 2 * k, bsd + 2 * k, (i > 0 || k > 0) ? 1u : 0u);                  // A_big . B_small
          wgmma_tf32(corr, asd + 2 * k, bd + 2 * k, 1u);                                         // A_small . B_big
        }
      } else {
        if (p.esz == 2) {
#pragma unroll
          for (int k = 0; k < 4; ++k) wgmma_bf16(acc, ad + 2 * k, bd + 2 * k, (i > 0 || k > 0) ? 1u : 0u);
        } else {
#pragma unroll
          for (int k = 0; k < 4; ++k) wgmma_tf32(acc, ad + 2 * k, bd + 2 * k, (i > 0 || k > 0) ? 1u : 0u);
        }
      }
      wgmma_commit();
      wgmma_wait0();
      __syncwarp();
      if (lane == 0) mbar_arrive(cempty0 + 8 * cs);     // the converted stage may be overwritten
      if constexpr (X3) {
#pragma unroll
        for (int r = 0; r < NR; ++r) acc[r] += part[r];   // this k-block's main product, fp32 round-to-nearest
      }
    }
    if constexpr (X3) {
#pragma unroll
      for (int r = 0; r < NR; ++r) acc[r] += corr[r];
    }
    // wgmma fragment: d[4j + 2h + e] is row 16 w + lane / 4 + 8 h, column 8 j + 2 (lane % 4) + e of the warpgroup
    const int row0 = m0 + g * 64 + (warp & 3) * 16 + (lane >> 2);
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int n = n0 + 8 * j + 2 * (lane & 3) + e;
        const bool n_ok = n < p.N;
        const float bv = (n_ok && p.bias != nullptr && z == 0) ? __ldg(p.bias + n) : 0.f;
        float cs = 0.f;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int m = row0 + 8 * h;
          if (n_ok && m < p.M) cs += epilogue_elem(p, m, n, acc[4 * j + 2 * h + e] + bv);
        }
        if (p.colsum != nullptr) {    // bias gradient: the 8 lanes of one column, then one red.add per warp
          cs += __shfl_xor_sync(0xffffffffu, cs, 4);
          cs += __shfl_xor_sync(0xffffffffu, cs, 8);
          cs += __shfl_xor_sync(0xffffffffu, cs, 16);
          if (lane < 4 && n_ok) b2_red_add(p.colsum + n, cs);
        }
      }
    }
  }
}

__global__ void __launch_bounds__(256)
split_tf32_kernel(const float* __restrict__ x, float* __restrict__ small, int64_t n) {
  b2_pdl_wait();
  b2_pdl_trigger();
  for (int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (int64_t) gridDim.x * blockDim.x) {
    small[i] = tf32_small(x[i]);
  }
}

// out (cols, rows) = in (rows, cols)^T through a padded shared tile; optionally also the
// small() part of the transposed values (for the 3xTF32 operands of dgrad / wgrad).
__global__ void __launch_bounds__(256)
transpose_kernel(const float* __restrict__ in, int64_t rows, int64_t cols, int64_t ld_in,
                 float* __restrict__ out, int64_t ld_out, float* __restrict__ out_small) {
  __shared__ float tile[32][33];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;  // 32 x 8
  const int64_t c0 = (int64_t) blockIdx.x * 32, r0 = (int64_t) blockIdx.y * 32;
#pragma unroll
  for (int i = 0; i < 32; i += 8) {
    const int64_t r = r0 + ty + i, c = c0 + tx;
    tile[ty + i][tx] = (r < rows && c < cols) ? __ldg(in + r * ld_in + c) : 0.f;
  }
  __syncthreads();
#pragma unroll
  for (int i = 0; i < 32; i += 8) {
    const int64_t c = c0 + ty + i, r = r0 + tx;  // out[c, r]
    if (c < cols && r < rows) {
      const float v = tile[tx][ty + i];
      out[c * ld_out + r] = v;
      if (out_small != nullptr)
        out_small[c * ld_out + r] = tf32_small(v);
    }
  }
}

// ---------------------------------------------------------------------------------
// Operand preparation for the K-major tensor-core GEMMs, one pass over a (R, C) matrix:
//   v      = act'(y) * x          (act-backward fused when y != NULL; y is the activation OUTPUT)
//   out    = v            (R, C)            out_small  = tf32_small(v)
//   outT   = v^T          (C, R)            outT_small = tf32_small(v^T)
//   colsum[c] += sum_r v[r, c]              (bias gradient)
// Any output pointer may be NULL.  32 x 32 tiles through padded shared memory.
// ---------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
prep_operand_kernel(const float* __restrict__ x, const float* __restrict__ y, int act, int64_t R,
                    int64_t C, int64_t ld_in, float* __restrict__ out, float* __restrict__ out_small,
                    float* __restrict__ outT, float* __restrict__ outT_small, float* __restrict__ colsum) {
  b2_pdl_wait();
  b2_pdl_trigger();
  __shared__ float tile[32][33];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;  // 32 x 8
  const int64_t c0 = (int64_t) blockIdx.x * 32, r0 = (int64_t) blockIdx.y * 32;
#pragma unroll
  for (int i = 0; i < 32; i += 8) {
    const int64_t r = r0 + ty + i, c = c0 + tx;
    float v = 0.f;
    if (r < R && c < C) {
      v = __ldg(x + r * ld_in + c);
      if (y != nullptr) {
        const float yv = __ldg(y + r * ld_in + c);
        if (act == B2_ACT_RELU) v = (yv > 0.f) ? v : 0.f;
        else if (act == B2_ACT_SIGMOID) v = v * ((1.f - yv) * yv);
        else if (act == B2_PREP_MUL) v = v * yv;
      }
      if (out != nullptr) out[r * C + c] = v;
      if (out_small != nullptr) out_small[r * C + c] = tf32_small(v);
    }
    tile[ty + i][tx] = v;
  }
  __syncthreads();
  if (outT != nullptr) {
#pragma unroll
    for (int i = 0; i < 32; i += 8) {
      const int64_t c = c0 + ty + i, r = r0 + tx;  // outT[c, r]
      if (c < C && r < R) {
        const float v = tile[tx][ty + i];
        outT[c * R + r] = v;
        if (outT_small != nullptr) outT_small[c * R + r] = tf32_small(v);
      }
    }
  }
  if (colsum != nullptr && ty == 0) {
    const int64_t c = c0 + tx;
    if (c < C) {
      float t = 0.f;
#pragma unroll
      for (int i = 0; i < 32; ++i) t += tile[i][tx];
      b2_red_add(colsum + c, t);
    }
  }
}

// ---------------------------------------------------------------------------------
// The N = 1 output head of an MLP (Linear(K, 1)): TMA cannot address a 4-byte row and a 128-wide
// MMA tile would be 1/128 full, so it is a warp-per-row GEMV forward and one fused backward:
//   fwd: y[m] = act(<x[m,:], w> + b)
//   bwd: gz = act'(y) * gy;  gx[m,:] = gz[m] * w;  gw += sum_m gz[m] * x[m,:];  gb += sum_m gz[m]
//   With prev_act != NONE the head's input x IS the previous layer's activation output, so that
//   layer's activation backward is fused here: gx <- prev_act'(x) * gx (= dZ of the previous layer),
//   together with its 3xTF32 small part (gx_small) and its bias gradient gb_prev[k] = sum_m gx[m,k].
// ---------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
head_fwd_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ b,
                int64_t M, int K, int act, float* __restrict__ y) {
  b2_pdl_wait();
  b2_pdl_trigger();
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t) blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t) gridDim.x * blockDim.x) >> 5;
  const float bv = (b != nullptr) ? __ldg(b) : 0.f;
  for (int64_t m = warp; m < M; m += nwarps) {
    float acc = 0.f;
    for (int k = lane; k < K; k += 32) acc = fmaf(__ldg(x + m * K + k), __ldg(w + k), acc);
    acc = b2_warp_sum(acc);
    if (lane == 0) {
      float v = acc + bv;
      if (act == B2_ACT_RELU) v = fmaxf(v, 0.f);
      else if (act == B2_ACT_SIGMOID) v = 1.f / (1.f + expf(-v));
      y[m] = v;
    }
  }
}

// CTA = 256 threads = 8 warps; each CTA owns a contiguous block of rows; lane k-strided columns.
__global__ void __launch_bounds__(256)
head_bwd_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ y,
                const float* __restrict__ gy, int64_t M, int K, int act, int64_t rows_per_cta,
                float* __restrict__ gx, float* __restrict__ gw, float* __restrict__ gb, int prev_act,
                float* __restrict__ gx_small, float* __restrict__ gb_prev) {
  b2_pdl_wait();
  b2_pdl_trigger();
  extern __shared__ float sgw[];  // K partial sums of gw, then K partial sums of gb_prev
  __shared__ float red[32];
  float* sgp = sgw + K;
  for (int k = threadIdx.x; k < K; k += blockDim.x) { sgw[k] = 0.f; sgp[k] = 0.f; }
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t r0 = (int64_t) blockIdx.x * rows_per_cta;
  const int64_t r1 = min(M, r0 + rows_per_cta);
  float gb_acc = 0.f;
  // each warp keeps per-lane partials of gw for its k-strided columns over its rows
  for (int kb = 0; kb < K; kb += 32 * 8) {       // 8 columns per lane per pass
    float part[8], cs[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) { part[j] = 0.f; cs[j] = 0.f; }
    for (int64_t m = r0 + warp; m < r1; m += 8) {
      float gz = __ldg(gy + m);
      if (y != nullptr) {
        const float yv = __ldg(y + m);
        if (act == B2_ACT_RELU) gz = (yv > 0.f) ? gz : 0.f;
        else if (act == B2_ACT_SIGMOID) gz = gz * ((1.f - yv) * yv);
      }
      if (kb == 0 && lane == 0) gb_acc += gz;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int k = kb + j * 32 + lane;
        if (k < K) {
          const float xv = __ldg(x + m * K + k);
          if (gx != nullptr) {
            float val = gz * __ldg(w + k);
            if (prev_act == B2_ACT_RELU) val = (xv > 0.f) ? val : 0.f;
            else if (prev_act == B2_ACT_SIGMOID) val = val * ((1.f - xv) * xv);
            gx[m * K + k] = val;
            if (gx_small != nullptr) gx_small[m * K + k] = tf32_small(val);
            cs[j] += val;
          }
          part[j] = fmaf(gz, xv, part[j]);
        }
      }
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int k = kb + j * 32 + lane;
      if (k < K) {
        atomicAdd(sgw + k, part[j]);
        if (gb_prev != nullptr) atomicAdd(sgp + k, cs[j]);
      }
    }
  }
  __syncthreads();
  for (int k = threadIdx.x; k < K; k += blockDim.x) {
    if (sgw[k] != 0.f) b2_red_add(gw + k, sgw[k]);
    if (gb_prev != nullptr && sgp[k] != 0.f) b2_red_add(gb_prev + k, sgp[k]);
  }
  if (gb != nullptr) {
    const float t = b2_block_sum(gb_acc, red);
    if (threadIdx.x == 0 && t != 0.f) b2_red_add(gb, t);
  }
}
}  // namespace tc

// ---------------------------------------------------------------------------------
// Host side
// ---------------------------------------------------------------------------------
typedef CUresult (*b2_encode_tiled_fn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                       const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                       const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                       CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static b2_encode_tiled_fn b2_get_encode() {
  static b2_encode_tiled_fn fn = nullptr;
  if (fn == nullptr) {
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<b2_encode_tiled_fn>(ptr);
  }
  return fn;
}

// K-major operand: memory (rows, K), K contiguous, leading dimension ld; box = 128 B of k x box_rows rows.
// MN-major operand: memory (K, rows), rows contiguous, leading dimension ld; box = box_rows rows x 128 B of k.
// Unswizzled: the converter warpgroup writes the swizzled layout wgmma reads.
static int encode_operand(CUtensorMap* map, const void* base, int64_t rows, int64_t K, int64_t ld,
                          int mn_major, int box_rows, int esz) {
  b2_encode_tiled_fn enc = b2_get_encode();
  if (enc == nullptr) return b2_fail(B2_E_CUDA, "cuTensorMapEncodeTiled is unavailable in this driver");
  const cuuint32_t per128 = (cuuint32_t) (128 / esz);
  cuuint64_t dims[2], strides[1] = {(cuuint64_t) ld * (cuuint64_t) esz};
  cuuint32_t box[2], estr[2] = {1, 1};
  if (!mn_major) {
    dims[0] = (cuuint64_t) K; dims[1] = (cuuint64_t) rows;
    box[0] = per128; box[1] = (cuuint32_t) box_rows;
  } else {
    dims[0] = (cuuint64_t) rows; dims[1] = (cuuint64_t) K;
    box[0] = (cuuint32_t) box_rows; box[1] = per128;
  }
  CUresult r = enc(map, esz == 2 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2,
                   const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return b2_fail(B2_E_CUDA, "cuTensorMapEncodeTiled failed with CUresult %d", (int) r);
  return B2_OK;
}

static bool tma_ok_e(const void* p, int64_t ld, int esz) {
  return (reinterpret_cast<uintptr_t>(p) % 16 == 0) && ((ld * esz) % 16 == 0);
}
static bool tma_ok(const float* p, int64_t ld) { return tma_ok_e(p, ld, 4); }

extern "C" B2_API int b2_gemm_tc_supported(const float* a, int64_t lda, const float* b, int64_t ldb,
                                           int64_t M, int64_t N, int64_t K) {
  return (tma_ok(a, lda) && tma_ok(b, ldb) && M >= 1 && N >= 1 && K >= 1 && M < (1ll << 31) &&
          N < (1ll << 31) && K < (1ll << 31)) ? 1 : 0;
}

// plan != NULL: fill in the launch plan (tile shape, ring depths, shared memory) and return without
// touching the device — pure host arithmetic, so the CPU test-suite can sweep it (tests/test_abi.py).
template <int BN, bool X3>
static size_t gemm_smem_bytes() {
  const size_t tile = (size_t) (tc::BM + BN) * 128;
  return tc::RSTAGES * tile + tc::CSTAGES * (X3 ? 2 : 1) * tile + 1024 + 128;   // + alignment slack, mbarriers
}
template <int BN, bool X3>
static int gemm_launch(const tc::Params& p, int grid, cudaStream_t st) {
  void (*kern)(tc::Params) = tc::gemm_tc_kernel<BN, X3>;
  const size_t smem = gemm_smem_bytes<BN, X3>();
  // opt-in to > 48 KB of dynamic shared memory: an idempotent per-process property of each instantiation
  // (C++11 guarantees the initialiser runs once, thread-safely)
  static const cudaError_t attr_rc = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) smem);
  if (attr_rc != cudaSuccess) return b2_fail(B2_E_CUDA, "b2_gemm_tc: smem attribute: %s", cudaGetErrorString(attr_rc));
  B2_LAUNCH(kern, grid, tc::NTHREADS, smem, st, p);
  B2_CUDA_LAUNCH_CHECK("b2_gemm_tc");
  return B2_OK;
}

static int gemm_tc_impl(const b2_gemm_desc* d, void* stream, b2_gemm_plan* plan) {
  B2_REQUIRE(d != nullptr, "NULL descriptor");
  const void* a = d->a; const void* b = d->b; float* c = d->c;
  const int64_t M = d->M, N = d->N, K = d->K, lda = d->lda, ldb = d->ldb, ldc = d->ldc;
  B2_REQUIRE(a && b && c, "NULL operand");
  B2_REQUIRE(d->elem_dtype == B2_F32 || d->elem_dtype == B2_BF16, "operand dtype must be B2_F32 or B2_BF16");
  const int esz = (d->elem_dtype == B2_BF16) ? 2 : 4;
  B2_REQUIRE(M >= 1 && N >= 1 && K >= 1 && ldc >= N, "bad shape");
  B2_REQUIRE(M < (1ll << 31) && N < (1ll << 31) && K < (1ll << 31), "shape exceeds 31 bits");
  B2_REQUIRE(lda >= (d->a_mn_major ? M : K) && ldb >= (d->b_mn_major ? N : K), "leading dimension too small");
  B2_REQUIRE(d->act >= B2_ACT_NONE && d->act <= B2_ACT_SIGMOID, "bad activation code %d", d->act);
  B2_REQUIRE(d->act_bwd >= B2_ACT_NONE && d->act_bwd <= B2_ACT_SIGMOID, "bad act_bwd code %d", d->act_bwd);
  B2_REQUIRE(d->act_bwd == B2_ACT_NONE || d->ybwd != nullptr, "act_bwd needs ybwd");
  B2_REQUIRE((d->a_small == nullptr) == (d->b_small == nullptr), "3xTF32 needs both small operands");
  B2_REQUIRE(esz == 4 || d->a_small == nullptr, "bf16 operands are single-pass (no small parts)");
  const bool inline_split = (d->flags & B2_GEMM_X3_INLINE) != 0;
  B2_REQUIRE(!inline_split || (esz == 4 && d->a_small == nullptr), "B2_GEMM_X3_INLINE: fp32 operands, no small parts");
  // The small parts are always derived from the fp32 operands in shared memory (the converter warpgroup).  A
  // caller's a_small / b_small hold the same values (b2_tf32_small of the operand) and select 3xTF32 alone.
  const bool three_pass = inline_split || d->a_small != nullptr;
  const int64_t ld_aux = d->ld_aux > 0 ? d->ld_aux : ldc;
  B2_REQUIRE(d->c_small == nullptr || ld_aux >= N, "ld_aux too small");
  if (!tma_ok_e(a, lda, esz) || !tma_ok_e(b, ldb, esz) ||
      (d->a_small != nullptr && !(tma_ok(d->a_small, lda) && tma_ok(d->b_small, ldb))))
    return b2_fail(B2_E_UNSUPPORTED, "operands are not TMA-addressable (16-byte base, 16-byte row pitch)");
  cudaStream_t st = (cudaStream_t) stream;

  // Tile-shape choice: BN in {32, 64, 128} (3xTF32: <= 64, its three accumulator sets live in registers);
  // minimise waves x per-CTA work, where one wave = 132 CTAs (one per SM).
  const int bke = 128 / esz;
  const int64_t tiles_m = b2_ceil_div(M, tc::BM);
  const int64_t num_kb = b2_ceil_div(K, bke);
  // split-K adds partial tiles with red.global: only for a plain linear epilogue
  const bool linear = (d->act == B2_ACT_NONE && d->mul == nullptr && d->add == nullptr && d->ybwd == nullptr &&
                       d->c_small == nullptr && d->c_pre == nullptr && d->colsum == nullptr);
  int best_bn = 0, best_split = 1;
  double best_cost = 1e300;
  const int bn_max = three_pass ? 64 : 128;
  // cycles per k-block: the tensor pipe needs passes x 4 instructions x bn/2 (m64 per warpgroup, two in
  // parallel), the converter warpgroup moves (128 + bn) rows of 128 bytes (2x for the small parts)
  const double mma_per_bn = (three_pass ? 3.0 : 1.0) * 2.0;
  const double conv_per_row = three_pass ? 4.0 : 3.0;
  for (int bn = 32; bn <= bn_max; bn *= 2) {
    const int64_t tiles_n = b2_ceil_div(N, bn);
    for (int split = 1; split <= 32; split *= 2) {
      if (split > 1 && (!linear || num_kb / split < 8)) break;
      const int64_t ctas = tiles_m * tiles_n * split;
      const int64_t waves = b2_ceil_div(ctas, B2_NUM_SMS);
      const double kb = (double) b2_ceil_div(num_kb, split);
      const double per_kb = fmax(mma_per_bn * bn, conv_per_row * (double) (tc::BM + bn));
      const double cost = (double) waves * (10000.0 + kb * per_kb);
      if (cost < best_cost) { best_cost = cost; best_bn = bn; best_split = split; }
    }
  }
  tc::Params p;
  memset(&p, 0, sizeof(p));
  if (plan == nullptr) {
    int rc = encode_operand(&p.map_a, a, M, K, lda, d->a_mn_major, tc::BM, esz);
    if (rc != B2_OK) return rc;
    rc = encode_operand(&p.map_b, b, N, K, ldb, d->b_mn_major, best_bn, esz);
    if (rc != B2_OK) return rc;
  }
  p.c = c; p.c_small = reinterpret_cast<float*>(d->c_small); p.c_pre = d->c_pre; p.ldc = ldc; p.ld_aux = ld_aux;
  p.bias = d->bias; p.mul = d->mul; p.add = d->add;
  p.ybwd = d->ybwd; p.colsum = d->colsum;
  p.M = (int) M; p.N = (int) N; p.K = (int) K; p.act = d->act; p.act_bwd = d->act_bwd; p.esz = esz;
  p.a_mn = d->a_mn_major ? 1 : 0; p.b_mn = d->b_mn_major ? 1 : 0;
  p.beta = d->beta_accumulate ? 1 : 0;
  p.kb_per_split = (int) b2_ceil_div(num_kb, best_split);
  const int splits = (int) b2_ceil_div(num_kb, p.kb_per_split);
  const int64_t tiles_n = b2_ceil_div(N, best_bn);
  const int64_t total_tiles = tiles_m * tiles_n * splits;
  B2_REQUIRE(total_tiles < (1ll << 31), "too many tiles");
  p.tiles_m = (int) tiles_m; p.tiles_n = (int) tiles_n; p.splits = splits;
  size_t smem = 0;
  switch (best_bn * 2 + (three_pass ? 1 : 0)) {
    case 64: smem = gemm_smem_bytes<32, false>(); break;
    case 65: smem = gemm_smem_bytes<32, true>(); break;
    case 128: smem = gemm_smem_bytes<64, false>(); break;
    case 129: smem = gemm_smem_bytes<64, true>(); break;
    default: smem = gemm_smem_bytes<128, false>(); break;
  }
  B2_REQUIRE(smem <= (size_t) 227 * 1024, "tile does not fit shared memory");
  if (plan != nullptr) {
    plan->bn = best_bn; plan->splits = splits; plan->stages = tc::RSTAGES; plan->cstages = tc::CSTAGES;
    plan->grid = (int) total_tiles; plan->threads = tc::NTHREADS; plan->tiles_m = p.tiles_m; plan->tiles_n = p.tiles_n;
    plan->passes = three_pass ? 3 : 1; plan->kb_per_split = p.kb_per_split; plan->smem_bytes = (int64_t) smem;
    return B2_OK;
  }
  if (splits > 1 && !p.beta && !(d->flags & B2_GEMM_C_IS_ZERO)) {
    cudaError_t e = cudaMemset2DAsync(c, (size_t) ldc * 4, 0, (size_t) N * 4, (size_t) M, st);
    if (e != cudaSuccess) return b2_fail(B2_E_CUDA, "b2_gemm_tc: memset: %s", cudaGetErrorString(e));
  }
  if (d->colsum != nullptr && !(d->flags & B2_GEMM_COLSUM_IS_ZERO)) {
    cudaError_t e = cudaMemsetAsync(d->colsum, 0, sizeof(float) * (size_t) N, st);
    if (e != cudaSuccess) return b2_fail(B2_E_CUDA, "b2_gemm_tc: memset: %s", cudaGetErrorString(e));
  }
  const int grid = (int) total_tiles;
  switch (best_bn * 2 + (three_pass ? 1 : 0)) {
    case 64: return gemm_launch<32, false>(p, grid, st);
    case 65: return gemm_launch<32, true>(p, grid, st);
    case 128: return gemm_launch<64, false>(p, grid, st);
    case 129: return gemm_launch<64, true>(p, grid, st);
    default: return gemm_launch<128, false>(p, grid, st);
  }
}

extern "C" B2_API int b2_gemm_tc_ex(const b2_gemm_desc* d, void* stream) { return gemm_tc_impl(d, stream, nullptr); }

extern "C" B2_API int b2_gemm_tc_plan(const b2_gemm_desc* d, b2_gemm_plan* plan) {
  B2_REQUIRE(plan != nullptr, "NULL plan");
  return gemm_tc_impl(d, nullptr, plan);
}

// fp32 (rows, cols; ld_in) -> bf16 (rows, cols; ld_out), round-to-nearest-even: the bf16-mode operand of a
// tensor whose producer is not one of our epilogues (weights once per step, the first layer's input).
namespace tc {
__global__ void __launch_bounds__(256)
to_bf16_kernel(const float* __restrict__ x, int64_t rows, int64_t cols, int64_t ld_in,
               __nv_bfloat16* __restrict__ out, int64_t ld_out) {
  const int64_t n = rows * cols;
  for (int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t) gridDim.x * blockDim.x) {
    const int64_t r = i / cols, c = i - r * cols;
    out[r * ld_out + c] = __float2bfloat16_rn(__ldg(x + r * ld_in + c));
  }
}
}  // namespace tc

extern "C" B2_API int b2_to_bf16(const float* x, int64_t rows, int64_t cols, int64_t ld_in, void* out,
                                 int64_t ld_out, void* stream) {
  B2_REQUIRE(x && out && rows >= 0 && cols >= 0 && ld_in >= cols && ld_out >= cols, "bad argument");
  if (rows == 0 || cols == 0) return B2_OK;
  int64_t blocks = b2_ceil_div(rows * cols, 256);
  if (blocks > (int64_t) B2_NUM_SMS * 8) blocks = (int64_t) B2_NUM_SMS * 8;
  tc::to_bf16_kernel<<<(int) blocks, 256, 0, (cudaStream_t) stream>>>(x, rows, cols, ld_in,
                                                                       reinterpret_cast<__nv_bfloat16*>(out), ld_out);
  B2_CUDA_LAUNCH_CHECK("b2_to_bf16");
  return B2_OK;
}

extern "C" B2_API int b2_gemm_tc(const float* a, int64_t lda, const float* b, int64_t ldb, float* c,
                                 int64_t ldc, int64_t M, int64_t N, int64_t K, const float* bias, int act,
                                 const float* mul, const float* add, int beta_accumulate,
                                 const float* a_small, const float* b_small, void* stream) {
  b2_gemm_desc d;
  memset(&d, 0, sizeof(d));
  d.a = a; d.b = b; d.a_small = a_small; d.b_small = b_small; d.c = c;
  d.bias = bias; d.mul = mul; d.add = add;
  d.lda = lda; d.ldb = ldb; d.ldc = ldc; d.M = M; d.N = N; d.K = K;
  d.act = act; d.beta_accumulate = beta_accumulate;
  return b2_gemm_tc_ex(&d, stream);
}

extern "C" B2_API int b2_split_tf32(const float* x, float* small, int64_t n, void* stream) {
  B2_REQUIRE(x && small, "NULL pointer");
  if (n <= 0) return B2_OK;
  int64_t blocks = b2_ceil_div(n, 256);
  if (blocks > (int64_t) B2_NUM_SMS * 8) blocks = (int64_t) B2_NUM_SMS * 8;
  B2_LAUNCH(tc::split_tf32_kernel, (int) blocks, 256, 0, (cudaStream_t) stream, x, small, n);
  B2_CUDA_LAUNCH_CHECK("b2_split_tf32");
  return B2_OK;
}

extern "C" B2_API int b2_transpose_f32(const float* in, int64_t rows, int64_t cols, int64_t ld_in,
                                       float* out, int64_t ld_out, float* out_small, void* stream) {
  B2_REQUIRE(in && out, "NULL pointer");
  B2_REQUIRE(rows >= 0 && cols >= 0 && ld_in >= cols && ld_out >= rows, "bad shape");
  if (rows == 0 || cols == 0) return B2_OK;
  dim3 grid((unsigned) b2_ceil_div(cols, 32), (unsigned) b2_ceil_div(rows, 32));
  B2_REQUIRE(grid.y <= 65535, "too many rows for this launch geometry");
  tc::transpose_kernel<<<grid, 256, 0, (cudaStream_t) stream>>>(in, rows, cols, ld_in, out, ld_out, out_small);
  B2_CUDA_LAUNCH_CHECK("b2_transpose_f32");
  return B2_OK;
}

extern "C" B2_API int b2_prep_operand(const float* x, const float* y, int act, int64_t R, int64_t C,
                                      float* out, float* out_small, float* outT, float* outT_small,
                                      float* colsum, void* stream) {
  B2_REQUIRE(x != nullptr, "NULL input");
  B2_REQUIRE(R >= 0 && C >= 0, "bad shape");
  B2_REQUIRE((act >= B2_ACT_NONE && act <= B2_ACT_SIGMOID) || act == B2_PREP_MUL, "bad activation code %d", act);
  cudaStream_t st = (cudaStream_t) stream;
  if (colsum != nullptr) {
    cudaError_t e = cudaMemsetAsync(colsum, 0, sizeof(float) * (size_t) C, st);
    if (e != cudaSuccess) return b2_fail(B2_E_CUDA, "b2_prep_operand: memset: %s", cudaGetErrorString(e));
  }
  if (R == 0 || C == 0) return B2_OK;
  dim3 grid((unsigned) b2_ceil_div(C, 32), (unsigned) b2_ceil_div(R, 32));
  B2_REQUIRE(grid.y <= 65535, "too many rows for this launch geometry");
  B2_LAUNCH(tc::prep_operand_kernel, grid, 256, 0, st, x, y, act, R, C, C, out, out_small, outT, outT_small, colsum);
  B2_CUDA_LAUNCH_CHECK("b2_prep_operand");
  return B2_OK;
}

extern "C" B2_API int b2_head_fwd(const float* x, const float* w, const float* b, int64_t M, int K, int act,
                                  float* y, void* stream) {
  B2_REQUIRE(x && w && y, "NULL pointer");
  B2_REQUIRE(K >= 1 && act >= B2_ACT_NONE && act <= B2_ACT_SIGMOID, "bad K/act");
  if (M <= 0) return B2_OK;
  int64_t blocks = b2_ceil_div(M * 32, 256);
  if (blocks > (int64_t) B2_NUM_SMS * 8) blocks = (int64_t) B2_NUM_SMS * 8;
  B2_LAUNCH(tc::head_fwd_kernel, (int) blocks, 256, 0, (cudaStream_t) stream, x, w, b, M, K, act, y);
  B2_CUDA_LAUNCH_CHECK("b2_head_fwd");
  return B2_OK;
}

extern "C" B2_API int b2_head_bwd(const float* x, const float* w, const float* y, const float* gy, int64_t M,
                                  int K, int act, float* gx, float* gw, float* gb, void* stream) {
  return b2_head_bwd_ex(x, w, y, gy, M, K, act, gx, gw, gb, B2_ACT_NONE, nullptr, nullptr, 0, stream);
}

extern "C" B2_API int b2_head_bwd_ex(const float* x, const float* w, const float* y, const float* gy, int64_t M,
                                     int K, int act, float* gx, float* gw, float* gb, int prev_act,
                                     float* gx_small, float* gb_prev, int grads_zeroed, void* stream) {
  B2_REQUIRE(x && w && gy && gw, "NULL pointer");
  B2_REQUIRE(K >= 1 && K <= 6144 && act >= B2_ACT_NONE && act <= B2_ACT_SIGMOID, "bad K/act");
  B2_REQUIRE(prev_act >= B2_ACT_NONE && prev_act <= B2_ACT_SIGMOID, "bad prev_act");
  B2_REQUIRE(act == B2_ACT_NONE || y != nullptr, "activation backward needs y");
  B2_REQUIRE(gx != nullptr || (gx_small == nullptr && gb_prev == nullptr && prev_act == B2_ACT_NONE),
             "prev_act / gx_small / gb_prev need gx");
  cudaStream_t st = (cudaStream_t) stream;
  cudaError_t e = cudaSuccess;
  if (!grads_zeroed) {    // the caller vouches that gw / gb / gb_prev are all-zero (a gradient arena cleared by Adam)
    e = cudaMemsetAsync(gw, 0, sizeof(float) * (size_t) K, st);
    if (e == cudaSuccess && gb_prev != nullptr) e = cudaMemsetAsync(gb_prev, 0, sizeof(float) * (size_t) K, st);
    if (e == cudaSuccess && gb != nullptr) e = cudaMemsetAsync(gb, 0, sizeof(float), st);
  }
  if (e != cudaSuccess) return b2_fail(B2_E_CUDA, "b2_head_bwd: memset: %s", cudaGetErrorString(e));
  if (M <= 0) return B2_OK;
  int64_t ctas = 2 * B2_NUM_SMS;
  if (ctas > b2_ceil_div(M, 8)) ctas = b2_ceil_div(M, 8);
  const int64_t rows_per_cta = b2_ceil_div(M, ctas);
  ctas = b2_ceil_div(M, rows_per_cta);
  const float* y_arg = (act == B2_ACT_NONE) ? nullptr : y;
  B2_LAUNCH(tc::head_bwd_kernel, (int) ctas, 256, 2 * sizeof(float) * (size_t) K, st,
            x, w, y_arg, gy, M, K, act, rows_per_cta, gx, gw, gb, prev_act, gx_small, gb_prev);
  B2_CUDA_LAUNCH_CHECK("b2_head_bwd");
  return B2_OK;
}

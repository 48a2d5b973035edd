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
// Structure (one CTA per 128 x BN output tile and K split; 384 threads), one ring of 2-4 stages whose layout
// depends on the operand majors (Ring):
//   K-major operands are loaded by TMA with the 128B swizzle, straight into the layout wgmma reads; wgmma
//   .tf32 reads an fp32 value as its truncation big(x), so the raw tile is the big part (DESIGN.md §4).
//   MN-major operands land unswizzled in a staging tile of the same stage; wgmma reads tf32 from shared memory
//   only K-major, so they are transposed into the swizzled tile in shared memory and stay as they lie in HBM.
//   warp 0         one thread issues the TMA loads of a stage as soon as the consumers release it.
//   warps 1-3      converter: MN-major staging -> swizzled tile; 3xTF32: the small parts of B and of an MN-major
//                  A, written at the offsets of the swizzled tile in their own tiles (no re-layout).
//   warpgroups 1-2 64 rows each: wgmma m64nBNk8 (tf32) / k16 (bf16), both operands from shared memory, except in
//                  3xTF32 with a K-major A: each thread loads its A fragment and splits it in registers.  3xTF32
//                  commits each k-block as two groups, the main product and then the cross terms; the main
//                  product is folded into the sum while the cross terms still run, and a stage is released
//                  one k-block later.  The single-pass modes likewise keep one group in flight.  Then the fused
//                  epilogue: the accumulators are staged as a row-major tile in the dead ring, and each thread walks
//                  it in 16-byte row segments, a batch at a time, with every global load of a batch issued before
//                  its first store.
// Dropout (MLP_Block's Linear -> act -> Dropout): a launch whose descriptor carries a dropout snapshot runs the
// DROP instantiation of its kernel, whose epilogue applies the layer's mask keep(seed, offset, m, n) (philox.cuh)
// after the activation and before the activation backward; launches without one keep the instantiations as
// they were.
// Kernels of a step are chained with programmatic dependent launch (prologue under the predecessor's tail).
// Every mbarrier wait is bounded: a pipeline bug traps with a message instead of hanging the GPU.
#include "b2_common.cuh"
#include "philox.cuh"
#include <string.h>
#include <cstdlib>
#include <cuda.h>  // CUtensorMap + enums only; cuTensorMapEncodeTiled is resolved at run time

namespace tc {
constexpr int BM = 128;          // two consumer warpgroups x wgmma M = 64
constexpr int NTHREADS = 384;    // producer / converter warpgroup + two wgmma warpgroups
constexpr int NCONV = 96;        // converter threads (warps 1-3)
constexpr int BACKFILL_KB = 16;  // least k-blocks per CTA of a B2_GEMM_BACKFILL launch split over K
enum Mode { TF32 = 0, BF16 = 1, X3 = 2 };

// Shared memory of one pipeline stage, sized per launch from the operand majors: the swizzled A and B tiles
// wgmma reads, the small parts the converter still makes (B always in 3xTF32; A only when it is MN-major, since a
// K-major A is split in registers), and unswizzled staging tiles only for an MN-major operand.  Every tile
// starts 1024-byte aligned.
struct Ring {
  uint32_t off_b, off_as, off_bs, off_sa, off_sb;   // byte offsets in a stage (A sits at 0)
  uint32_t stage;                                    // bytes per stage
  int stages;                                        // 2-4
  size_t smem;                                       // dynamic shared memory of the launch
};
constexpr uint32_t RING_EXTRA = 1024 + 128;          // alignment slack, mbarriers
constexpr uint32_t SMEM_MAX = 227u * 1024u;
constexpr Ring ring_layout(int bn, int mode, bool a_mn, bool b_mn) {
  const uint32_t a = BM * 128, b = (uint32_t) bn * 128;
  Ring r{};
  uint32_t o = a;
  r.off_b = o;  o += b;
  r.off_as = o; o += (mode == X3 && a_mn) ? a : 0;
  r.off_bs = o; o += mode == X3 ? b : 0;
  r.off_sa = o; o += a_mn ? a : 0;
  r.off_sb = o; o += b_mn ? b : 0;
  r.stage = o;
  r.stages = (SMEM_MAX - RING_EXTRA) / o >= 4 ? 4 : (int) ((SMEM_MAX - RING_EXTRA) / o);
  r.smem = (size_t) r.stages * o + RING_EXTRA;
  return r;
}
// The largest ring an instantiation launches with, over the four operand-major pairs: its shared-memory attribute.
// (Not always both MN-major: a smaller stage can buy a deeper ring.)
constexpr size_t ring_smem_max(int bn, int mode) {
  size_t m = 0;
  for (int a_mn = 0; a_mn < 2; ++a_mn)
    for (int b_mn = 0; b_mn < 2; ++b_mn) {
      const size_t s = ring_layout(bn, mode, a_mn != 0, b_mn != 0).smem;
      m = s > m ? s : m;
    }
  return m;
}
static_assert(ring_layout(128, TF32, true, true).stages >= 2 && ring_layout(64, X3, true, true).stages >= 2,
              "ring does not fit shared memory");
// The epilogue stages the accumulators in the dead ring: a row-major fp32 tile of BM x BN with a row pitch of BN + 8
// floats, then 256 x 4 column partial sums.  A pitch of 8 (mod 32) words makes the float2 fragment stores (8 rows x
// 32 bytes per instruction) hit 32 distinct banks per 128 bytes; a quarter-warp's float4 row reads are contiguous.
constexpr int epi_pitch(int bn) { return bn + 8; }
constexpr uint32_t epi_bytes(int bn) { return (uint32_t) (BM * epi_pitch(bn) + 256 * 4) * 4u; }
constexpr bool epi_fits(int bn, int mode) {
  for (int a_mn = 0; a_mn < 2; ++a_mn)
    for (int b_mn = 0; b_mn < 2; ++b_mn) {
      const Ring r = ring_layout(bn, mode, a_mn != 0, b_mn != 0);
      if ((uint32_t) r.stages * r.stage < epi_bytes(bn)) return false;
    }
  return true;
}
static_assert(epi_fits(32, TF32) && epi_fits(64, TF32) && epi_fits(128, TF32) && epi_fits(32, BF16) &&
              epi_fits(64, BF16) && epi_fits(128, BF16) && epi_fits(32, X3) && epi_fits(64, X3),
              "epilogue tile does not fit the ring");

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
  int vec;                // every epilogue pointer and leading dimension allows 16-byte row segments (bf16 c_small: 8)
  int tiles_m, tiles_n, splits;
  Ring ring;              // this launch's stage layout (ring_layout of its tile width, mode and operand majors)
  const int64_t* drop_rng;  // DROP instantiations only: the forward's {seed, offset} snapshot
  int64_t drop_layer;       // counter offset of the mask: snapshot offset + drop_layer
  uint32_t drop_thresh;     // keep iff the element's Philox word < drop_thresh
  float drop_scale;         // 1 / (1 - p) as fp32
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
// Bounded wait: ~2 s at 2 GHz, then trap (never hang the device).  No printf: a function call anywhere in the
// kernel makes ptxas serialise every wgmma (C7510).
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  const long long t0 = clock64();
  while (!mbar_try_wait(bar, parity))
    if (clock64() - t0 > 4000000000LL) __trap();
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
__device__ __forceinline__ void wgmma_wait1() { asm volatile("wgmma.wait_group.sync.aligned 1;" ::: "memory"); }

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
// The same m64nNk8 tf32 with A from registers: a[] is this thread's fragment of the warp's 16 rows x 8 k —
// a[0] (row l/4, k l%4), a[1] (row l/4 + 8, k l%4), a[2] (row l/4, k l%4 + 4), a[3] (row l/4 + 8, k l%4 + 4).
__device__ __forceinline__ void wgmma_tf32_rs(float (&d)[16], const uint32_t (&a)[4], uint64_t b, uint32_t scale_d) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %21, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, {%16, %17, %18, %19}, %20, p, 1, 1;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "r"(scale_d));
}
__device__ __forceinline__ void wgmma_tf32_rs(float (&d)[32], const uint32_t (&a)[4], uint64_t b, uint32_t scale_d) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %37, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, {%32, %33, %34, %35}, %36, p, 1, 1;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "r"(scale_d));
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

// What the converter writes for 16 bytes of operand: bf16 as it is; for fp32 the big part (13 low mantissa bits
// cleared), or the big part and, at the same offset in the small tile, the small part.
enum Split { RAW = 0, BIG = 1, BIG_SMALL = 2 };
template <int SPLIT>
__device__ __forceinline__ void store_split(uint8_t* dst, uint32_t small_off, uint32_t off, const float4& v) {
  static_assert(SPLIT != RAW, "fp32 tiles are stored split");
  *reinterpret_cast<float4*>(dst + off) = make_float4(tf32_big(v.x), tf32_big(v.y), tf32_big(v.z), tf32_big(v.w));
  if (SPLIT == BIG_SMALL)
    *reinterpret_cast<float4*>(dst + small_off + off) =
        make_float4(tf32_small(v.x), tf32_small(v.y), tf32_small(v.z), tf32_small(v.w));
}

// One MN-major k-block as TMA wrote it — (k, rows): 32 fp32 or 64 bf16 k-rows of `rows` elements — into the
// K-major 128B-swizzled tile of `rows` rows, transposed in registers (4 x 4 fp32 or 8 x 8 bf16 per thread).
template <bool BF, int SPLIT>
__device__ __forceinline__ void transpose_tile(const uint8_t* src, uint8_t* dst, uint32_t small_off, int rows, int ct) {
  if constexpr (BF) {
    for (int b = ct; b < rows; b += NCONV) {
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
  } else {
    // Thread b takes 4 rows from r0 and k-chunk kq.  Each group of 64 covers 8 row quads x 8 chunks: the 8 lanes of a
    // quarter-warp take 8 consecutive row quads (16-byte loads in 8 different bank groups, whatever the k-row pitch)
    // and chunks kq = q ^ s; the swizzled stores of row r0 + i then land in chunks kq ^ (r0 + i) % 8 =
    // q ^ 4 (q & 1) ^ s ^ i, distinct over q: both sides are conflict-free.  rows is a multiple of 32.
    for (int b = ct; b < 2 * rows; b += NCONV) {
      const int q = b & 7, s = (b >> 3) & 7;
      const int kq = q ^ s, r0 = ((b >> 6) * 8 + q) * 4;
      float4 v[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) v[j] = *reinterpret_cast<const float4*>(src + ((4 * kq + j) * rows + r0) * 4);
      store_split<SPLIT>(dst, small_off, swz(r0 + 0, kq), make_float4(v[0].x, v[1].x, v[2].x, v[3].x));
      store_split<SPLIT>(dst, small_off, swz(r0 + 1, kq), make_float4(v[0].y, v[1].y, v[2].y, v[3].y));
      store_split<SPLIT>(dst, small_off, swz(r0 + 2, kq), make_float4(v[0].z, v[1].z, v[2].z, v[3].z));
      store_split<SPLIT>(dst, small_off, swz(r0 + 3, kq), make_float4(v[0].w, v[1].w, v[2].w, v[3].w));
    }
  }
}

// The small part of a swizzled fp32 tile, written at the same offsets of the small tile: no re-layout.
__device__ __forceinline__ void small_tile(const uint8_t* src, uint8_t* dst, int rows, int ct) {
  for (int q = ct; q < rows * 8; q += NCONV) {
    const float4 v = *reinterpret_cast<const float4*>(src + 16 * q);
    *reinterpret_cast<float4*>(dst + 16 * q) = make_float4(tf32_small(v.x), tf32_small(v.y), tf32_small(v.z), tf32_small(v.w));
  }
}

// A row segment of the epilogue: 4 consecutive fp32 of one row as one 16-byte access when `vec` (whole and aligned),
// else the first `nv` of them one by one (the rest read as 0).  NC: read-only for the whole kernel.
template <bool NC>
__device__ __forceinline__ float4 seg_load(const float* p, bool vec, int nv) {
  if (vec) return NC ? __ldg(reinterpret_cast<const float4*>(p)) : *reinterpret_cast<const float4*>(p);
  float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
  if (nv > 0) v.x = NC ? __ldg(p) : p[0];
  if (nv > 1) v.y = NC ? __ldg(p + 1) : p[1];
  if (nv > 2) v.z = NC ? __ldg(p + 2) : p[2];
  if (nv > 3) v.w = NC ? __ldg(p + 3) : p[3];
  return v;
}
__device__ __forceinline__ void seg_store(float* p, const float4& v, bool vec, int nv) {
  if (vec) { *reinterpret_cast<float4*>(p) = v; return; }
  if (nv > 0) p[0] = v.x;
  if (nv > 1) p[1] = v.y;
  if (nv > 2) p[2] = v.z;
  if (nv > 3) p[3] = v.w;
}
__device__ __forceinline__ void seg_red_add(float* p, const float4& v, bool vec, int nv) {
  if (vec) { b2_red_add_v4(p, v); return; }
  if (nv > 0) b2_red_add(p, v.x);
  if (nv > 1) b2_red_add(p + 1, v.y);
  if (nv > 2) b2_red_add(p + 2, v.z);
  if (nv > 3) b2_red_add(p + 3, v.w);
}
__device__ __forceinline__ void seg_store_bf16(__nv_bfloat16* p, const float4& v, bool vec, int nv) {
  const __nv_bfloat162 lo = __floats2bfloat162_rn(v.x, v.y), hi = __floats2bfloat162_rn(v.z, v.w);
  if (vec) {
    *reinterpret_cast<uint2*>(p) = make_uint2(*reinterpret_cast<const uint32_t*>(&lo), *reinterpret_cast<const uint32_t*>(&hi));
    return;
  }
  if (nv > 0) p[0] = lo.x;
  if (nv > 1) p[1] = lo.y;
  if (nv > 2) p[2] = hi.x;
  if (nv > 3) p[3] = hi.y;
}

// The fused epilogue of one element after c_pre: t = accumulator + bias; mv, av, yv, cv are its mul, add, ybwd and
// (beta) C.  Every operation is rounded on its own (no contraction into fma).
// DROP: keep is the element's dropout mask bit.  The mask multiplies after the activation (forward: y = act(z) *
// keep * scale) and before the activation backward (dgrad: dZ = act'(.) * keep * scale * dH), where ybwd holds the
// dropped output: ReLU's act' is ybwd > 0 as before; sigmoid's s is recovered as ybwd / scale on kept elements.
// LEAKY: the instantiation that also knows B2_ACT_LEAKY_RELU (forward and act_bwd; its act' is ybwd > 0 ? 1 : slope,
// which a dropped element's zero gradient leaves zero).  Every other launch runs the LEAKY = false code, which is the
// epilogue without it.
template <bool DROP, bool LEAKY>
__device__ __forceinline__ float epilogue_elem(const Params& p, float t, float mv, float av, float yv, float cv,
                                              bool keep) {
  if (p.mul != nullptr) t = __fmul_rn(t, mv);
  if (p.add != nullptr) t = __fadd_rn(t, av);
  if (p.act == B2_ACT_RELU) t = fmaxf(t, 0.f);
  else if (p.act == B2_ACT_SIGMOID) t = 1.f / (1.f + expf(-t));
  if constexpr (LEAKY) {
    if (p.act == B2_ACT_LEAKY_RELU) t = t > 0.f ? t : __fmul_rn(t, B2_LEAKY_SLOPE);
  }
  if constexpr (DROP) t = keep ? __fmul_rn(t, p.drop_scale) : 0.f;
  if (p.ybwd != nullptr) {     // activation backward of the PRODUCER of this gradient, fused
    if (p.act_bwd == B2_ACT_RELU) t = (yv > 0.f) ? t : 0.f;
    else if (p.act_bwd == B2_ACT_SIGMOID) {
      const float s = DROP ? __fdiv_rn(yv, p.drop_scale) : yv;
      t = __fmul_rn(t, __fmul_rn(__fsub_rn(1.f, s), s));
    }
    if constexpr (LEAKY) {
      if (p.act_bwd == B2_ACT_LEAKY_RELU) t = (yv > 0.f) ? t : __fmul_rn(t, B2_LEAKY_SLOPE);
    }
  }
  if (p.beta) t = __fadd_rn(t, cv);
  return t;
}

// The two consumer warpgroups (threads 128-383) meet; barrier 0 is __syncthreads.
__device__ __forceinline__ void consumer_sync() { asm volatile("bar.sync 1, 256;" ::: "memory"); }

template <int BN, int MODE, bool DROP, bool LEAKY>
__global__ void __launch_bounds__(NTHREADS, 1)
gemm_tc_kernel(const __grid_constant__ Params p) {
  constexpr int NR = BN / 2;                            // accumulators per thread: 64 x BN per warpgroup
  constexpr int BKE = MODE == BF16 ? 64 : 32;           // k elements per k-block: one 128-byte swizzle row
  const Ring& R = p.ring;
  const int S = R.stages;
  extern __shared__ uint8_t smem_raw[];
  // 128B-swizzled tiles need 1024-byte aligned bases: align by hand (1 KB of slack is requested).
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + S * R.stage);
  // per stage: TMA landed; converter done; consumers done (the producer may refill it)
  const uint32_t full0 = smem_u32(bars), conv0 = smem_u32(bars + S), empty0 = smem_u32(bars + 2 * S);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int num_kb_total = (p.K + BKE - 1) / BKE;
  const int tiles_mn = p.tiles_m * p.tiles_n;
  const int z = blockIdx.x / tiles_mn, rr = blockIdx.x - z * tiles_mn;
  const int m0 = (rr / p.tiles_n) * BM, n0 = (rr % p.tiles_n) * BN;
  const int kb_begin = z * p.kb_per_split;
  const int nkb = min(num_kb_total, kb_begin + p.kb_per_split) - kb_begin;
  const bool conv = MODE == X3 || p.a_mn || p.b_mn;    // the converter has work in every stage

  if (threadIdx.x == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&p.map_a)) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&p.map_b)) : "memory");
    for (int s = 0; s < S; ++s) {
      mbar_init(full0 + 8 * s, 1);
      mbar_init(conv0 + 8 * s, NCONV / 32);   // one arrival per converter warp
      mbar_init(empty0 + 8 * s, 8);           // one arrival per consumer warp
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
    // ---------------- warpgroup 0: TMA producer (warp 0) and converter (warps 1-3) ----------------
    if (warp == 0) {
      if (lane == 0) {
        int s = 0;
        uint32_t ph = 0;
        for (int i = 0; i < nkb; ++i) {
          const int kb = kb_begin + i;
          if (i >= S) mbar_wait(empty0 + 8 * s, ph ^ 1u);
          const uint32_t st = smem_u32(smem + s * R.stage), bar = full0 + 8 * s;
          mbar_expect_tx(bar, (BM + BN) * 128);   // out-of-range parts of a box arrive zero-filled, count in full
          if (p.a_mn) tma_load_2d(st + R.off_sa, &p.map_a, bar, m0, kb * BKE);
          else tma_load_2d(st, &p.map_a, bar, kb * BKE, m0);
          if (p.b_mn) tma_load_2d(st + R.off_sb, &p.map_b, bar, n0, kb * BKE);
          else tma_load_2d(st + R.off_b, &p.map_b, bar, kb * BKE, n0);
          if (++s == S) { s = 0; ph ^= 1u; }
        }
      }
    } else if (conv) {
      const int ct = threadIdx.x - 32;
      int s = 0;
      uint32_t ph = 0;
      for (int i = 0; i < nkb; ++i) {
        mbar_wait(full0 + 8 * s, ph);
        uint8_t* st = smem + s * R.stage;
        if constexpr (MODE == BF16) {
          if (p.a_mn) transpose_tile<true, RAW>(st + R.off_sa, st, 0, BM, ct);
          if (p.b_mn) transpose_tile<true, RAW>(st + R.off_sb, st + R.off_b, 0, BN, ct);
        } else if constexpr (MODE == TF32) {
          if (p.a_mn) transpose_tile<false, BIG>(st + R.off_sa, st, 0, BM, ct);
          if (p.b_mn) transpose_tile<false, BIG>(st + R.off_sb, st + R.off_b, 0, BN, ct);
        } else {
          // a K-major A is split by the consumers in registers
          if (p.a_mn) transpose_tile<false, BIG_SMALL>(st + R.off_sa, st, R.off_as, BM, ct);
          if (p.b_mn) transpose_tile<false, BIG_SMALL>(st + R.off_sb, st + R.off_b, R.off_bs - R.off_b, BN, ct);
          else small_tile(st + R.off_b, st + R.off_bs, BN, ct);
        }
        // generic-proxy stores -> visible to wgmma (async proxy) before the consumers are told
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        __syncwarp();
        if (lane == 0) mbar_arrive(conv0 + 8 * s);
        if (++s == S) { s = 0; ph ^= 1u; }
      }
    }
  } else {
    // ---------------- warpgroups 1-2: wgmma on rows 64 g .. 64 g + 63 of the tile, then the epilogue ----------
    const int g = (warp >> 2) - 1;
    int rs = 0, fs = 0;                // stage of the next k-block to consume / to release
    uint32_t rph = 0;
    auto ready = [&]() -> const uint8_t* {
      mbar_wait(full0 + 8 * rs, rph);
      if (conv) mbar_wait(conv0 + 8 * rs, rph);
      const uint8_t* st = smem + rs * R.stage;
      if (++rs == S) { rs = 0; rph ^= 1u; }
      return st;
    };
    auto release = [&]() {             // the oldest unreleased k-block's wgmma groups have completed
      __syncwarp();
      if (lane == 0) mbar_arrive(empty0 + 8 * fs);
      if (++fs == S) fs = 0;
    };
    float acc[NR];
#pragma unroll
    for (int r = 0; r < NR; ++r) acc[r] = 0.f;
    if constexpr (MODE == X3) {
      float corr[NR], part[NR];
#pragma unroll
      for (int r = 0; r < NR; ++r) { corr[r] = 0.f; part[r] = 0.f; }
      // Per k-block two groups: the main product A_big.B_big from zero into part, then the cross terms
      // A_big.B_small + A_small.B_big into corr.  Once all but the cross group just committed are done, this
      // k-block's main product is folded (fp32 round-to-nearest) while the cross terms run, and the previous
      // k-block's stage is released.  One instruction consumes 32 bytes of K per row (8 tf32): +2 in the
      // (addr >> 4) field of a descriptor.
      if (p.a_mn) {
        // A transposed by the converter: both parts of A from shared memory
        for (int i = 0; i < nkb; ++i) {
          const uint32_t base = smem_u32(ready());
          const uint64_t ad = make_smem_desc(base + g * 64 * 128), bd = make_smem_desc(base + R.off_b),
                         asd = make_smem_desc(base + R.off_as + g * 64 * 128), bsd = make_smem_desc(base + R.off_bs);
          wgmma_fence();
#pragma unroll
          for (int k = 0; k < 4; ++k) wgmma_tf32(part, ad + 2 * k, bd + 2 * k, k > 0 ? 1u : 0u);        // A_big . B_big
          wgmma_commit();
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            wgmma_tf32(corr, ad + 2 * k, bsd + 2 * k, (i > 0 || k > 0) ? 1u : 0u);                    // A_big . B_small
            wgmma_tf32(corr, asd + 2 * k, bd + 2 * k, 1u);                                           // A_small . B_big
          }
          wgmma_commit();
          wgmma_wait1();
#pragma unroll
          for (int r = 0; r < NR; ++r) acc[r] += part[r];
          if (i > 0) release();
        }
        wgmma_wait0();
      } else {
        // K-major A: each thread loads its wgmma fragment of the swizzled tile (rows l/4 and l/4 + 8 of its warp's
        // 16, one 4-byte word of 16-byte chunk c: 8 rows x one chunk per load, the chunks distinct under the
        // swizzle, so conflict-free) and splits it in registers.  One fragment set: it is rewritten only after the
        // previous k-block's cross group has completed (a second set does not fit the 168-register launch bound,
        // which ptxas keeps even under setmaxnreg).  Meanwhile the other warpgroup keeps the tensor cores busy.
        const int ra = g * 64 + (warp & 3) * 16 + (lane >> 2);
        const uint32_t aoff = (uint32_t) ra * 128 + 4 * (lane & 3);
        const int rx = ra & 7;
        uint32_t ab[4][4], as[4][4];
        for (int i = 0; i < nkb; ++i) {
          const uint8_t* st = ready();
          if (i > 0) {
            wgmma_wait0();
            release();
          }
          const float* tile = reinterpret_cast<const float*>(st);
#pragma unroll
          for (int k = 0; k < 4; ++k) {
#pragma unroll
            for (int j = 0; j < 4; ++j) {   // j: row + 8 (j & 1), chunk 2k + (j >> 1)
              const float v = tile[(aoff + 1024 * (j & 1) + (((2 * k + (j >> 1)) ^ rx) << 4)) >> 2];
              ab[k][j] = __float_as_uint(tf32_big(v));
              as[k][j] = __float_as_uint(tf32_small(v));
            }
          }
          const uint32_t base = smem_u32(st);
          const uint64_t bd = make_smem_desc(base + R.off_b), bsd = make_smem_desc(base + R.off_bs);
          wgmma_fence();
#pragma unroll
          for (int k = 0; k < 4; ++k) wgmma_tf32_rs(part, ab[k], bd + 2 * k, k > 0 ? 1u : 0u);          // A_big . B_big
          wgmma_commit();
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            wgmma_tf32_rs(corr, ab[k], bsd + 2 * k, (i > 0 || k > 0) ? 1u : 0u);                      // A_big . B_small
            wgmma_tf32_rs(corr, as[k], bd + 2 * k, 1u);                                             // A_small . B_big
          }
          wgmma_commit();
          wgmma_wait1();
#pragma unroll
          for (int r = 0; r < NR; ++r) acc[r] += part[r];
        }
        wgmma_wait0();
      }
#pragma unroll
      for (int r = 0; r < NR; ++r) acc[r] += corr[r];
    } else {
      for (int i = 0; i < nkb; ++i) {
        const uint32_t base = smem_u32(ready());
        // one instruction consumes 32 bytes of K per row (8 tf32 / 16 bf16): +2 in the (addr >> 4) field
        const uint64_t ad = make_smem_desc(base + g * 64 * 128), bd = make_smem_desc(base + R.off_b);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          if constexpr (MODE == BF16) wgmma_bf16(acc, ad + 2 * k, bd + 2 * k, (i > 0 || k > 0) ? 1u : 0u);
          else wgmma_tf32(acc, ad + 2 * k, bd + 2 * k, (i > 0 || k > 0) ? 1u : 0u);
        }
        wgmma_commit();
        wgmma_wait1();
        if (i > 0) release();
      }
      wgmma_wait0();
    }
    // ---------------- epilogue ----------------
    // Once both warpgroups are past the mainloop the ring is dead (warpgroup 0 finished with it before the last
    // k-block was consumed): the accumulators go through a row-major tile in it.
    // wgmma fragment: d[4j + 2h + e] is row 16 w + lane / 4 + 8 h, column 8 j + 2 (lane % 4) + e of the warpgroup
    constexpr int P = epi_pitch(BN);
    float* tile = reinterpret_cast<float*>(smem);
    consumer_sync();
    {
      float* row = tile + (g * 64 + (warp & 3) * 16 + (lane >> 2)) * P + 2 * (lane & 3);
#pragma unroll
      for (int j = 0; j < BN / 8; ++j)
#pragma unroll
        for (int h = 0; h < 2; ++h)
          *reinterpret_cast<float2*>(row + 8 * h * P + 8 * j) = make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
    }
    consumer_sync();
    // Each thread walks segments of 4 columns x 1 row, in batches: every global load of a batch is issued before its
    // first store, so a thread waits for one round trip to L2 per batch rather than one per element.  A warp covers
    // 512 contiguous bytes of output rows.  Whole, aligned segments take 16-byte accesses; the others (the N tail, or
    // a launch with a misaligned pointer or leading dimension) element by element in the same loop.
    constexpr int SPR = BN / 4;                        // segments per row; divides 256
    constexpr int SEG = BM * SPR / 256;                // segments per thread: 4, 8, 16
    constexpr int BATCH = 4;                           // sized to the 168-register launch bound (worst case 16 / segment)
    const int et = threadIdx.x - 128;
    const int c4 = et % SPR, r0 = et / SPR;            // a thread keeps its columns in every segment
    const int n = n0 + 4 * c4;
    const int nv = min(4, p.N - n);                    // columns of the segment inside N (<= 0: none)
    const bool vec_n = p.vec && nv == 4;
    const float4 bv = (p.bias != nullptr && z == 0 && nv > 0) ? seg_load<true>(p.bias + n, vec_n, nv)
                                                             : make_float4(0.f, 0.f, 0.f, 0.f);
    float cs[4] = {0.f, 0.f, 0.f, 0.f};
    uint64_t dseed = 0, doff = 0;
    if constexpr (DROP) {
      dseed = (uint64_t) p.drop_rng[0];
      doff = (uint64_t) p.drop_rng[1] + (uint64_t) p.drop_layer;
    }
#pragma unroll 1
    for (int b0 = 0; b0 < SEG; b0 += BATCH) {
      float4 mv[BATCH], av[BATCH], yv[BATCH], cv[BATCH];
#pragma unroll
      for (int i = 0; i < BATCH; ++i) {                // loads
        const int m = m0 + r0 + (256 / SPR) * (b0 + i);
        const int k = m < p.M ? nv : 0;
        const bool v = vec_n && m < p.M;
        const int64_t o = (int64_t) m * p.ldc + n;
        const float4 zero = make_float4(0.f, 0.f, 0.f, 0.f);
        mv[i] = p.mul != nullptr ? seg_load<true>(p.mul + o, v, k) : zero;
        av[i] = p.add != nullptr ? seg_load<true>(p.add + o, v, k) : zero;
        yv[i] = p.ybwd != nullptr ? seg_load<true>(p.ybwd + o, v, k) : zero;
        cv[i] = (p.beta && p.splits == 1) ? seg_load<false>(p.c + o, v, k) : zero;   // split-K adds with red.add
      }
#pragma unroll
      for (int i = 0; i < BATCH; ++i) {                // arithmetic and stores
        const int r = r0 + (256 / SPR) * (b0 + i);
        const int m = m0 + r;
        const int k = m < p.M ? nv : 0;
        const bool v = vec_n && m < p.M;
        const int64_t o = (int64_t) m * p.ldc + n;
        const float4 a = *reinterpret_cast<const float4*>(tile + r * P + 4 * c4);
        float4 t = make_float4(__fadd_rn(a.x, bv.x), __fadd_rn(a.y, bv.y), __fadd_rn(a.z, bv.z), __fadd_rn(a.w, bv.w));
        if (p.splits > 1) {        // split-K: partial sums of a plain linear output (C was zeroed by the host)
          seg_red_add(p.c + o, t, v, k);
          continue;
        }
        if (p.c_pre != nullptr) seg_store(p.c_pre + o, t, v, k);
        uint32_t kb = 0;       // keep bits of the segment's elements: one Philox call when it starts on a group
        if constexpr (DROP) {
          if (k > 0) kb = b2_drop_keep4(dseed, doff, (uint64_t) m * (uint64_t) p.N + (uint64_t) n, k, p.drop_thresh);
        }
        t.x = epilogue_elem<DROP, LEAKY>(p, t.x, mv[i].x, av[i].x, yv[i].x, cv[i].x, kb & 1u);
        t.y = epilogue_elem<DROP, LEAKY>(p, t.y, mv[i].y, av[i].y, yv[i].y, cv[i].y, kb & 2u);
        t.z = epilogue_elem<DROP, LEAKY>(p, t.z, mv[i].z, av[i].z, yv[i].z, cv[i].z, kb & 4u);
        t.w = epilogue_elem<DROP, LEAKY>(p, t.w, mv[i].w, av[i].w, yv[i].w, cv[i].w, kb & 8u);
        seg_store(p.c + o, t, v, k);
        if (p.c_small != nullptr) {
          const int64_t oa = (int64_t) m * p.ld_aux + n;
          if (p.esz == 4)          // the consumer's 3xTF32 small part, produced where C is
            seg_store(p.c_small + oa, make_float4(tf32_small(t.x), tf32_small(t.y), tf32_small(t.z), tf32_small(t.w)), v, k);
          else                     // bf16 mode operand
            seg_store_bf16(reinterpret_cast<__nv_bfloat16*>(p.c_small) + oa, t, v, k);
        }
        if (k > 0) cs[0] += t.x;
        if (k > 1) cs[1] += t.y;
        if (k > 2) cs[2] += t.z;
        if (k > 3) cs[3] += t.w;
      }
    }
    if (p.colsum != nullptr) {
      // bias gradient: the threads' partial sums meet in shared memory past the tile; one red.add per column and CTA
      float* part = tile + BM * P;
      *reinterpret_cast<float4*>(part + 4 * et) = make_float4(cs[0], cs[1], cs[2], cs[3]);
      consumer_sync();
      if (et < BN && n0 + et < p.N) {
        float s = 0.f;
#pragma unroll
        for (int u = et >> 2; u < 256; u += SPR) s += part[4 * u + (et & 3)];
        b2_red_add(p.colsum + n0 + et, s);
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

// ---------------------------------------------------------------------------------
// Operand preparation for the K-major tensor-core GEMMs, one pass over a (R, C) matrix:
//   v      = act'(y) * x          (act-backward fused when y != NULL; y is the activation OUTPUT)
//   out    = v            (R, C)            out_small  = tf32_small(v)
//   outT   = v^T          (C, R)            outT_small = tf32_small(v^T)
//   colsum[c] += sum_r v[r, c]              (bias gradient)
// Any output pointer may be NULL, but outT_small comes with outT.  32 x 32 tiles through padded shared memory.
// DROP: x is the gradient of a dropout layer's output, y that dropped output: v = act'(y) * keep * scale * x
// (the mask first; sigmoid's s = y / scale on kept elements).
// ---------------------------------------------------------------------------------
template <bool DROP, bool LEAKY>      // LEAKY: the twin that also knows B2_ACT_LEAKY_RELU (as the GEMM's)
__global__ void __launch_bounds__(256)
prep_operand_kernel(const float* __restrict__ x, const float* __restrict__ y, int act, int64_t R,
                    int64_t C, int64_t ld_in, float* __restrict__ out, float* __restrict__ out_small,
                    float* __restrict__ outT, float* __restrict__ outT_small, float* __restrict__ colsum,
                    const int64_t* __restrict__ drop_rng, int64_t drop_layer, uint32_t drop_thresh, float drop_scale) {
  b2_pdl_wait();
  b2_pdl_trigger();
  __shared__ float tile[32][33];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;  // 32 x 8
  const int64_t c0 = (int64_t) blockIdx.x * 32, r0 = (int64_t) blockIdx.y * 32;
  uint64_t dseed = 0, doff = 0;
  if constexpr (DROP) {
    dseed = (uint64_t) drop_rng[0];
    doff = (uint64_t) drop_rng[1] + (uint64_t) drop_layer;
  }
#pragma unroll
  for (int i = 0; i < 32; i += 8) {
    const int64_t r = r0 + ty + i, c = c0 + tx;
    float v = 0.f;
    if (r < R && c < C) {
      v = __ldg(x + r * ld_in + c);
      if constexpr (DROP)
        v = b2_drop_keep(dseed, doff, (uint64_t) (r * C + c), drop_thresh) ? __fmul_rn(v, drop_scale) : 0.f;
      if (y != nullptr) {
        const float yv = __ldg(y + r * ld_in + c);
        if (act == B2_ACT_RELU) v = (yv > 0.f) ? v : 0.f;
        else if (act == B2_ACT_SIGMOID) {
          const float s = DROP ? __fdiv_rn(yv, drop_scale) : yv;
          v = v * ((1.f - s) * s);
        }
        else if (act == B2_PREP_MUL) v = v * yv;
        if constexpr (LEAKY) {
          if (act == B2_ACT_LEAKY_RELU) v = (yv > 0.f) ? v : __fmul_rn(v, B2_LEAKY_SLOPE);
        }
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
//   DROP: the previous layer ends on dropout, x is its dropped output: its mask multiplies gx before prev_act'.
// ---------------------------------------------------------------------------------
template <bool LEAKY>
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
      if constexpr (LEAKY) {
        if (act == B2_ACT_LEAKY_RELU) v = v > 0.f ? v : __fmul_rn(v, B2_LEAKY_SLOPE);
      }
      y[m] = v;
    }
  }
}

// CTA = 256 threads = 8 warps; each CTA owns a contiguous block of rows; lane k-strided columns.
template <bool DROP, bool LEAKY>
__global__ void __launch_bounds__(256)
head_bwd_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ y,
                const float* __restrict__ gy, int64_t M, int K, int act, int64_t rows_per_cta,
                float* __restrict__ gx, float* __restrict__ gw, float* __restrict__ gb, int prev_act,
                float* __restrict__ gx_small, float* __restrict__ gb_prev,
                const int64_t* __restrict__ drop_rng, int64_t drop_layer, uint32_t drop_thresh, float drop_scale) {
  b2_pdl_wait();
  b2_pdl_trigger();
  uint64_t dseed = 0, doff = 0;
  if constexpr (DROP) {
    dseed = (uint64_t) drop_rng[0];
    doff = (uint64_t) drop_rng[1] + (uint64_t) drop_layer;
  }
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
        if constexpr (LEAKY) {
          if (act == B2_ACT_LEAKY_RELU) gz = (yv > 0.f) ? gz : __fmul_rn(gz, B2_LEAKY_SLOPE);
        }
      }
      if (kb == 0 && lane == 0) gb_acc += gz;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int k = kb + j * 32 + lane;
        if (k < K) {
          const float xv = __ldg(x + m * K + k);
          if (gx != nullptr) {
            float val = gz * __ldg(w + k);
            if constexpr (DROP)
              val = b2_drop_keep(dseed, doff, (uint64_t) m * (uint64_t) K + (uint64_t) k, drop_thresh)
                        ? __fmul_rn(val, drop_scale) : 0.f;
            if (prev_act == B2_ACT_RELU) val = (xv > 0.f) ? val : 0.f;
            else if (prev_act == B2_ACT_SIGMOID) {
              const float s = DROP ? __fdiv_rn(xv, drop_scale) : xv;
              val = val * ((1.f - s) * s);
            }
            if constexpr (LEAKY) {
              if (prev_act == B2_ACT_LEAKY_RELU) val = (xv > 0.f) ? val : __fmul_rn(val, B2_LEAKY_SLOPE);
            }
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

// ---------------------------------------------------------------------------------
// Dropout RNG state and the elementwise mask (philox.cuh).
//   rng_take: snapshot = state; state.offset += n_layers   (one thread: one per chain forward with dropout)
//   apply:    y[m, n] = keep(m, n) ? x[m, n] * scale : 0   (one Philox call per element group of 4)
// ---------------------------------------------------------------------------------
__global__ void dropout_rng_take_kernel(int64_t* __restrict__ state, int64_t* __restrict__ snapshot, int n_layers) {
  b2_pdl_wait();
  b2_pdl_trigger();
  const int64_t seed = state[0], off = state[1];
  snapshot[0] = seed;
  snapshot[1] = off;
  state[1] = (int64_t) ((uint64_t) off + (uint64_t) n_layers);
}

__global__ void __launch_bounds__(256)
dropout_apply_kernel(const float* x, float* y, int64_t M, int64_t N, int64_t ld,     // y may be x (in place)
                     const int64_t* __restrict__ drop_rng, int64_t drop_layer, uint32_t thresh, float scale) {
  b2_pdl_wait();
  b2_pdl_trigger();
  const uint64_t seed = (uint64_t) drop_rng[0], off = (uint64_t) drop_rng[1] + (uint64_t) drop_layer;
  const int64_t n_el = M * N, groups = (n_el + 3) >> 2;
  for (int64_t g = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; g < groups; g += (int64_t) gridDim.x * blockDim.x) {
    const b2_u32x4 r = b2_drop_group(seed, off, (uint64_t) g);
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int64_t i = 4 * g + e;
      if (i < n_el) {
        const int64_t m = i / N, o = m * ld + (i - m * N);
        y[o] = r.v[e] < thresh ? __fmul_rn(x[o], scale) : 0.f;
      }
    }
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
// K-major boxes land 128B-swizzled, the layout wgmma reads; MN-major ones unswizzled, for the converter to transpose.
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
                   mn_major ? CU_TENSOR_MAP_SWIZZLE_NONE : CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return b2_fail(B2_E_CUDA, "cuTensorMapEncodeTiled failed with CUresult %d", (int) r);
  return B2_OK;
}

static bool tma_ok_e(const void* p, int64_t ld, int esz) {
  return (reinterpret_cast<uintptr_t>(p) % 16 == 0) && ((ld * esz) % 16 == 0);
}
static bool tma_ok(const float* p, int64_t ld) { return tma_ok_e(p, ld, 4); }

// plan != NULL: fill in the launch plan (tile shape, ring depths, shared memory) and return without
// touching the device — pure host arithmetic, so the CPU test-suite can sweep it (tests/test_abi.py).
template <int BN, int MODE, bool DROP, bool LEAKY>
static int gemm_launch(const tc::Params& p, int grid, cudaStream_t st) {
  void (*kern)(tc::Params) = tc::gemm_tc_kernel<BN, MODE, DROP, LEAKY>;
  // opt-in to > 48 KB of dynamic shared memory, for the largest ring this instantiation launches with: an
  // idempotent per-process property (C++11 guarantees the initialiser runs once, thread-safely)
  static const cudaError_t attr_rc =
      cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) tc::ring_smem_max(BN, MODE));
  if (attr_rc != cudaSuccess) return b2_fail(B2_E_CUDA, "b2_gemm_tc_ex: smem attribute: %s", cudaGetErrorString(attr_rc));
  B2_REQUIRE(p.ring.smem <= tc::ring_smem_max(BN, MODE), "ring exceeds the shared-memory attribute");
  B2_LAUNCH(kern, grid, tc::NTHREADS, p.ring.smem, st, p);
  B2_CUDA_LAUNCH_CHECK("b2_gemm_tc_ex");
  return B2_OK;
}

// One kernel instantiation per tile width and arithmetic mode (tf32 and bf16 single pass, 3xTF32 up to bn = 64),
// per dropout (a launch with a dropout mask in its epilogue runs the DROP twin of its instantiation) and per
// LeakyReLU (a launch with B2_ACT_LEAKY_RELU as act or act_bwd runs the LEAKY twin, so no other launch pays for it).
typedef int (*GemmLaunch)(const tc::Params&, int, cudaStream_t);
template <bool DROP, bool LEAKY>
static GemmLaunch gemm_inst_t(int bn, int mode) {
  switch (bn * 4 + mode) {
    case 32 * 4 + tc::TF32: return gemm_launch<32, tc::TF32, DROP, LEAKY>;
    case 64 * 4 + tc::TF32: return gemm_launch<64, tc::TF32, DROP, LEAKY>;
    case 128 * 4 + tc::TF32: return gemm_launch<128, tc::TF32, DROP, LEAKY>;
    case 32 * 4 + tc::BF16: return gemm_launch<32, tc::BF16, DROP, LEAKY>;
    case 64 * 4 + tc::BF16: return gemm_launch<64, tc::BF16, DROP, LEAKY>;
    case 128 * 4 + tc::BF16: return gemm_launch<128, tc::BF16, DROP, LEAKY>;
    case 32 * 4 + tc::X3: return gemm_launch<32, tc::X3, DROP, LEAKY>;
    case 64 * 4 + tc::X3: return gemm_launch<64, tc::X3, DROP, LEAKY>;
    default: return nullptr;
  }
}
static GemmLaunch gemm_inst(int bn, int mode, bool drop, bool leaky) {
  if (leaky) return drop ? gemm_inst_t<true, true>(bn, mode) : gemm_inst_t<false, true>(bn, mode);
  return drop ? gemm_inst_t<true, false>(bn, mode) : gemm_inst_t<false, false>(bn, mode);
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
  B2_REQUIRE(b2_act_ok(d->act), "bad activation code %d", d->act);
  B2_REQUIRE(b2_act_ok(d->act_bwd), "bad act_bwd code %d", d->act_bwd);
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
  const bool drop = d->drop_rng != nullptr;
  B2_REQUIRE(!drop || (d->drop_scale > 0.f && d->drop_scale < 3.0e38f && d->drop_layer >= 0),
             "dropout needs a positive finite scale and a layer index >= 0");
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
                       d->c_small == nullptr && d->c_pre == nullptr && d->colsum == nullptr && !drop);
  const bool backfill = (d->flags & B2_GEMM_BACKFILL) != 0;
  int best_bn = 0, best_split = 1;
  double best_cost = 1e300;
  const int bn_max = three_pass ? 64 : 128;
  for (int bn = 32; bn <= bn_max; bn *= 2) {
    // Cycles per k-block: the larger of the tensor pipe — passes x 2 warpgroups x 4 instructions x bn/2 (an
    // m64nBNk8 tf32 takes bn/2 cycles of the SM's tensor cores, which the two warpgroups share) — and shared memory
    // at 128 B (one tile row) a cycle.  Shared-memory rows: TMA writes A and B; the converter reads and writes an
    // MN-major tile again, and in 3xTF32 writes the small part of B and of an MN-major A (a K-major B is read
    // once more for it; a K-major A is split in registers); wgmma reads bn rows of B per pass and warpgroup, and
    // 64 rows of A — per pass from shared memory, or once into registers for a K-major A in 3xTF32.
    const bool mn_a = d->a_mn_major != 0, mn_b = d->b_mn_major != 0;
    const double passes = three_pass ? 3.0 : 1.0;
    const double rows_tma = tc::BM + bn;
    const double rows_conv = (mn_a ? 2.0 : 0.0) * tc::BM + (mn_b ? 2.0 : 0.0) * bn +
                             (three_pass ? (mn_a ? 1.0 : 0.0) * tc::BM + (mn_b ? 1.0 : 2.0) * bn : 0.0);
    const double rows_mma = passes * 2.0 * bn + (three_pass && !mn_a ? 1.0 : passes) * tc::BM;
    const double per_kb = fmax(passes * 4.0 * bn, rows_tma + rows_conv + rows_mma);
    const int64_t tiles_n = b2_ceil_div(N, bn);
    for (int split = 1; split <= 32; split *= 2) {
      if (split > 1 && (!linear || num_kb / split < 8)) break;
      const int64_t ctas = tiles_m * tiles_n * split;
      const int64_t waves = b2_ceil_div(ctas, B2_NUM_SMS);
      const double kb = (double) b2_ceil_div(num_kb, split);
      const double cost = (double) waves * (10000.0 + kb * per_kb);
      if (cost < best_cost) { best_cost = cost; best_bn = bn; best_split = split; }
    }
  }
  if (backfill && linear) {
    // A backfill launch fills the SMs a chain of launches on another stream leaves idle, so its own wave count does
    // not matter; what does is how long one of its CTAs holds an SM the chain's next launch wants.  Same tile width,
    // and the most K splits (up to 32) that leave every CTA at least BACKFILL_KB k-blocks, never fewer than the plain
    // plan's.  Measured on the DeepFM C2 MLP backward (H100 80GB HBM3, 400 W): floors of 32 / 16 / 8 / 4 k-blocks took
    // 217 / 191 / 206 / 225 us.
    while (best_split < 32 && num_kb / (2 * best_split) >= tc::BACKFILL_KB) best_split *= 2;
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
  p.drop_rng = d->drop_rng; p.drop_layer = d->drop_layer; p.drop_thresh = d->drop_thresh; p.drop_scale = d->drop_scale;
  {
    auto al = [](const void* q, uintptr_t b) { return reinterpret_cast<uintptr_t>(q) % b == 0; };
    p.vec = al(c, 16) && ldc % 4 == 0 && al(d->c_pre, 16) && al(d->bias, 16) && al(d->mul, 16) &&
            al(d->add, 16) && al(d->ybwd, 16) && al(d->c_small, esz == 4 ? 16 : 8) &&
            (d->c_small == nullptr || ld_aux % 4 == 0);
  }
  p.kb_per_split = (int) b2_ceil_div(num_kb, best_split);
  const int splits = (int) b2_ceil_div(num_kb, p.kb_per_split);
  const int64_t tiles_n = b2_ceil_div(N, best_bn);
  const int64_t total_tiles = tiles_m * tiles_n * splits;
  B2_REQUIRE(total_tiles < (1ll << 31), "too many tiles");
  p.tiles_m = (int) tiles_m; p.tiles_n = (int) tiles_n; p.splits = splits;
  const int mode = three_pass ? tc::X3 : (esz == 2 ? tc::BF16 : tc::TF32);
  const GemmLaunch launch = gemm_inst(best_bn, mode, drop,
                                       d->act == B2_ACT_LEAKY_RELU || d->act_bwd == B2_ACT_LEAKY_RELU);
  B2_REQUIRE(launch != nullptr, "no GEMM instantiation for bn %d", best_bn);
  p.ring = tc::ring_layout(best_bn, mode, p.a_mn != 0, p.b_mn != 0);
  B2_REQUIRE(p.ring.stages >= 2 && p.ring.smem <= tc::SMEM_MAX, "tile does not fit shared memory");
  if (plan != nullptr) {
    plan->bn = best_bn; plan->splits = splits; plan->stages = p.ring.stages; plan->cstages = p.ring.stages;
    plan->grid = (int) total_tiles; plan->threads = tc::NTHREADS; plan->tiles_m = p.tiles_m; plan->tiles_n = p.tiles_n;
    plan->passes = three_pass ? 3 : 1; plan->kb_per_split = p.kb_per_split; plan->smem_bytes = (int64_t) p.ring.smem;
    return B2_OK;
  }
  if (splits > 1 && !p.beta && !(d->flags & B2_GEMM_C_IS_ZERO)) {
    cudaError_t e = cudaMemset2DAsync(c, (size_t) ldc * 4, 0, (size_t) N * 4, (size_t) M, st);
    if (e != cudaSuccess) return b2_fail(B2_E_CUDA, "b2_gemm_tc_ex: memset: %s", cudaGetErrorString(e));
  }
  if (d->colsum != nullptr && !(d->flags & B2_GEMM_COLSUM_IS_ZERO)) {
    cudaError_t e = cudaMemsetAsync(d->colsum, 0, sizeof(float) * (size_t) N, st);
    if (e != cudaSuccess) return b2_fail(B2_E_CUDA, "b2_gemm_tc_ex: memset: %s", cudaGetErrorString(e));
  }
  return launch(p, (int) total_tiles, st);
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

extern "C" B2_API int b2_split_tf32(const float* x, float* small, int64_t n, void* stream) {
  B2_REQUIRE(x && small, "NULL pointer");
  if (n <= 0) return B2_OK;
  int64_t blocks = b2_ceil_div(n, 256);
  if (blocks > (int64_t) B2_NUM_SMS * 8) blocks = (int64_t) B2_NUM_SMS * 8;
  B2_LAUNCH(tc::split_tf32_kernel, (int) blocks, 256, 0, (cudaStream_t) stream, x, small, n);
  B2_CUDA_LAUNCH_CHECK("b2_split_tf32");
  return B2_OK;
}

// The dropout arguments shared by the entry points that apply a mask: drop_rng == NULL means no dropout.
static int check_drop(const int64_t* drop_rng, int64_t drop_layer, float drop_scale) {
  B2_REQUIRE(drop_rng == nullptr || (drop_scale > 0.f && drop_scale < 3.0e38f && drop_layer >= 0),
             "dropout needs a positive finite scale and a layer index >= 0");
  return B2_OK;
}

extern "C" B2_API int b2_prep_operand(const float* x, const float* y, int act, int64_t R, int64_t C,
                                      float* out, float* out_small, float* outT, float* outT_small,
                                      float* colsum, const int64_t* drop_rng, int64_t drop_layer,
                                      uint32_t drop_thresh, float drop_scale, void* stream) {
  B2_REQUIRE(x != nullptr, "NULL input");
  B2_REQUIRE(R >= 0 && C >= 0, "bad shape");
  B2_REQUIRE(b2_act_ok(act) || act == B2_PREP_MUL, "bad activation code %d", act);
  B2_REQUIRE(drop_rng == nullptr || act != B2_PREP_MUL, "B2_PREP_MUL takes no dropout mask");
  B2_REQUIRE(outT_small == nullptr || outT != nullptr, "outT_small needs outT");
  const int rc = check_drop(drop_rng, drop_layer, drop_scale);
  if (rc != B2_OK) return rc;
  cudaStream_t st = (cudaStream_t) stream;
  if (colsum != nullptr) {
    cudaError_t e = cudaMemsetAsync(colsum, 0, sizeof(float) * (size_t) C, st);
    if (e != cudaSuccess) return b2_fail(B2_E_CUDA, "b2_prep_operand: memset: %s", cudaGetErrorString(e));
  }
  if (R == 0 || C == 0) return B2_OK;
  dim3 grid((unsigned) b2_ceil_div(C, 32), (unsigned) b2_ceil_div(R, 32));
  B2_REQUIRE(grid.y <= 65535, "too many rows for this launch geometry");
#define PREP_LAUNCH(DROP, LEAKY)                                                                                 \
  B2_LAUNCH((tc::prep_operand_kernel<DROP, LEAKY>), grid, 256, 0, st, x, y, act, R, C, C, out, out_small, outT,      \
            outT_small, colsum, drop_rng, drop_layer, drop_thresh, drop_scale)
  if (act == B2_ACT_LEAKY_RELU) {
    if (drop_rng != nullptr) PREP_LAUNCH(true, true);
    else PREP_LAUNCH(false, true);
  } else {
    if (drop_rng != nullptr) PREP_LAUNCH(true, false);
    else PREP_LAUNCH(false, false);
  }
#undef PREP_LAUNCH
  B2_CUDA_LAUNCH_CHECK("b2_prep_operand");
  return B2_OK;
}

extern "C" B2_API int b2_head_fwd(const float* x, const float* w, const float* b, int64_t M, int K, int act,
                                  float* y, void* stream) {
  B2_REQUIRE(x && w && y, "NULL pointer");
  B2_REQUIRE(K >= 1 && b2_act_ok(act), "bad K/act");
  if (M <= 0) return B2_OK;
  int64_t blocks = b2_ceil_div(M * 32, 256);
  if (blocks > (int64_t) B2_NUM_SMS * 8) blocks = (int64_t) B2_NUM_SMS * 8;
  if (act == B2_ACT_LEAKY_RELU)
    B2_LAUNCH(tc::head_fwd_kernel<true>, (int) blocks, 256, 0, (cudaStream_t) stream, x, w, b, M, K, act, y);
  else
    B2_LAUNCH(tc::head_fwd_kernel<false>, (int) blocks, 256, 0, (cudaStream_t) stream, x, w, b, M, K, act, y);
  B2_CUDA_LAUNCH_CHECK("b2_head_fwd");
  return B2_OK;
}

extern "C" B2_API int b2_head_bwd(const float* x, const float* w, const float* y, const float* gy, int64_t M,
                                  int K, int act, float* gx, float* gw, float* gb, void* stream) {
  return b2_head_bwd_ex(x, w, y, gy, M, K, act, gx, gw, gb, B2_ACT_NONE, nullptr, nullptr, 0, nullptr, 0, 0, 0.f,
                        stream);
}

// head_bwd_kernel stages 2 * K floats (the partial sums of gw and gb_prev) in dynamic shared memory.  A launch whose
// dynamic and static shared memory together pass the default 48 KB per block needs the instantiation's opt-in first.
template <bool DROP, bool LEAKY>
static int head_bwd_smem_optin(size_t dyn) {
  const void* kern = (const void*) tc::head_bwd_kernel<DROP, LEAKY>;
  cudaFuncAttributes fa;
  cudaError_t e = cudaFuncGetAttributes(&fa, kern);
  if (e == cudaSuccess && fa.sharedSizeBytes + dyn > 48 * 1024)
    e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) dyn);
  if (e != cudaSuccess) return b2_fail(B2_E_CUDA, "b2_head_bwd: smem attribute: %s", cudaGetErrorString(e));
  return B2_OK;
}

extern "C" B2_API int b2_head_bwd_ex(const float* x, const float* w, const float* y, const float* gy, int64_t M,
                                     int K, int act, float* gx, float* gw, float* gb, int prev_act,
                                     float* gx_small, float* gb_prev, int grads_zeroed, const int64_t* prev_drop_rng,
                                     int64_t prev_drop_layer, uint32_t prev_drop_thresh, float prev_drop_scale,
                                     void* stream) {
  B2_REQUIRE(x && w && gy && gw, "NULL pointer");
  B2_REQUIRE(K >= 1 && K <= B2_HEAD_MAX_K, "K=%d outside [1, B2_HEAD_MAX_K=%d]", K, B2_HEAD_MAX_K);
  B2_REQUIRE(b2_act_ok(act), "bad activation code %d", act);
  B2_REQUIRE(b2_act_ok(prev_act), "bad prev_act");
  B2_REQUIRE(act == B2_ACT_NONE || y != nullptr, "activation backward needs y");
  B2_REQUIRE(gx != nullptr || (gx_small == nullptr && gb_prev == nullptr && prev_act == B2_ACT_NONE &&
                               prev_drop_rng == nullptr),
             "prev_act / gx_small / gb_prev / a dropout mask need gx");
  const int rc = check_drop(prev_drop_rng, prev_drop_layer, prev_drop_scale);
  if (rc != B2_OK) return rc;
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
  const size_t smem = 2 * sizeof(float) * (size_t) K;
  const bool leaky = act == B2_ACT_LEAKY_RELU || prev_act == B2_ACT_LEAKY_RELU;
#define HEAD_BWD(DROP, LEAKY)                                                                                      \
  do {                                                                                                             \
    const int smem_rc = head_bwd_smem_optin<DROP, LEAKY>(smem);                                                    \
    if (smem_rc != B2_OK) return smem_rc;                                                                          \
    B2_LAUNCH((tc::head_bwd_kernel<DROP, LEAKY>), (int) ctas, 256, smem, st, x, w, y_arg, gy, M, K, act,           \
              rows_per_cta, gx, gw, gb, prev_act, gx_small, gb_prev, prev_drop_rng, prev_drop_layer,               \
              prev_drop_thresh, prev_drop_scale);                                                                  \
  } while (0)
  if (leaky) {
    if (prev_drop_rng != nullptr) HEAD_BWD(true, true);
    else HEAD_BWD(false, true);
  } else {
    if (prev_drop_rng != nullptr) HEAD_BWD(true, false);
    else HEAD_BWD(false, false);
  }
#undef HEAD_BWD
  B2_CUDA_LAUNCH_CHECK("b2_head_bwd");
  return B2_OK;
}

extern "C" B2_API int b2_dropout_rng_take(int64_t* state, int64_t* snapshot, int n_layers, void* stream) {
  B2_REQUIRE(state && snapshot, "NULL pointer");
  B2_REQUIRE(n_layers >= 1, "n_layers must be >= 1");
  B2_LAUNCH(tc::dropout_rng_take_kernel, 1, 1, 0, (cudaStream_t) stream, state, snapshot, n_layers);
  B2_CUDA_LAUNCH_CHECK("b2_dropout_rng_take");
  return B2_OK;
}

extern "C" B2_API int b2_dropout_apply(const float* x, float* y, int64_t M, int64_t N, int64_t ld,
                                       const int64_t* snapshot, int64_t layer, uint32_t thresh, float scale,
                                       void* stream) {
  B2_REQUIRE(x && y && snapshot, "NULL pointer");
  B2_REQUIRE(M >= 0 && N >= 0 && ld >= N, "bad shape");
  const int rc = check_drop(snapshot, layer, scale);
  if (rc != B2_OK) return rc;
  if (M == 0 || N == 0) return B2_OK;
  int64_t blocks = b2_ceil_div(b2_ceil_div(M * N, 4), 256);
  if (blocks > (int64_t) B2_NUM_SMS * 8) blocks = (int64_t) B2_NUM_SMS * 8;
  B2_LAUNCH(tc::dropout_apply_kernel, (int) blocks, 256, 0, (cudaStream_t) stream, x, y, M, N, ld, snapshot, layer,
            thresh, scale);
  B2_CUDA_LAUNCH_CHECK("b2_dropout_apply");
  return B2_OK;
}

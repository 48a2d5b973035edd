// adam_common.cuh — the ONE definition of the Adam element update, shared by the dense arena pass
// (dense.cu) and the lazy row-wise kernels (lazy_adam.cu, fused_front.cu).  Explicit round-to-nearest
// intrinsics (no compiler-chosen FMA contraction) make the dense and the lazy evaluation of the same
// update sequence bit-identical.
//
// torch.optim.Adam (single tensor, defaults; called from BaseModel.train_step,
// fuxictr/pytorch/models/rank_model.py:322):
//   exp_avg.lerp_(g, 1-b1); exp_avg_sq.mul_(b2).addcmul_(g, g, 1-b2)
//   denom = exp_avg_sq.sqrt() / sqrt(1-b2^t) + eps;  p.addcdiv_(exp_avg, denom, -lr/(1-b1^t))
#pragma once
#include <cuda_runtime.h>

// 1 - beta is taken in double from the caller's double beta and rounded to fp32 once, as torch rounds the
// Python float 1 - beta2 it passes to addcmul_ (adam_const in dense.cu, make_const in lazy_adam.cu and
// LazyTables._new_ctx in arena.py form the same three floats).
struct B2AdamConst {
  float w1;    // fl32(1 - beta1)
  float b2;    // fl32(beta2)
  float w2;    // fl32(1 - beta2)
  float eps;
};

// per optimizer step t (1-based): sched[t] = { lr / (1 - beta1^t), 1 / sqrt(1 - beta2^t) }
typedef float2 B2AdamSched;

__device__ __forceinline__ void b2_adam_apply(float& p, float g, float& m, float& v,
                                              const B2AdamConst& c, float step_size, float inv_bc2_sqrt) {
  m = __fmaf_rn(__fsub_rn(g, m), c.w1, m);
  v = __fmaf_rn(__fmul_rn(c.w2, g), g, __fmul_rn(v, c.b2));
  const float denom = __fmaf_rn(__fsqrt_rn(v), inv_bc2_sqrt, c.eps);
  p = __fsub_rn(p, __fmul_rn(step_size, __fdiv_rn(m, denom)));
}

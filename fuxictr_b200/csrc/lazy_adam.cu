// lazy_adam.cu — row-wise evaluation of the reference's DENSE Adam semantics for embedding tables
// (see b2_lazy_ctx in include/fuxictr_b200.h), sm_90a.
//
// BaseModel.train_step (fuxictr/pytorch/models/rank_model.py:321-322) clips and then lets
// torch.optim.Adam update EVERY row of every table, although only ~B*F rows carry a gradient.  A row
// that received no gradient at step k still changes (m *= b1, v *= b2, p -= lr_k*m/(sqrt(v)/c_k+eps)),
// so skipping it changes the training trajectory.  These kernels keep the trajectory bit-identical
// while touching only the rows a batch touches: each row remembers the step it is current for, and
// the missed zero-gradient updates are REPLAYED (same scalars sched[k], same rounded arithmetic,
// adam_common.cuh) right before the row is read (fused_front.cu) or really updated (here).
// HBM-bound on O(batch) rows instead of O(vocabulary): 4 x 64 B per touched D=16 row.
#include "b2_common.cuh"
#include "adam_common.cuh"

namespace {
__device__ __forceinline__ int find_table(const b2_lazy_table* __restrict__ t, int n, int64_t grow) {
  int lo = 0, hi = n;  // invariant: t[lo].grow_base <= grow < t[hi].grow_base
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (t[mid].grow_base <= grow) lo = mid; else hi = mid;
  }
  return lo;
}

// one 4-lane group per enqueued row (a D=16 row is 4 float4; D=1 rows use lane 0 only)
__global__ void __launch_bounds__(256)
lazy_sumsq_kernel(const b2_lazy_table* __restrict__ tables, int ntables,
                  const int32_t* __restrict__ worklist, const int32_t* __restrict__ counter, int capacity,
                  int64_t delta_g, float* __restrict__ sumsq) {
  __shared__ float red[32];
  const int n = min(*counter, capacity);
  const int sub = threadIdx.x & 3;
  float acc = 0.f;
  for (int64_t i = ((int64_t) blockIdx.x * blockDim.x + threadIdx.x) >> 2; i < n;
       i += ((int64_t) gridDim.x * blockDim.x) >> 2) {
    const int64_t grow = worklist[i];
    const b2_lazy_table tb = tables[find_table(tables, ntables, grow)];
    const float* g = tb.param + (grow - tb.grow_base) * tb.dim + delta_g;
    for (int e = sub; e < tb.dim; e += 4) {
      const float v = g[e];
      acc = fmaf(v, v, acc);
    }
  }
  const float t = b2_block_sum(acc, red);
  if (threadIdx.x == 0 && t != 0.f) b2_red_add(sumsq, t);
}

__global__ void __launch_bounds__(256)
lazy_adam_kernel(const b2_lazy_table* __restrict__ tables, int ntables,
                 const int32_t* __restrict__ worklist, const int32_t* __restrict__ counter, int capacity,
                 int64_t delta_g, int64_t delta_m, int64_t delta_v, int32_t* __restrict__ last_step,
                 const B2AdamSched* __restrict__ sched, const int64_t* __restrict__ step_dev,
                 const float* __restrict__ sumsq, float max_norm, B2AdamConst c) {
  extern __shared__ b2_lazy_table stab[];
  for (int i = threadIdx.x; i < ntables; i += blockDim.x) stab[i] = tables[i];
  __syncthreads();
  tables = stab;
  const int n = min(*counter, capacity);
  const int t = (int) *step_dev;                  // the step being applied (already incremented)
  float clip = 1.f;
  if (sumsq != nullptr) clip = fminf(max_norm / (sqrtf(*sumsq) + 1e-6f), 1.f);
  const B2AdamSched now = sched[t];
  const int sub = threadIdx.x & 3;
  for (int64_t i = ((int64_t) blockIdx.x * blockDim.x + threadIdx.x) >> 2; i < n;
       i += ((int64_t) gridDim.x * blockDim.x) >> 2) {
    const int64_t grow = worklist[i];
    const b2_lazy_table tb = tables[find_table(tables, ntables, grow)];
    float* p = tb.param + (grow - tb.grow_base) * tb.dim;
    const int last = last_step[grow];
    if ((tb.dim & 3) == 0 && (delta_g & 3) == 0 && (delta_m & 3) == 0 && (delta_v & 3) == 0 &&
        (reinterpret_cast<uintptr_t>(p) & 15) == 0) {
      for (int e = sub * 4; e < tb.dim; e += 16) {   // 16-byte accesses: a D=16 row is one float4 per lane
        float4 pv = *reinterpret_cast<float4*>(p + e), mv = *reinterpret_cast<float4*>(p + e + delta_m);
        float4 vv = *reinterpret_cast<float4*>(p + e + delta_v), gv = *reinterpret_cast<float4*>(p + e + delta_g);
        for (int k = last + 1; k < t; ++k) {
          const B2AdamSched sc = sched[k];
          b2_adam_apply(pv.x, 0.f, mv.x, vv.x, c, sc.x, sc.y);
          b2_adam_apply(pv.y, 0.f, mv.y, vv.y, c, sc.x, sc.y);
          b2_adam_apply(pv.z, 0.f, mv.z, vv.z, c, sc.x, sc.y);
          b2_adam_apply(pv.w, 0.f, mv.w, vv.w, c, sc.x, sc.y);
        }
        b2_adam_apply(pv.x, __fmul_rn(gv.x, clip), mv.x, vv.x, c, now.x, now.y);
        b2_adam_apply(pv.y, __fmul_rn(gv.y, clip), mv.y, vv.y, c, now.x, now.y);
        b2_adam_apply(pv.z, __fmul_rn(gv.z, clip), mv.z, vv.z, c, now.x, now.y);
        b2_adam_apply(pv.w, __fmul_rn(gv.w, clip), mv.w, vv.w, c, now.x, now.y);
        *reinterpret_cast<float4*>(p + e) = pv;
        *reinterpret_cast<float4*>(p + e + delta_m) = mv;
        *reinterpret_cast<float4*>(p + e + delta_v) = vv;
        *reinterpret_cast<float4*>(p + e + delta_g) = make_float4(0.f, 0.f, 0.f, 0.f);
      }
    } else {
      for (int e = sub; e < tb.dim; e += 4) {
        float pv = p[e], mv = p[e + delta_m], vv = p[e + delta_v];
        for (int k = last + 1; k < t; ++k) {        // missed zero-gradient steps
          const B2AdamSched sc = sched[k];
          b2_adam_apply(pv, 0.f, mv, vv, c, sc.x, sc.y);
        }
        b2_adam_apply(pv, __fmul_rn(p[e + delta_g], clip), mv, vv, c, now.x, now.y);
        p[e] = pv; p[e + delta_m] = mv; p[e + delta_v] = vv;
        p[e + delta_g] = 0.f;                       // the gradient arena stays all-zero between steps
      }
    }
    __syncwarp(0xFu << (threadIdx.x & 28));   // the 4 lanes of this row have read `last`
    if (sub == 0) last_step[grow] = t;
  }
}

// every row up to date with all completed steps (dense pass; checkpoints, evaluation, sharding ...)
__global__ void __launch_bounds__(256)
lazy_materialize_kernel(const b2_lazy_table* __restrict__ tables, int ntables, int64_t total_rows,
                        int64_t delta_m, int64_t delta_v, int32_t* __restrict__ last_step,
                        const B2AdamSched* __restrict__ sched, const int64_t* __restrict__ step_dev,
                        B2AdamConst c) {
  const int done = (int) *step_dev;
  const int sub = threadIdx.x & 3;
  for (int64_t grow = ((int64_t) blockIdx.x * blockDim.x + threadIdx.x) >> 2; grow < total_rows;
       grow += ((int64_t) gridDim.x * blockDim.x) >> 2) {
    const int last = last_step[grow];
    if (last >= done) continue;
    const b2_lazy_table tb = tables[find_table(tables, ntables, grow)];
    float* p = tb.param + (grow - tb.grow_base) * tb.dim;
    for (int e = sub; e < tb.dim; e += 4) {
      float pv = p[e], mv = p[e + delta_m], vv = p[e + delta_v];
      for (int k = last + 1; k <= done; ++k) {
        const B2AdamSched sc = sched[k];
        b2_adam_apply(pv, 0.f, mv, vv, c, sc.x, sc.y);
      }
      p[e] = pv; p[e + delta_m] = mv; p[e + delta_v] = vv;
    }
    __syncwarp(0xFu << (threadIdx.x & 28));
    if (sub == 0) last_step[grow] = done;
  }
}

int grid_rows(int64_t rows) {
  int64_t blocks = b2_ceil_div(rows * 4, 256);
  if (blocks > (int64_t) B2_NUM_SMS * 8) blocks = (int64_t) B2_NUM_SMS * 8;
  return (int) (blocks < 1 ? 1 : blocks);
}
B2AdamConst make_const(float beta1, float beta2, float eps) {
  B2AdamConst c;
  c.w1 = (float) (1.0 - (double) beta1);
  c.b2 = beta2;
  c.w2 = (float) (1.0 - (double) beta2);
  c.eps = eps;
  return c;
}
}  // namespace

extern "C" B2_API int b2_lazy_sumsq(const b2_lazy_table* tables_dev, int ntables, const int32_t* worklist,
                                    const int32_t* counter, int capacity, int64_t delta_g, float* sumsq,
                                    void* stream) {
  B2_REQUIRE(tables_dev && worklist && counter && sumsq && ntables >= 1 && capacity >= 1, "bad argument");
  lazy_sumsq_kernel<<<grid_rows(capacity), 256, 0, (cudaStream_t) stream>>>(tables_dev, ntables, worklist, counter,
                                                                           capacity, delta_g, sumsq);
  B2_CUDA_LAUNCH_CHECK("b2_lazy_sumsq");
  return B2_OK;
}

extern "C" B2_API int b2_lazy_adam_step(const b2_lazy_table* tables_dev, int ntables, const int32_t* worklist,
                                        const int32_t* counter, int capacity, int64_t delta_g, int64_t delta_m,
                                        int64_t delta_v, int32_t* last_step, const float* sched,
                                        const int64_t* step_dev, const float* sumsq, float max_norm,
                                        float beta1, float beta2, float eps, void* stream) {
  B2_REQUIRE(tables_dev && worklist && counter && last_step && sched && step_dev && ntables >= 1 && capacity >= 1,
             "bad argument");
  lazy_adam_kernel<<<grid_rows(capacity), 256, sizeof(b2_lazy_table) * ntables, (cudaStream_t) stream>>>(
      tables_dev, ntables, worklist, counter, capacity, delta_g, delta_m, delta_v, last_step,
      reinterpret_cast<const B2AdamSched*>(sched), step_dev, sumsq, max_norm, make_const(beta1, beta2, eps));
  B2_CUDA_LAUNCH_CHECK("b2_lazy_adam_step");
  return B2_OK;
}

extern "C" B2_API int b2_lazy_materialize(const b2_lazy_table* tables_dev, int ntables, int64_t total_rows,
                                          int64_t delta_m, int64_t delta_v, int32_t* last_step,
                                          const float* sched, const int64_t* step_dev, float beta1, float beta2,
                                          float eps, void* stream) {
  B2_REQUIRE(tables_dev && last_step && sched && step_dev && ntables >= 1 && total_rows >= 1, "bad argument");
  lazy_materialize_kernel<<<grid_rows(total_rows), 256, 0, (cudaStream_t) stream>>>(
      tables_dev, ntables, total_rows, delta_m, delta_v, last_step, reinterpret_cast<const B2AdamSched*>(sched),
      step_dev, make_const(beta1, beta2, eps));
  B2_CUDA_LAUNCH_CHECK("b2_lazy_materialize");
  return B2_OK;
}

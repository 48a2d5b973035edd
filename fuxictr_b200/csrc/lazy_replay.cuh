// lazy_replay.cuh — the two device-side halves of lazy tables (b2_lazy_ctx, include/fuxictr_b200.h) that
// the kernels READING the tables share: the fused front (fused_front.cu) and the row-sharded push/pull
// (shard.cu).  One definition, so that every reader replays and enqueues exactly alike.
//
// Replay: a row read from a lazily evaluated table is brought up to date IN REGISTERS before it is used,
//   by applying the zero-gradient Adam updates of the steps it missed (same scalars sched[k], same
//   rounded arithmetic as the dense pass, adam_common.cuh).  Nothing is written back: a row's p/m/v and
//   last_step change only in b2_lazy_adam_step and b2_lazy_materialize.
// Enqueue: the first toucher of a row in a step claims it (atomicExch on mark) and appends its global
//   row number to the worklist — one atomicAdd per warp, not per row.
#pragma once
#include "embed_common.cuh"
#include "adam_common.cuh"

// N rows per lane, all last_step loads and then all moment loads of stale rows in flight.
// Row u is field f[u], row row[u] of the tables staged in sf (embedding) / lf (LR); on_e[u] / on_l[u]:
// this lane holds the 4 embedding elements [e, e+4) / the LR weight of that row in v[u] / w[u].
// `done` = optimizer steps completed (*lz.step_dev); lz.grow_emb / grow_lr map a field's rows to global rows.
template <int N>
__device__ __forceinline__ void b2_lazy_replay(const b2_lazy_ctx& lz, int done, const SmemFields& sf,
                                               const SmemFields& lf, int dim, int e, const int (&f)[N],
                                               const int64_t (&row)[N], const bool (&on_e)[N],
                                               const bool (&on_l)[N], float4 (&v)[N], float (&w)[N]) {
  const B2AdamConst ac = {lz.w1, lz.beta2, lz.w2, lz.eps};
  const B2AdamSched* sched = reinterpret_cast<const B2AdamSched*>(lz.sched);
  int last_e[N], last_l[N];
#pragma unroll
  for (int u = 0; u < N; ++u) {   // all last_step loads in flight
    last_e[u] = on_e[u] ? __ldg(lz.last_step + lz.grow_emb[f[u]] + row[u]) : done;
    last_l[u] = on_l[u] ? __ldg(lz.last_step + lz.grow_lr[f[u]] + row[u]) : done;
  }
  float4 m4[N], v4[N];
  float m1[N], v1[N];
#pragma unroll
  for (int u = 0; u < N; ++u) {   // all moment loads of stale rows in flight
    m4[u] = v4[u] = make_float4(0.f, 0.f, 0.f, 0.f);
    m1[u] = v1[u] = 0.f;
    if (last_e[u] < done) {
      const float* pp = reinterpret_cast<const float*>(sf.f[f[u]].table) + row[u] * dim + e;
      m4[u] = *reinterpret_cast<const float4*>(pp + lz.delta_m);
      v4[u] = *reinterpret_cast<const float4*>(pp + lz.delta_v);
    }
    if (last_l[u] < done) {
      const float* pp = reinterpret_cast<const float*>(lf.f[f[u]].table) + row[u];
      m1[u] = pp[lz.delta_m];
      v1[u] = pp[lz.delta_v];
    }
  }
#pragma unroll
  for (int u = 0; u < N; ++u) {   // replay the missed zero-gradient updates
    for (int k = last_e[u] + 1; k <= done; ++k) {
      const B2AdamSched sc = sched[k];
      b2_adam_apply(v[u].x, 0.f, m4[u].x, v4[u].x, ac, sc.x, sc.y);
      b2_adam_apply(v[u].y, 0.f, m4[u].y, v4[u].y, ac, sc.x, sc.y);
      b2_adam_apply(v[u].z, 0.f, m4[u].z, v4[u].z, ac, sc.x, sc.y);
      b2_adam_apply(v[u].w, 0.f, m4[u].w, v4[u].w, ac, sc.x, sc.y);
    }
    for (int k = last_l[u] + 1; k <= done; ++k) {
      const B2AdamSched sc = sched[k];
      b2_adam_apply(w[u], 0.f, m1[u], v1[u], ac, sc.x, sc.y);
    }
  }
}

// Claims global row `grow` for the step marked `tmark` (= *lz.step_dev + 1): true for the first toucher only.
__device__ __forceinline__ bool b2_lazy_claim(const b2_lazy_ctx& lz, int grow, int tmark) {
  return atomicExch(lz.mark + grow, tmark) != tmark;
}

// Warp-aggregated append of the rows this lane claimed (enq_e / enq_l >= 0) to the worklist.
// Every lane of the warp calls it.  Entries past worklist_capacity are dropped (the capacity is the
// row count, which no step can exceed).
__device__ __forceinline__ void b2_lazy_append(const b2_lazy_ctx& lz, int enq_e, int enq_l, int lane) {
  const unsigned me = __ballot_sync(0xffffffffu, enq_e >= 0);
  const unsigned ml = __ballot_sync(0xffffffffu, enq_l >= 0);
  const int ne = __popc(me), nl = __popc(ml);
  if (ne + nl == 0) return;
  int base = 0;
  if (lane == 0) base = atomicAdd(lz.counter, ne + nl);
  base = __shfl_sync(0xffffffffu, base, 0);
  const unsigned lt = (1u << lane) - 1u;
  if (enq_e >= 0) {
    const int pos = base + __popc(me & lt);
    if (pos < lz.worklist_capacity) lz.worklist[pos] = enq_e;
  }
  if (enq_l >= 0) {
    const int pos = base + ne + __popc(ml & lt);
    if (pos < lz.worklist_capacity) lz.worklist[pos] = enq_l;
  }
}

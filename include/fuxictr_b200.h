/*
 * fuxictr_b200.h — C-ABI of the H100 (sm_90a) hot path for FuxiCTR models.
 *
 * The reference (reczoo/FuxiCTR v2.3.10) has no FFI: its hot path is a set of
 * torch.nn.Module classes that dispatch to stock ATen ops.  Every entry point
 * below replaces one of those ATen call sites; the citation beside each
 * declaration is the reference file:line (relative to the reference root) whose
 * arithmetic the kernel reproduces.  INTEGRATION.md shows the Python (ctypes)
 * binding a FuxiCTR maintainer would add on the reference side.
 *
 * Conventions
 *  - plain C types only: raw DEVICE pointers, explicit sizes/strides, a
 *    cudaStream_t passed as void* (0 = legacy default stream).
 *  - every call is asynchronous on `stream`; nothing synchronises internally,
 *    nothing is allocated; outputs/workspaces are caller-allocated.
 *  - return value: 0 on success, negative B2_E_* on failure; the message for
 *    the calling thread's last failure is b2_last_error().
 *  - all matrices are row-major unless a stride argument says otherwise.
 *  - "f32" everywhere means IEEE binary32 with round-to-nearest FMA
 *    arithmetic; global atomics flush subnormals (PTX red.global.add.f32).
 */
#ifndef FUXICTR_B200_H_
#define FUXICTR_B200_H_

#include <stdint.h>

#if defined(__GNUC__)
#define B2_API __attribute__((visibility("default")))
#else
#define B2_API
#endif

#ifdef __cplusplus
extern "C" {
#endif

/* ---- error codes ------------------------------------------------------- */
#define B2_OK 0
#define B2_E_INVALID (-1)    /* bad argument (null pointer, unsupported size/dtype) */
#define B2_E_CUDA (-2)       /* CUDA runtime/driver error; see b2_last_error() */
#define B2_E_UNSUPPORTED (-3)/* valid request this build cannot serve */

/* ---- dtype codes --------------------------------------------------------- */
#define B2_F32 0
#define B2_BF16 1
#define B2_F64 2  /* index matrices arrive as float64 (npz_dataloader.py:63-66) */
#define B2_I64 3
#define B2_I32 4

/* ---- pooling modes of a sequence field (feature_encoder) ---------------- */
#define B2_POOL_NONE 0 /* emit (B, L, D) */
#define B2_POOL_SUM 1  /* MaskedSumPooling, layers/pooling.py:62-73 */
#define B2_POOL_MEAN 2 /* MaskedAveragePooling, layers/pooling.py:33-49 */

/* ---- activation codes for fused GEMM epilogues --------------------------- */
#define B2_ACT_NONE 0
#define B2_ACT_RELU 1
#define B2_ACT_SIGMOID 2
#define B2_ACT_LEAKY_RELU 4 /* nn.LeakyReLU(): y = z > 0 ? z : z * B2_LEAKY_SLOPE; its backward reads y (y > 0 iff z > 0) */
#define B2_LEAKY_SLOPE 0.01f
#define B2_PREP_MUL 3 /* b2_prep_operand only: v = x * y (plain elementwise product, CrossNetV2 backward) */

#define B2_MAX_FIELDS 128

/* Library/version probes (no GPU needed). */
B2_API const char* b2_version(void);
B2_API const char* b2_last_error(void);
/* Returns the compute capability major*10+minor of `device`, or a negative
 * error.  The library only contains sm_90a code. */
B2_API int b2_device_cc(int device);
/* Sets cudaLimitMaxL2FetchGranularity (32, 64 or 128 bytes) on the current device: how much L2 pulls
 * from HBM around a missing 32-byte sector.  Embedding rows are 64 bytes (D=16 fp32) at random
 * addresses; with 128-byte fetches every row read costs 128 bytes of DRAM traffic.  A context-wide hint;
 * no effect on results. */
B2_API int b2_set_l2_fetch_granularity(int bytes);

/*
 * One feature of the fused multi-field gather.  Mirrors one iteration of the
 * per-feature loop in FeatureEmbeddingDict.forward
 * (fuxictr/pytorch/layers/embeddings/feature_embedding.py:261-297): `idx` is
 * the (B,) [or (B, L)] column view the BatchCollator produced
 * (dataloaders/npz_dataloader.py:111-125), `table` is the nn.Embedding weight
 * (feature_embedding.py:172-175), `out` is where the caller wants this
 * feature's slice of the stacked (B,F,D) / concatenated (B,sum D) tensor that
 * dict2tensor would build (feature_embedding.py:230-259), or a separate
 * (B,L,D) buffer for an unpooled sequence.
 */
typedef struct b2_field {
  const void* table;   /* (vocab, dim) row-major table, or its dense-grad twin in *_bwd */
  const void* idx;     /* index of sample 0, position 0 */
  void* out;           /* output element of sample 0 (fwd: written, bwd: grad read) */
  int64_t vocab;       /* rows in table */
  int64_t idx_stride;  /* index elements between consecutive samples */
  int64_t out_stride;  /* output elements between consecutive samples */
  int32_t dim;         /* embedding dim of this field */
  int32_t seq_len;     /* 1 = categorical; L = sequence, positions contiguous */
  int32_t pool;        /* B2_POOL_* (only meaningful when seq_len > 1) */
  int32_t padding_idx; /* row that receives no gradient; -1 = none */
} b2_field;

/*
 * Fused multi-field embedding gather, forward.
 * Replaces, for all F features in one launch: the `.long()` cast + aten::embedding
 * per feature (feature_embedding.py:283-288), the optional Masked{Sum,Average}Pooling
 * encoder (layers/pooling.py:45-49,73) and the torch.stack/torch.cat of
 * dict2tensor (feature_embedding.py:255-258).
 *   fields     HOST array of nfields descriptors (copied into the launch)
 *   idx_dtype  B2_F64 | B2_I64 | B2_I32 (f64 is truncated toward zero like .long())
 *   elem_dtype B2_F32 (tables and outputs)
 *   mean_count device f32[nfields * batch] or NULL; required when a field uses
 *              B2_POOL_MEAN: receives at [f*batch + b] the MaskedAveragePooling
 *              denominator (positions whose embedding vector sums to non-zero,
 *              pooling.py:46-47) for the backward.
 *   status     device int32[1], or NULL.  Set (atomicMax) to 1+field if an index is
 *              outside [0, vocab) (the reference raises IndexError); the row is zero-filled.
 *   hot_rows   >= 0; 0 = no staging.  The first `hot_rows` rows of every table are staged once per CTA
 *              in shared memory and served from there (north_star "shared-memory staging of hot rows"):
 *              FuxiCTR's tokenizer numbers ids by descending frequency, so the small ids are the hot
 *              ones.  Applies when every field is one slot of one common dim (% 4) and the staging area
 *              fits 44 KB per CTA; otherwise ignored.  The result is bit-identical either way.
 */
B2_API int b2_embed_gather_fwd(const b2_field* fields, int nfields, int64_t batch, int idx_dtype,
                               int elem_dtype, float* mean_count, int32_t* status, int hot_rows,
                               void* stream);

/*
 * Touched-granule flags of a gradient arena's table prefix: one byte per 64-byte granule (16 floats)
 * of [base, base + n).  A backward kernel given a b2_touch sets the byte of every granule it adds a
 * gradient into (a plain store: idempotent, no atomic); writes outside [base, base + n) mark nothing.
 * Invariant the optimizer relies on: every nonzero float of [base, base + n) lies in a flagged granule
 * (b2_sumsq_ex / b2_adam_step_ex skip the others).  Marking more is always safe.
 * flags == NULL or n == 0: no flags.
 */
typedef struct b2_touch {
  uint8_t* flags;      /* [(n + 15) / 16] */
  const float* base;   /* first element covered (16-byte aligned) */
  int64_t n;           /* elements covered */
} b2_touch;

/*
 * Backward of the fused gather: dense-gradient scatter-add with warp-level
 * aggregation of duplicate rows.  Replaces F x aten::embedding_dense_backward
 * (autograd of feature_embedding.py:285,288).  In each descriptor `table` is the
 * (vocab, dim) f32 GRADIENT buffer (accumulated into: the caller zeroes it when it
 * wants "=" semantics), `out` is the incoming gradient laid out exactly like the
 * forward output; rows whose index equals padding_idx receive no gradient
 * (nn.Embedding(padding_idx)).  mean_count is the buffer the forward filled
 * (NULL when no field uses B2_POOL_MEAN).  touch (NULL = none): marks the granules
 * of every gradient row it adds into (b2_touch).
 */
B2_API int b2_embed_scatter_bwd(const b2_field* fields, int nfields, int64_t batch, int idx_dtype,
                                int elem_dtype, const float* mean_count, const b2_touch* touch,
                                void* stream);

/*
 * LogisticRegression.forward (layers/blocks/logistic_regression.py:55-58):
 * out[b] = sum over features (and sequence positions, MaskedSumPooling,
 * feature_embedding.py:135-138) of table_f[idx] + bias[0].  Tables are
 * (vocab,1) f32; `fields[i].out/out_stride/dim/pool` are ignored.
 *   bias  device f32[1] or NULL;  out  device f32[batch]
 */
B2_API int b2_lr_fwd(const b2_field* fields, int nfields, int64_t batch, int idx_dtype, const float* bias,
              float* out, int32_t* status, void* stream);
/* Backward: table_f[idx] += gout[b] (skipping padding_idx); if gbias != NULL,
 * gbias[0] += sum_b gout[b]. `table` fields point at the (vocab,1) gradient buffers.
 * touch (NULL = none): marks the granules of every gradient row it adds into (b2_touch). */
B2_API int b2_lr_bwd(const b2_field* fields, int nfields, int64_t batch, int idx_dtype,
                     const float* gout, float* gbias, const b2_touch* touch, void* stream);


/*
 * Lazy evaluation of the DENSE Adam semantics for embedding tables (an exact "next row" of SURVEY
 * 8f-2).  The reference updates every row of every table every step (rows with zero gradient still
 * move: m *= b1, v *= b2, p -= lr_t*m/(sqrt(v)/sqrt(bc2_t)+eps)).  In lazy mode a row is brought up
 * to date only when a batch touches it: the fused front reads p and, when last_step[row] < steps
 * done, replays the zero-gradient updates of the missed steps in registers (b2_front_fwd); the
 * backward enqueues every touched row once (b2_front_bwd); b2_lazy_adam_step then replays the missed
 * steps for the enqueued rows and applies the real update.  Every replayed update uses the same
 * scalars (sched[t], written by b2_adam_sched) and the same explicitly rounded arithmetic as the
 * dense pass, so the result is BIT-IDENTICAL to dense Adam (tests/test_gpu_parity.py).
 * Rows are numbered globally: table i owns rows [grow_base[i], grow_base[i] + vocab_i).
 * Row-sharded tables (b2_shard_push / b2_shard_pull): the same protocol over the rows THIS rank
 * owns.  The push replays a stale row before it stores it into the requester's buffer; the pull, where
 * several requesters may send gradients for one row, enqueues the row once.  grow_emb / grow_lr and
 * the worklist then count this rank's LOCAL rows (shard row r of table i is row grow_base[i] + r);
 * worklist entries are int32, so a rank holds at most 2^31 - 1 lazy rows.
 * The readers of a lazy table are these four kernels only; every other read of the parameters needs
 * b2_lazy_materialize first.
 */
typedef struct b2_lazy_ctx {
  const int32_t* last_step; /* [total rows] optimizer step each row is current for */
  const float* sched;       /* float2[sched_len]: {lr/(1-b1^t), 1/sqrt(1-b2^t)} per step t */
  const int64_t* step_dev;  /* device scalar: optimizer steps completed so far */
  int32_t* mark;            /* [total rows] scratch: step at which the row was last enqueued */
  int32_t* worklist;        /* [capacity] global row ids touched this step */
  int32_t* counter;         /* device scalar: worklist length */
  int64_t delta_m, delta_v; /* element offsets from a parameter to its Adam moments (arena layout) */
  float w1, beta2, w2, eps; /* fl32(1-beta1), fl32(beta2), fl32(1-beta2) from the double betas; eps */
  int32_t worklist_capacity, pad_;
  int64_t grow_emb[B2_MAX_FIELDS]; /* global row base of the embedding table of each field */
  int64_t grow_lr[B2_MAX_FIELDS];  /* ... and of its LR table */
} b2_lazy_ctx;

/*
 * The sparse front of an FM-style model in one launch each way (DeepFM, xDeepFM's LR term):
 *   emb   = FeatureEmbedding.forward  (feature_embedding.py:73-88)      -> written through emb_fields[i].out
 *   logit = InnerProductInteraction "product_sum" (inner_product.py:56-62, if want_fm)
 *         + LogisticRegression (logistic_regression.py:55-58, if lr_fields != NULL) + bias
 * Requirements: categorical fields only (seq_len 1), one common emb dim with dim % 4 == 0 and
 * dim <= 128, 16-byte aligned rows; lr_fields[i] shares idx/idx_stride with emb_fields[i] and
 * points at the (vocab,1) tables.  sum_out (B, dim) receives sum_f e (saved for the backward).
 */
B2_API int b2_front_fwd(const b2_field* emb_fields, const b2_field* lr_fields, int nfields, int64_t batch,
                        int idx_dtype, int want_fm, const float* bias, float* logit_out, float* sum_out,
                        int32_t* status, const b2_lazy_ctx* lazy /* NULL = tables are up to date */,
                        float* emb_small /* NULL, or a second arena of the output's layout that receives the
                                            3xTF32 small part of every row (the first GEMM's A operand) */,
                        void* stream);
/*
 * Backward of b2_front_fwd.  In emb_fields, `table` is the (vocab, dim) gradient buffer (NULL =
 * no gradient wanted) and `out` addresses the incoming gradient arena gx (same layout as the
 * forward output); emb_saved is the forward output itself.  Per row:
 *   g = gx[b,f,:] + glogit[b] * (sums[b,:] - emb_saved[b,f,:])      (second term only if want_fm)
 * is scatter-added (warp-aggregated) into the gradient table, rows equal to padding_idx skipped;
 * lr_fields[i].table (vocab,1) += glogit[b]; gbias[0] += sum_b glogit[b].
 * touch (NULL = none): marks (b2_touch) every embedding and LR gradient it writes.
 */
B2_API int b2_front_bwd(const b2_field* emb_fields, const b2_field* lr_fields, int nfields, int64_t batch,
                        int idx_dtype, int want_fm, const float* emb_saved, const float* gx,
                        const float* sums, const float* glogit, float* gbias,
                        const b2_lazy_ctx* lazy /* non-NULL: enqueue every touched row once */,
                        const b2_touch* touch, void* stream);
/*
 * Flags (b2_touch over the PARAMETER arena) every granule of every row a fused front or fused gather reads
 * for this batch: emb_fields[i].table / lr_fields[i].table are the parameter tables, idx as in b2_front_fwd
 * (same id decoding; out-of-range ids mark nothing, padding rows are marked).  That covers every granule the
 * backward writes, so the marks are final as soon as the ids are (see b2_adam_untouched).
 */
B2_API int b2_table_mark(const b2_field* emb_fields, const b2_field* lr_fields, int nfields, int64_t batch,
                         int idx_dtype, const b2_touch* touch, void* stream);
/*
 * Lazy optimizer step over the rows enqueued by b2_front_bwd (tables[i]: parameter pointer, rows, dim,
 * global row base, sorted by base; gradients/moments at the arena deltas):
 *   b2_lazy_sumsq      sumsq[0] += sum of g^2 over the enqueued rows
 *   b2_lazy_adam_step  for each enqueued row: replay the missed zero-gradient steps, apply step t with
 *                      clip_coef*g, store p/m/v, last_step = t, zero the gradient row
 *   b2_lazy_materialize bring EVERY row up to date (before checkpoints / reads outside the kernels)
 */
typedef struct b2_lazy_table {
  float* param;      /* (rows, dim) parameter slice inside the arena */
  int64_t rows;
  int64_t grow_base; /* first global row id */
  int32_t dim, pad_;
} b2_lazy_table;
B2_API int b2_lazy_sumsq(const b2_lazy_table* tables_dev, int ntables, const int32_t* worklist,
                         const int32_t* counter, int capacity, int64_t delta_g, float* sumsq, void* stream);
B2_API int b2_lazy_adam_step(const b2_lazy_table* tables_dev, int ntables, const int32_t* worklist,
                             const int32_t* counter, int capacity, int64_t delta_g, int64_t delta_m,
                             int64_t delta_v, int32_t* last_step, const float* sched,
                             const int64_t* step_dev, const float* sumsq, float max_norm, double beta1,
                             double beta2, float eps, void* stream);
B2_API int b2_lazy_materialize(const b2_lazy_table* tables_dev, int ntables, int64_t total_rows,
                               int64_t delta_m, int64_t delta_v, int32_t* last_step, const float* sched,
                               const int64_t* step_dev, double beta1, double beta2, float eps, void* stream);

/*
 * Row-sharded tables across the GPUs of one NVSwitch box (SURVEY.md 8e): row r of every table
 * lives on rank r % world at local row r / world.  The lookup and its exchange are one kernel
 * over NVLink peer memory.  In emb_fields/lr_fields: `table` = this rank's shard (or its gradient
 * shard in b2_shard_pull), `vocab` = GLOBAL vocabulary, `idx_stride` = COLUMN of the field in the
 * batch matrix, `padding_idx` = global padding row; `idx`/`out` are unused.
 *   peer_ids[p]   (B_local, ids_stride) batch matrix of rank p       (peer-mapped, read)
 *   peer_emb[p]   (B_local, F*D) fp32 embedding output of rank p     (peer-mapped, written)
 *   peer_lrw[p]   (B_local, F)   fp32 LR weights of rank p's samples (peer-mapped, written)
 * b2_shard_push gathers the rows THIS rank owns for every rank's samples and stores them into the
 * requester's buffers.  With `owned` != NULL it also records every (requester, sample*F+field, local
 * row, field|flags) it served as one int32[4] entry of `owned` (16-byte aligned, `owned_capacity`
 * entries; world * B_local * F can never overflow) and the entry count in `owned_count` (zeroed by
 * the call).  b2_shard_pull walks that list: it reads the requester's gradient rows peer_gemb[p]
 * (B_local, F*D) / peer_glogit[p] (B_local) and scatter-adds `scale *` them into the local gradient
 * shards — ~B_local*F entries instead of world*B_local*F candidates, and no second pass over the
 * peers' ids.  Cross-rank ordering is the caller's barrier.  world <= 16.
 * Lazy tables (see b2_lazy_ctx): lazy == NULL means the tables are up to date.  Otherwise the push
 * brings every served row with last_step[grow] < *step_dev up to date in registers before the store
 * (nothing is written back), and the pull appends every owned, non-padding row it scatters a gradient
 * into to the worklist, once per step (claimed through mark).  grow = grow_emb[f] / grow_lr[f] + local
 * row.  The caller zeroes lazy->counter before the pull of a step.  touch (NULL = none): the pull marks
 * the granules of every gradient row it scatters into (b2_touch).
 * Padding rows: with pad_rows != NULL every rank fills its OWN padding slots (id == padding_idx) from
 * pad_rows, this rank's (F*D + F)-float buffer (16-byte aligned) that b2_shard_publish_ids filled before
 * the push (padding row of field f at f*D, its LR weight at F*D + f): no rank serves the padding slots of
 * the others, and the copy is bit-exact whatever the padding row holds.  Padding slots get no gradient.
 * pad_rows == NULL: the owner of the padding row serves it like any other row.
 * Sequence fields: a field with seq_len L > 1 (pool must be B2_POOL_NONE: a pooled sequence's rows come from
 * several owners) is L consecutive SLOTS, with its ids in columns idx_stride .. idx_stride + L - 1.  With
 * S = sum of seq_len, slot s of sample b lands at b*S*D + s*D of peer_emb / is read at the same offset of
 * peer_gemb, and an owned-list entry keeps b*S + s where a one-slot field keeps b*F + f.  Requires
 * batch_local * S < 2^31; an owned list of world * batch_local * S entries never overflows.  LR tables
 * (lr_fields != NULL) need seq_len == 1 on every field.
 */
B2_API int b2_shard_push(const b2_field* emb_fields, const b2_field* lr_fields, int nfields,
                         int64_t batch_local, int world, int rank, const void* const* peer_ids,
                         int idx_dtype, int64_t ids_stride, float* const* peer_emb,
                         float* const* peer_lrw, int32_t* status, int32_t* owned, int32_t* owned_count,
                         int32_t owned_capacity, const b2_lazy_ctx* lazy, const float* pad_rows,
                         void* stream);
B2_API int b2_shard_pull(const b2_field* emb_fields, const b2_field* lr_fields, int nfields,
                         int64_t batch_local, int world, int rank, const float* const* peer_gemb,
                         const float* const* peer_glogit, float scale, const int32_t* owned,
                         const int32_t* owned_count, int32_t owned_capacity, const b2_lazy_ctx* lazy,
                         const b2_touch* touch, void* stream);
/* The id exchange, compressed: `count` contiguous ids of dtype idx_dtype (B2_F64 truncates like .long())
 * are narrowed to int32 and stored into peer_dst[p] (16-byte aligned) for every p < world.  In the same
 * launch the padding rows: for every field whose padding row this rank owns, the row (emb_fields[f].table =
 * this rank's shard) and its LR weight are stored into peer_pad[p] (16-byte aligned, F*D + F floats, layout
 * as pad_rows above) for every p < world. */
B2_API int b2_shard_publish_ids(const void* src, int idx_dtype, int64_t count, int32_t* const* peer_dst,
                                const b2_field* emb_fields, const b2_field* lr_fields, int nfields, int world,
                                int rank, float* const* peer_pad, void* stream);
/*
 * The evaluation round: a forward-only lookup of a ragged batch (0 <= rows <= batch_local samples on each rank,
 * which may differ between ranks and between rounds).
 * b2_shard_publish_rows: b2_shard_publish_ids of the first `rows` rows of a (rows, width) batch matrix — only
 * rows * width ids are read and stored into peer_dst[p] — and, in the same launch, the row count into word
 * `rank` of peer_rows[p] (int32[world] on every rank, 4-byte aligned) for every p < world.  Refused: rows
 * outside [0, capacity_rows] (capacity_rows = the batch_local of the peer buffers), NULL src with rows > 0.
 * b2_shard_lookup: b2_shard_push over the candidates (requester p, sample b < rows_all[p], slot), where
 * rows_all is this rank's int32[world] buffer that every rank's publish filled before the barrier: the bound
 * comes from device memory, so no rank needs its peers' counts on the host, and a rank with 0 rows still
 * serves the others.  peer_ids hold the int32 ids the publish stored (row pitch ids_stride).  It keeps no
 * owned-row list and takes no lazy context: it reads the tables as they are (materialise lazy tables first),
 * and leaves the owned list and the lazy bookkeeping of the next training step untouched.  Out-of-range ids
 * set *status (if not NULL) and land as zero rows, as in the push.  Follow it with b2_front_reduce over
 * `rows` samples. */
B2_API int b2_shard_publish_rows(const void* src, int idx_dtype, int64_t rows, int64_t width, int64_t capacity_rows,
                                 int32_t* const* peer_dst, const b2_field* emb_fields, const b2_field* lr_fields,
                                 int nfields, int world, int rank, float* const* peer_pad, int32_t* const* peer_rows,
                                 void* stream);
B2_API int b2_shard_lookup(const b2_field* emb_fields, const b2_field* lr_fields, int nfields, int64_t batch_local,
                           int world, int rank, const int32_t* const* peer_ids, int64_t ids_stride,
                           float* const* peer_emb, float* const* peer_lrw, const int32_t* rows_all, int32_t* status,
                           const float* pad_rows, void* stream);
/* After the push: logit[b] = [FM product_sum of emb[b]] (if want_fm) + sum_f lrw[b,f] + bias;
 * sums[b,:] = sum_f emb[b,f,:] (saved for the backward). */
B2_API int b2_front_reduce(const float* emb, const float* lrw, const float* bias, int64_t batch,
                           int nfields, int dim, int want_fm, float* logit, float* sums, void* stream);
/* Before the pull: gemb[b,f,:] = gx[b,f,:] + glogit[b] * (sums[b,:] - emb[b,f,:]) (2nd term if want_fm);
 * glogit_out (optional, peer-visible) receives a copy of glogit for the owners of the LR rows;
 * gbias (optional, 1 float) receives sum_b glogit[b], the LogisticRegression bias gradient (cleared by the
 * call unless gbias_is_zero). */
B2_API int b2_front_gprep(const float* gx, const float* emb, const float* sums, const float* glogit,
                          int64_t batch, int nfields, int dim, int want_fm, float* gemb, float* glogit_out,
                          float* gbias, int gbias_is_zero, void* stream);

/*
 * InnerProductInteraction (layers/interactions/inner_product.py:55-70).
 * emb is (B, F, D) f32 contiguous.
 *   mode 0 "product_sum":    out (B,1)   = sum_d 0.5*((sum_f e)^2 - sum_f e^2)   (:56-62)
 *   mode 1 "bi_interaction": out (B,D)   = 0.5*((sum_f e)^2 - sum_f e^2)         (:56-60)
 *   mode 2 "inner_product":  out (B,F(F-1)/2) = triu(E E^T, 1), row-major pairs  (:64-66)
 * *_bwd writes gemb (B,F,D) ("=" semantics).
 */
B2_API int b2_fm_fwd(const float* emb, int64_t batch, int nfields, int dim, int mode, float* out,
              void* stream);
B2_API int b2_fm_bwd(const float* emb, const float* gout, int64_t batch, int nfields, int dim, int mode,
              float* gemb, void* stream);

/*
 * CrossNet (layers/interactions/cross_net.py:44-55,80-92), all layers in one
 * launch: x_{i+1} = x_i + (w_i . x_i) * x_0 + b_i.
 *   x0 (B,d); w (L,d); b (L,d); out (B,d); s (B,L) saved dot products w_i.x_i
 * bwd: gx0 (B,d) "="; gw, gb (L,d) "+=" (caller zeroes).
 */
B2_API int b2_crossnet_fwd(const float* x0, const float* w, const float* b, int64_t batch, int d,
                    int nlayers, float* out, float* s, void* stream);
B2_API int b2_crossnet_bwd(const float* x0, const float* w, const float* b, const float* s,
                    const float* gout, int64_t batch, int d, int nlayers, float* gx0, float* gw,
                    float* gb, void* stream);

/*
 * CrossNetMix (layers/interactions/cross_net.py:132-201), one layer of the low-rank mixture of experts:
 *   h_e = tanh(x_l V_e), v_e = tanh(h_e C_e^T), p = softmax_e(x_l g_e^T),
 *   x_{l+1} = x_l + x0 * (A2 @ W2^T + b),  A2 = [p_1 v_1 | ... | p_E v_E]   (exact because sum_e p_e = 1)
 * as GEMM1 P = x_l @ W1^T, the row kernel P -> A2, and GEMM2 with the CrossNetV2 epilogue.
 * U, V (E, d, r) and C (E, r, r) are the layer's U_list[i], V_list[i], C_list[i]; G (E, d) the rows
 * gating[e].weight.  With R = E*r, N1 = round_up(R + E, 4), K2 = round_up(R, 4), all row-major fp32:
 *   W1 (N1, d) K-major:  W1[e*r + j, :] = V[e, :, j];  W1[R + e, :] = G[e, :];  rows R+E .. N1-1 zero
 *   W2 (d, K2) K-major:  W2[n, e*r + j] = U[e, n, j];  columns R .. K2-1 zero
 *   P  (B, N1) = x_l W1^T: columns 0..R-1 the pre-tanh h, R..R+E-1 the gate logits
 *   A2 (B, K2), dA2 (B, K2): columns R .. K2-1 of A2 are written zero, those of dA2 are not read
 *   dA1 (B, N1) = [dP | dlogit | 0]: the gradient of P
 * Supported range: 1 <= r <= B2_CROSSMIX_MAX_RANK and E*r <= B2_CROSSMIX_MAX_COLS (all experts' C in one
 * CTA's shared memory); outside it every entry point returns B2_E_INVALID.
 * Saved for the backward: x_l, P, A2 and the packed W1, W2 of the forward; the backward recomputes h, v, p
 * from P and C.
 * b2_crossmix_pack: W1, W2 ("=") from U, V, G; one launch.
 * b2_crossmix_fwd:  A2 "=" from P and C; a2_aux (optional, row pitch ld_aux) receives A2's GEMM operand
 *   copy: its bf16 rounding (aux_dtype B2_BF16) or its 3xTF32 small part (B2_F32).
 * b2_crossmix_bwd:  dA1 "=" (+ da1_aux as above) from P, C, dA2; dC (E, r, r) "+=" (caller zeroes): a
 *   per-CTA sum in shared memory, then one float atomic per element and CTA.
 * b2_crossmix_unpack: gU, gV (E, d, r) and gG (E, d) "=" from dW1 (N1, d) and dW2 (d, K2).
 */
#define B2_CROSSMIX_MAX_RANK 64
#define B2_CROSSMIX_MAX_COLS 256
B2_API int b2_crossmix_pack(const float* U, const float* V, const float* G, int d, int r, int E, float* W1,
                            float* W2, void* stream);
B2_API int b2_crossmix_fwd(const float* P, const float* C, int64_t batch, int r, int E, float* A2, void* a2_aux,
                           int aux_dtype, int64_t ld_aux, void* stream);
B2_API int b2_crossmix_bwd(const float* P, const float* C, const float* dA2, int64_t batch, int r, int E,
                           float* dA1, void* da1_aux, int aux_dtype, int64_t ld_aux, float* dC, void* stream);
B2_API int b2_crossmix_unpack(const float* dW1, const float* dW2, int d, int r, int E, float* gU, float* gV,
                              float* gG, void* stream);

/*
 * GDCN's gated cross layer (model_zoo/GDCN/src/GDCN.py, GateCorssLayer), one layer:
 *   x_{i+1} = x_0 * (x_i W^T + b) * sigmoid(x_i Wg^T) + x_i
 * as one GEMM P = x_i Wp^T on the stacked weight and one row kernel.  W, Wg (d, d) are the layer's
 * w[i].weight and wg[i].weight, b (d) its b[i].  All row-major fp32:
 *   Wp (2d, d) K-major: rows 0 .. d-1 are W, rows d .. 2d-1 are Wg
 *   P  (B, 2d) = x_i Wp^T: columns 0 .. d-1 u = x_i W^T, columns d .. 2d-1 z = x_i Wg^T
 *   dP (B, 2d): the gradient of P, [g x_0 s | g x_0 lin s (1 - s)] with lin = u + b, s = sigmoid(z)
 *   dWp (2d, d) = dP^T x_i: rows 0 .. d-1 the gradient of W, rows d .. 2d-1 that of Wg
 * Saved for the backward: x_0, x_i, P and the forward's Wp; the backward recomputes lin and s from P and b.
 * Range: any d >= 1 and batch >= 0 with batch * 2d < 2^31; d % 4 == 0 with 16-byte aligned rows takes a float4
 * path, anything else a scalar one.  Outside the range, or given a NULL pointer, every entry point returns
 * B2_E_INVALID.
 * b2_gdcn_pack:   Wp "=" from W, Wg; one launch.
 * b2_gdcn_fwd:    out (B, d) "=" from P, b, x_0, x_i; out_aux (optional, row pitch ld_aux) receives out's GEMM
 *   operand copy for the next layer: its bf16 rounding (aux_dtype B2_BF16) or its 3xTF32 small part (B2_F32).
 * b2_gdcn_bwd:    dP "=" (+ dp_aux as above, row width 2d) and gx0 (B, d) "=" g lin s from P, b, x_0 and the
 *   output gradient g; db (d) "+=" (caller zeroes) the column sums of dP's first half: a per-CTA sum, then one
 *   float atomic per column and CTA.
 * b2_gdcn_unpack: gW, gWg (d, d) "=" from dWp.
 */
B2_API int b2_gdcn_pack(const float* W, const float* Wg, int d, float* Wp, void* stream);
B2_API int b2_gdcn_fwd(const float* P, const float* b, const float* x0, const float* xi, int64_t batch, int d,
                       float* out, void* out_aux, int aux_dtype, int64_t ld_aux, void* stream);
B2_API int b2_gdcn_bwd(const float* P, const float* b, const float* x0, const float* g, int64_t batch, int d,
                       float* dP, void* dp_aux, int aux_dtype, int64_t ld_aux, float* gx0, float* db, void* stream);
B2_API int b2_gdcn_unpack(const float* dWp, int d, float* gW, float* gWg, void* stream);

/*
 * FinalMLP (model_zoo/FinalMLP/src/FinalMLP.py): FeatureSelection's gating products and InteractionAggregation at
 * output_dim 1.  All row-major fp32.
 *
 * Gate: e (B, d) is the flattened embedding; g1, g2 the two gate MLPs' sigmoid outputs, each one broadcast row (1, d)
 * (per_row 0: the gate has no context features) or one row per sample (B, d) (per_row 1).
 * b2_fs_gate_fwd: f1, f2 (B, d) "=" e * (2 g1), e * (2 g2) (2 g first, then the product, as the reference rounds);
 *   f1_aux, f2_aux (both or neither, row pitch ld_aux) receive their GEMM operand copies for the towers' first
 *   layers: the bf16 rounding (aux_dtype B2_BF16) or the 3xTF32 small part (B2_F32).
 * b2_fs_gate_bwd: de (B, d) "=" df1 (2 g1) + df2 (2 g2); dg_s = 2 (df_s e): (B, d) "=" for a per-row gate, or for a
 *   broadcast gate its column sum (d) "+=" (caller zeroes): a per-CTA sum, then one float atomic per column and CTA.
 *
 * Aggregation: x (B, dx), y (B, dy) the towers' outputs, H heads of widths hx = dx / H, hy = dy / H, and
 *   out_b = w_x.x_b + b_x + w_y.y_b + b_y + sum_h x_{b,h}^T W_h y_{b,h},  W_h[i, j] = w_xy[(h hx + i) hy + j]
 * with w_x (dx), w_y (dy), b_x, b_y (1) and w_xy (H hx hy) the reference's w_x, w_y and w_xy.  With
 * n_aug = B2_AGG_COLS(dy), the smallest multiple of 4 above dy:
 *   W_aug (n_aug, dx) K-major: row h hy + j holds W_h[:, j] in columns h hx .. h hx + hx - 1 and zeros elsewhere,
 *     row dy is w_x, rows dy + 1 .. are zero; bias_aug (n_aug) = [w_y, 0 ...]
 *   Q (B, n_aug) = x W_aug^T + bias_aug (the caller's GEMM): Q[:, :dy] = T + w_y with T_b = [x_{b,h}^T W_h]_h,
 *     Q[:, dy] = x w_x
 *   ys (B, n_aug) = [g y | g | 0] for the output gradient g (B): dx = ys W_aug, dW_aug = ys^T x (the caller's GEMMs)
 * Range: dx, dy >= 1, H divides both, batch * n_aug < 2^31; dy % 4 == 0 with 16-byte aligned rows takes a float4
 * path, anything else a scalar one.  Outside the range, or given a NULL pointer, every entry point returns
 * B2_E_INVALID.
 * b2_agg_pack:   W_aug, bias_aug "=" from w_xy, w_x, w_y; one launch.
 * b2_agg_fwd:    out (B) "=" sum_{j < dy} y_j Q_j + Q_dy + b_x + b_y; one warp per row.
 * b2_agg_bwd:    gy (B, dy) "=" g Q[:, :dy]; ys "=" (+ ys_aux as the gate's f1_aux, row width n_aug); gw_y (dy) "+="
 *   the column sums of g y, gb_x and gb_y (1) each "+=" the sum of g (caller zeroes all three).
 * b2_agg_unpack: gw_xy (H hx hy) "=" the diagonal blocks of dW_aug, gw_x (dx) "=" its row dy.
 */
#define B2_AGG_COLS(dy) (((dy) + 4) / 4 * 4)
B2_API int b2_fs_gate_fwd(const float* e, const float* g1, const float* g2, int per_row1, int per_row2, int64_t batch,
                          int d, float* f1, float* f2, void* f1_aux, void* f2_aux, int aux_dtype, int64_t ld_aux,
                          void* stream);
B2_API int b2_fs_gate_bwd(const float* e, const float* g1, const float* g2, int per_row1, int per_row2,
                          const float* df1, const float* df2, int64_t batch, int d, float* de, float* dg1, float* dg2,
                          void* stream);
B2_API int b2_agg_pack(const float* w_xy, const float* w_x, const float* w_y, int dx, int dy, int heads, float* W_aug,
                       float* bias_aug, void* stream);
B2_API int b2_agg_fwd(const float* Q, const float* y, const float* b_x, const float* b_y, int64_t batch, int dy,
                      float* out, void* stream);
B2_API int b2_agg_bwd(const float* Q, const float* y, const float* g, int64_t batch, int dy, float* gy, float* ys,
                      void* ys_aux, int aux_dtype, int64_t ld_aux, float* gw_y, float* gb_x, float* gb_y,
                      void* stream);
B2_API int b2_agg_unpack(const float* dW_aug, int dx, int dy, int heads, float* gw_xy, float* gw_x, void* stream);

/*
 * MaskNet (model_zoo/MaskNet/src/MaskNet.py).  All row-major fp32.  LayerNorm is nn.LayerNorm's: biased variance
 * over the row, eps inside the square root, y = (x - mean) rstd gamma + beta; the kernels take the mean first and
 * then the variance from the centred values.  Widths (dim, n) lie in [1, B2_MASKNET_MAX_WIDTH]; dim % 4 == 0 (n % 4)
 * with 16-byte aligned rows, parameters and pitches takes a float4 path, anything else a scalar one.  Outside the
 * range, or given a NULL pointer, every entry point returns B2_E_INVALID.
 *
 * Embedding LayerNorm: x (B, F, D) = the embedding, field f normalised by its own nn.LayerNorm(D), whose weight and
 * bias lie at gamma + f pstride and beta + f pstride (pstride in floats; the fused optimizer's arena interleaves
 * them as [gamma_0 | beta_0 | gamma_1 | ...], so gamma = &gamma_0, beta = &beta_0 and pstride = 2 round4(D)).  One
 * launch each way covers all F fields.
 * b2_field_ln_fwd: out (B, F, D) "="; mean, rstd (B, F) "=" (saved for the backward).
 * b2_field_ln_bwd: dx (B, F, D) "=" (accumulate 0) or "+=" (accumulate 1) the input gradient for the output
 *   gradient g (B, F, D); dgamma, dbeta (at the parameters' stride) "+=" (caller zeroes) the sums over the batch:
 *   a per-CTA sum, then one float atomic per column and CTA.
 *
 * MaskBlock, out = dropout(act(LN(z))) with z = (V_mask * v_in) W^T (B, n) the hidden Linear's output (the GEMM
 * before this kernel).  gamma, beta (n) NULL: the block has no LayerNorm (out = dropout(act(z))).  act: B2_ACT_NONE,
 * B2_ACT_RELU or B2_ACT_SIGMOID.  drop_rng != NULL: dropout with the mask of "Dropout masks" over the (B, n) block
 * output at counter offset snapshot offset + drop_layer.
 * b2_mask_row_fwd: out "=" at row pitch ld_out (a column slice of a wider buffer); out_aux (optional, row pitch ld_aux)
 *   receives out's GEMM operand copy: its bf16 rounding (aux_dtype B2_BF16) or its 3xTF32 small part (B2_F32);
 *   mean, rstd (B) "=" with LayerNorm.
 * b2_mask_row_bwd: dz (B, n) "=" from the output gradient g (row pitch ld_g): the mask regenerated, act' of the LN
 *   output recomputed from z, mean and rstd (the value the forward had before dropout), the LN backward; dz_aux as
 *   out_aux; dgamma, dbeta (n) "+=" (caller zeroes) as in b2_field_ln_bwd.
 * b2_mask_mul: out (n) "=" (accumulate 0) or "+=" (accumulate 1) a * b: the gradient of the block input
 *   v_in = du * V_mask, du the hidden Linear's input gradient.
 */
#define B2_MASKNET_MAX_WIDTH 1024
B2_API int b2_field_ln_fwd(const float* x, int64_t batch, int fields, int dim, const float* gamma, const float* beta,
                           int64_t pstride, float eps, float* out, float* mean, float* rstd, void* stream);
B2_API int b2_field_ln_bwd(const float* x, const float* mean, const float* rstd, const float* g, int64_t batch,
                           int fields, int dim, const float* gamma, int64_t pstride, float* dx, int accumulate,
                           float* dgamma, float* dbeta, void* stream);
B2_API int b2_mask_row_fwd(const float* z, int64_t batch, int n, const float* gamma, const float* beta, float eps,
                           int act, const int64_t* drop_rng, int64_t drop_layer, uint32_t drop_thresh,
                           float drop_scale, float* out, int64_t ld_out, void* out_aux, int aux_dtype,
                           int64_t ld_aux, float* mean, float* rstd, void* stream);
B2_API int b2_mask_row_bwd(const float* z, const float* mean, const float* rstd, const float* gamma, const float* beta,
                           int act, const int64_t* drop_rng, int64_t drop_layer, uint32_t drop_thresh,
                           float drop_scale, const float* g, int64_t ld_g, int64_t batch, int n, float* dz,
                           void* dz_aux, int aux_dtype, int64_t ld_aux, float* dgamma, float* dbeta, void* stream);
B2_API int b2_mask_mul(const float* a, const float* b, int64_t n, float* out, int accumulate, void* stream);

/*
 * AutoInt's multi-head field self-attention (model_zoo/AutoInt/src/AutoInt.py, MultiHeadSelfAttention), one layer on
 * X (B, F, d_in):
 *   Z = concat_h dropout(softmax(Q_h K_h^T [/ scale])) V_h + R,   out = ReLU(LN(Z))   (LN optional)
 * with Q, K, V = X W_q^T, X W_k^T, X W_v^T of width A = attention_dim, H heads of width dh = A / H, scale = sqrt(dh)
 * or 0 (no scaling), and R = X (res_mode 1, d_in == A), X W_res^T (res_mode 2) or 0 (res_mode 0).  All row-major
 * fp32; NP = 4A with W_res, 3A without:
 *   Wp (NP, d_in) K-major: rows 0 .. A-1 W_q, A .. 2A-1 W_k, 2A .. 3A-1 W_v, 3A .. 4A-1 W_res
 *   P  (B F, NP) = X Wp^T (the caller's GEMM): columns [Q | K | V | X W_res^T] per field row
 *   dP (B F, NP): [dQ | dK | dV | dR]; dX = dP Wp (+ dR for an identity residual) and dWp = dP^T X (the caller's
 *     GEMMs)
 * Saved for the backward: P, X, out, the softmax max and sum per (b, h, i) (stat_max, stat_sum (B, H, F)) and with
 * LayerNorm its mean and rstd per row (ln_mean, ln_rstd (B F)).  No (B, H, F, F) tensor is stored: the backward
 * recomputes the probabilities.  Dropout (drop_rng != NULL) drops attention weight (b, h, i, j) with the mask of
 * "Dropout masks" over the (B H F, F) weights at counter offset snapshot offset + drop_layer.  LayerNorm is
 * nn.LayerNorm(A)'s (mean first, then the biased variance from the centred values, eps inside the square root).
 * Range: 1 <= F <= B2_AUTOINT_MAX_FIELDS, 1 <= A <= B2_AUTOINT_MAX_DIM, any H dividing A, d_in >= 1, batch >= 0
 * (0: no launch) with batch F 4A < 2^31.  A % 4 == 0 with a 16-byte aligned P stages through float4 loads, anything
 * else through scalar ones.  Outside the range, or given a NULL pointer, every entry point returns B2_E_INVALID.
 * b2_autoint_pack:   Wp "=" from W_q, W_k, W_v and W_res (NULL: none); one launch.
 * b2_autoint_fwd:    out (B F, A) "="; out_aux (optional, row pitch ld_aux) receives out's GEMM operand copy for the
 *   next layer: its bf16 rounding (aux_dtype B2_BF16) or its 3xTF32 small part (B2_F32); the statistics "=".
 * b2_autoint_bwd:    dP "=" (+ dp_aux as out_aux, row width NP) from the output gradient g (B F, A) and the saved
 *   tensors; gres (B F, A) "=" dR for an identity residual; dgamma, dbeta (A) "+=" (caller zeroes): a per-CTA sum,
 *   then one float atomic per column and CTA.
 * b2_autoint_unpack: gW_q, gW_k, gW_v (, gW_res) (A, d_in) "=" from dWp.
 */
#define B2_AUTOINT_MAX_FIELDS 64
#define B2_AUTOINT_MAX_DIM 64
B2_API int b2_autoint_pack(const float* Wq, const float* Wk, const float* Wv, const float* Wres, int din, int A,
                           float* Wp, void* stream);
B2_API int b2_autoint_fwd(const float* P, const float* X, int64_t batch, int fields, int din, int A, int heads,
                          int res_mode, float scale, const float* gamma, const float* beta, float eps,
                          const int64_t* drop_rng, int64_t drop_layer, uint32_t drop_thresh, float drop_scale,
                          float* out, void* out_aux, int aux_dtype, int64_t ld_aux, float* stat_max, float* stat_sum,
                          float* ln_mean, float* ln_rstd, void* stream);
B2_API int b2_autoint_bwd(const float* P, const float* X, const float* out, const float* g, const float* stat_max,
                          const float* stat_sum, const float* ln_mean, const float* ln_rstd, int64_t batch,
                          int fields, int din, int A, int heads, int res_mode, float scale, const float* gamma,
                          const int64_t* drop_rng, int64_t drop_layer, uint32_t drop_thresh, float drop_scale,
                          float* dP, void* dp_aux, int aux_dtype, int64_t ld_aux, float* gres, float* dgamma,
                          float* dbeta, void* stream);
B2_API int b2_autoint_unpack(const float* dWp, int din, int A, float* gWq, float* gWk, float* gWv, float* gWres,
                             void* stream);

/*
 * BST, the Behavior Sequence Transformer (model_zoo/BST/src/BST.py): TransformerBlocks over the L = max_len + 1 tokens
 * of a (target, sequence) pair, model_dim md = D (nf + use_pos) for nf fields per token of width D.  All row-major
 * fp32.  Token b L + t of X (B L, md) is [seq_0[b, t] .. seq_{nf-1}[b, t] | pos[t]] for t < L - 1 and
 * [tgt_0[b] .. tgt_{nf-1}[b] | pos[L - 1]] for t = L - 1.  valid (B, L - 1) bytes: 1 for a real history slot,
 * 0 for padding (sequence id 0).  A block on X, with the caller's GEMMs (bias in their epilogues):
 *   QKV = X W_in^T + b_in (B L, 3 md)            columns [Q | K | V], head h the columns h dh .. h dh + dh - 1
 *   ctx = b2_bst_attn_fwd(QKV)                   per head: dropout(softmax((q scale) k^T + mask)) v, scale =
 *                                                sqrt(1 / dh) as the caller rounds it; key j masked for query i iff
 *                                                j != i and (j is padding, or causal and j > i)
 *   s   = b2_bst_addnorm_fwd(ctx W_o^T + b_o, X)  LN1(X + dropout1(.))
 *   out = b2_bst_addnorm_fwd(FFN(s), s)           LN2(s + FFN(s)), FFN = dropout2(W2 LeakyReLU(W1 s + b1) + b2) as a
 *                                                two-layer MLP chain (B2_ACT_LEAKY_RELU in the first epilogue)
 * Saved for the backward: QKV, ctx and the softmax max and sum per (b, h, i) (stat_max, stat_sum (B, H, L)); no
 * (B H, L, L) tensor is stored.  Attention dropout drops weight (b, h, i, j) with the mask of "Dropout masks" over the
 * (B H L, L) weights, the add-norm's dropout element (r, c) of its (rows, n) input a; each at counter offset
 * snapshot offset + drop_layer.  LayerNorm is nn.LayerNorm's (mean first, then the biased variance from the centred
 * values, eps inside the square root).  Every output with an aux argument (row pitch ld_aux) also receives its GEMM
 * operand copy: bf16 rounding (aux_dtype B2_BF16) or 3xTF32 small part (B2_F32).
 * Range: 2 <= L <= B2_BST_MAX_LEN, 1 <= md <= B2_BST_MAX_DIM, 1 <= heads <= B2_BST_MAX_HEADS dividing md with
 * dh = md / heads <= B2_BST_MAX_HEAD_DIM, 1 <= nf <= B2_BST_MAX_PARTS, batch >= 0 (0: no launch) with batch L < 2^31.
 * The attention kernels stage 2 L (dh + 1) floats per (sample, head) in shared memory.  Outside the range, or given a
 * NULL pointer, every entry point returns B2_E_INVALID.
 * b2_bst_tokens_fwd:  X "=" from nf sequence views seq[f] (B, L - 1, D; sample b at seq[f] + b seq_ld[f], its tokens
 *   contiguous), nf target views tgt[f] (B, D; row pitch tgt_ld[f]) and the position table pos (L, D; NULL: none).
 *   seq, seq_ld, tgt, tgt_ld are host arrays of nf entries.
 * b2_bst_tokens_bwd:  from G = g (+ g2, NULL: none) (B L, md): dseq[f] (B, L - 1, D) and dtgt[f] (B, D) "=" (host
 *   arrays of device pointers, contiguous), dpos (L, D) "+=" the batch sum of G's position columns (use_pos).
 * b2_bst_attn_fwd:    ctx (B L, md) and the statistics "=".
 * b2_bst_attn_bwd:    dQKV (B L, 3 md) "=" [dQ | dK | dV] from dctx and the saved tensors.
 * b2_bst_addnorm_fwd: out (rows, n) "=" LN(res + dropout(a)); res NULL: no residual; gamma, beta NULL: no LayerNorm
 *   (then ln_mean, ln_rstd are not written).
 * b2_bst_addnorm_bwd: from G = g (+ g2): dres "=" dz (NULL: not written), da "=" keep scale dz, with
 *   dz = LN'(G); dgamma, dbeta (n) "+=" (caller zeroes): a per-CTA sum, then one float atomic per column and CTA.
 * b2_bst_pool_fwd:    out[b, :] (row pitch ld_out) "=" the pooling of sample b's L tokens of x (B L, md):
 *   B2_BST_POOL_SUM sum of the real slots and the target, B2_BST_POOL_MEAN that sum / (count + 1e-12),
 *   B2_BST_POOL_TARGET the last token.  (concat pooling is X's flat view and needs no kernel.)
 * b2_bst_pool_bwd:    dx (B L, md) "=" from g (row pitch ld_g).
 */
#define B2_BST_MAX_LEN 256
#define B2_BST_MAX_DIM 512
#define B2_BST_MAX_HEAD_DIM 64
#define B2_BST_MAX_HEADS 16
#define B2_BST_MAX_PARTS 8
#define B2_BST_POOL_MEAN 0
#define B2_BST_POOL_SUM 1
#define B2_BST_POOL_TARGET 2
B2_API int b2_bst_tokens_fwd(const float* const* seq, const int64_t* seq_ld, const float* const* tgt,
                             const int64_t* tgt_ld, int nf, const float* pos, int64_t batch, int L, int D, float* tok,
                             void* tok_aux, int aux_dtype, int64_t ld_aux, void* stream);
B2_API int b2_bst_tokens_bwd(const float* g, const float* g2, int64_t batch, int L, int D, int nf, int use_pos,
                             float* const* dseq, float* const* dtgt, float* dpos, void* stream);
B2_API int b2_bst_attn_fwd(const float* qkv, const uint8_t* valid, int64_t batch, int L, int md, int heads, int causal,
                           float scale, const int64_t* drop_rng, int64_t drop_layer, uint32_t drop_thresh,
                           float drop_scale, float* ctx, void* ctx_aux, int aux_dtype, int64_t ld_aux, float* stat_max,
                           float* stat_sum, void* stream);
B2_API int b2_bst_attn_bwd(const float* qkv, const uint8_t* valid, const float* ctx, const float* dctx,
                           const float* stat_max, const float* stat_sum, int64_t batch, int L, int md, int heads,
                           int causal, float scale, const int64_t* drop_rng, int64_t drop_layer, uint32_t drop_thresh,
                           float drop_scale, float* dqkv, void* dqkv_aux, int aux_dtype, int64_t ld_aux, void* stream);
B2_API int b2_bst_addnorm_fwd(const float* a, const float* res, int64_t rows, int n, const float* gamma,
                              const float* beta, float eps, const int64_t* drop_rng, int64_t drop_layer,
                              uint32_t drop_thresh, float drop_scale, float* out, void* out_aux, int aux_dtype,
                              int64_t ld_aux, float* ln_mean, float* ln_rstd, void* stream);
B2_API int b2_bst_addnorm_bwd(const float* a, const float* res, const float* g, const float* g2, int64_t rows, int n,
                              const float* gamma, const float* ln_mean, const float* ln_rstd, const int64_t* drop_rng,
                              int64_t drop_layer, uint32_t drop_thresh, float drop_scale, float* da, void* da_aux,
                              int aux_dtype, int64_t ld_aux, float* dres, float* dgamma, float* dbeta, void* stream);
B2_API int b2_bst_pool_fwd(const float* x, const uint8_t* valid, int64_t batch, int L, int md, int mode, float* out,
                           int64_t ld_out, void* stream);
B2_API int b2_bst_pool_bwd(const float* g, int64_t ld_g, const uint8_t* valid, int64_t batch, int L, int md, int mode,
                           float* dx, void* stream);

/*
 * TransAct (model_zoo/TransAct/src/TransAct.py): a post-norm nn.TransformerEncoder over the L = max_len early-fusion
 * tokens of a (target, sequence) pair.  All row-major fp32.  Token b L + t of X (B L, md), md = D (ns + nt), is
 * [seq_0[b, t] .. seq_{ns-1}[b, t] | tgt_0[b] .. tgt_{nt-1}[b]].  valid (B, L) bytes: 1 where the first sequence
 * field's id is non-zero, and the last slot of a sample with no such slot (TransActTransformer.adjust_mask).  A layer
 * on X, with the caller's GEMMs (bias in their epilogues) and bst.cu's add-norm:
 *   QKV = X W_in^T + b_in (B L, 3 md)            columns [Q | K | V], head h the columns h dh .. h dh + dh - 1
 *   ctx = b2_transact_attn_fwd(QKV)              per head: dropout(softmax((q scale) k^T + mask)) v, scale =
 *                                                sqrt(1 / dh) as the caller rounds it; key j masked iff !valid[b, j]
 *   s   = b2_bst_addnorm_fwd(ctx W_o^T + b_o, X)  norm1(X + dropout1(.))
 *   out = b2_bst_addnorm_fwd(FFN(s), s)           norm2(s + dropout2(W2 dropout(relu(W1 s + b1)) + b2))
 * The attention skips padded query rows: their ctx, dQ, dK and dV rows are 0 (the model zeroes those rows, and as
 * keys they are masked in every layer).  Saved for the backward: QKV, ctx and the softmax max and sum per (b, h, i)
 * (stat_max, stat_sum (B, H, L)); no (B H, L, L) tensor is stored.  Attention dropout drops weight (b, h, i, j) with
 * the mask of "Dropout masks" over the (B H L, L) weights, at counter offset snapshot offset + drop_layer.  Every
 * output with an aux argument (row pitch ld_aux) also receives its GEMM operand copy: bf16 rounding (aux_dtype
 * B2_BF16) or 3xTF32 small part (B2_F32).
 * Range: 1 <= L <= B2_TRANSACT_MAX_LEN, 1 <= md <= B2_TRANSACT_MAX_DIM, 1 <= heads <= B2_TRANSACT_MAX_HEADS dividing
 * md with dh = md / heads <= B2_TRANSACT_MAX_HEAD_DIM, ns, nt >= 1 with ns + nt <= B2_TRANSACT_MAX_PARTS,
 * 1 <= k <= L, batch >= 0 (0: no launch) with batch L < 2^31.  Shared memory holds tiles of 32 rows of dh (+ 1)
 * floats, independent of L.  Outside the range, or given a NULL pointer, every entry point returns B2_E_INVALID.
 * b2_transact_tokens_fwd: X "=" from ns sequence views seq[f] (B, L, D; sample b at seq[f] + b seq_ld[f], its tokens
 *   contiguous) and nt target views tgt[f] (B, D; row pitch tgt_ld[f]) (host arrays of ns / nt entries), and valid
 *   "=" from ids (B, L; row pitch ld_ids; B2_F64, B2_I64, B2_I32 or B2_F32), in one launch.
 * b2_transact_tokens_bwd: from G (B L, md): dseq[f] (B, L, D) "=" and dtgt[f] (B, D) "=" the sum over t (host arrays
 *   of device pointers, contiguous); no float atomics.
 * b2_transact_attn_fwd: ctx (B L, md) and the statistics "=".
 * b2_transact_attn_bwd: dQKV (B L, 3 md) "=" [dQ | dK | dV] from dctx and the saved tensors, in two launches: dQ
 *   query-block outer (also delta (B, H, L) "=" dO_i . O_i, a workspace), then dK and dV key-block outer; no float
 *   atomics.
 * b2_transact_out_fwd: last (B, k md) "=" the last k slots of y (B L, md), 0 where padded; maxv (B, md) "=" the max
 *   over L of y with padded slots at -1e9 and argmax (B, md) its slot, the first on ties (NULL, NULL: no pooling).
 * b2_transact_out_bwd: dy (B L, md) "=" from dlast and dmax (NULL: no pooling) through argmax; 0 at padded slots.
 */
#define B2_TRANSACT_MAX_LEN 256
#define B2_TRANSACT_MAX_DIM 512
#define B2_TRANSACT_MAX_HEAD_DIM 256
#define B2_TRANSACT_MAX_HEADS 16
#define B2_TRANSACT_MAX_PARTS 8
B2_API int b2_transact_tokens_fwd(const float* const* seq, const int64_t* seq_ld, int ns, const float* const* tgt,
                                  const int64_t* tgt_ld, int nt, const void* ids, int ids_dtype, int64_t ld_ids,
                                  int64_t batch, int L, int D, float* tok, void* tok_aux, int aux_dtype,
                                  int64_t ld_aux, uint8_t* valid, void* stream);
B2_API int b2_transact_tokens_bwd(const float* g, int64_t batch, int L, int D, int ns, int nt, float* const* dseq,
                                  float* const* dtgt, void* stream);
B2_API int b2_transact_attn_fwd(const float* qkv, const uint8_t* valid, int64_t batch, int L, int md, int heads,
                                float scale, const int64_t* drop_rng, int64_t drop_layer, uint32_t drop_thresh,
                                float drop_scale, float* ctx, void* ctx_aux, int aux_dtype, int64_t ld_aux,
                                float* stat_max, float* stat_sum, void* stream);
B2_API int b2_transact_attn_bwd(const float* qkv, const uint8_t* valid, const float* ctx, const float* dctx,
                                const float* stat_max, const float* stat_sum, int64_t batch, int L, int md, int heads,
                                float scale, const int64_t* drop_rng, int64_t drop_layer, uint32_t drop_thresh,
                                float drop_scale, float* delta, float* dqkv, void* dqkv_aux, int aux_dtype,
                                int64_t ld_aux, void* stream);
B2_API int b2_transact_out_fwd(const float* y, const uint8_t* valid, int64_t batch, int L, int md, int k, float* last,
                               float* maxv, int32_t* argmax, void* max_aux, int aux_dtype, int64_t ld_aux,
                               void* stream);
B2_API int b2_transact_out_bwd(const float* dlast, const float* dmax, const int32_t* argmax, const uint8_t* valid,
                               int64_t batch, int L, int md, int k, float* dy, void* stream);

/*
 * DIEN, the Deep Interest Evolution Network (model_zoo/DIEN/src/DIEN.py): the interest extractor (nn.GRU), the
 * attention between the interests and the target, and the interest-evolution GRU (AUGRU, AGRU or nn.GRU) over a
 * behaviour sequence.  All row-major fp32.
 * A GRU over x (B, L, H) (sample b at x + b ld_x, its L tokens contiguous) with W_ih, W_hh (3H, H), b_ih, b_hh (3H):
 *   gi = W_ih x_t + b_ih, gh = W_hh h + b_hh, chunks c0, c1, c2 of H each; one update h' = h + g (n - h) with
 *   B2_DIEN_GRU   (nn.GRU, chunks r, z, n):     r = s(gi0 + gh0), z = s(gi1 + gh1), n = tanh(gi2 + r gh2), g = 1 - z
 *   B2_DIEN_AUGRU (AUGRUCell, chunks u, r, n): u = s(gi0 + gh0), r = s(gi1 + gh1), n = tanh(gi2 + r gh2), g = a_t u
 *   B2_DIEN_AGRU  (AGRUCell, chunks u, r, n):  r = s(gi1 + gh1), n = tanh(gi2 + r gh2), g = a_t (chunk u unused)
 * with s the logistic sigmoid and a (B, L) the attention (NULL for B2_DIEN_GRU).  Sample b's length len_b is the number
 * of non-zero bytes of its row of mask (B, L) (pad_mask.sum(1), the first sequence field's id > 0); the recurrence runs
 * over positions [0, len_b) from h = 0, wherever the zeros are (as pack_padded_sequence does).
 * b2_gru_fwd: h_seq (B, L, H) "=": the state after step t for t < len_b, 0 from len_b on (pad_packed_sequence's
 *   padding); h_last (B, H) "=" (NULL: not written): the state after step len_b - 1, 0 for an empty history.
 * b2_gru_bwd: the reverse-time recurrence from the saved h_seq, recomputing the gates from h_{t-1} and x_t.
 *   dh_seq (B, L, H) (NULL: none) and dh_last (B, H) (NULL: none) are the gradients of the forward's outputs.
 *   dx (B, L, H) "=" (accumulate 0: zero from len_b on) or "+=" (accumulate 1); da (B, L) "=" (zero from len_b on;
 *   NULL for B2_DIEN_GRU); dW_ih, dW_hh (3H, H), db_ih, db_hh (3H) "+=" (caller zeroes): a per-CTA sum in shared
 *   memory, then one float atomic per element and CTA.
 * Both keep W_ih and W_hh in shared memory and give each sample a group of G threads, G the power of two >= H: thread j
 *   of the group owns hidden unit j.  No (B L, 3H) gate tensor is formed.
 * b2_dien_scores_fwd: the bilinear (W (H, H)) or dot (W NULL) attention of AttentionLayer: q_b = W t_b (t_b for dot),
 *   q (B, H) "=", s (B, L) "=" <h_seq[b, t], q_b> mask[b, t].  t (B, H) at row pitch ld_t.
 * b2_dien_scores_bwd: from ds (B, L): dh_seq[b, t] "+=" (accumulate 1) or "=" (0) ds mask q_b; dq (B, H) "=" the sum
 *   over t of ds mask h_seq[b, t]; dt (B, H) "=" W^T dq (dq for dot).  dW = dq^T t is the caller's GEMM.
 * b2_dien_sum_pool_fwd: out[b] (row pitch ld_out) "=" [sum_t x[b, t] | t_b * sum_t x[b, t]] (2H), DIEN's sum pooling of
 *   the zero-padded sequence and its product with the target (enable_sum_pooling).
 * b2_dien_sum_pool_bwd: from g (B, 2H) at row pitch ld_g: dx[b, t] "+=" (accumulate 1) or "=" (0) g1 + t_b g2 for every
 *   t; dt (B, H) "+=" (accumulate 1) or "=" (0) sum_t x[b, t] g2.
 * Range: 1 <= H <= B2_DIEN_MAX_DIM, 1 <= L <= B2_DIEN_MAX_LEN, batch >= 0 (0: no launch), batch L < 2^31.  Outside the
 * range, or given a NULL pointer, every entry point returns B2_E_INVALID.
 */
#define B2_DIEN_MAX_DIM 64
#define B2_DIEN_MAX_LEN 1024
#define B2_DIEN_GRU 0
#define B2_DIEN_AUGRU 1
#define B2_DIEN_AGRU 2
B2_API int b2_gru_fwd(const float* x, int64_t ld_x, const uint8_t* mask, const float* W_ih, const float* b_ih,
                      const float* W_hh, const float* b_hh, const float* att, int cell, int64_t batch, int L, int H,
                      float* h_seq, float* h_last, void* stream);
B2_API int b2_gru_bwd(const float* x, int64_t ld_x, const uint8_t* mask, const float* W_ih, const float* b_ih,
                      const float* W_hh, const float* b_hh, const float* att, int cell, int64_t batch, int L, int H,
                      const float* h_seq, const float* dh_seq, const float* dh_last, float* dx, int accumulate,
                      float* da, float* dW_ih, float* db_ih, float* dW_hh, float* db_hh, void* stream);
B2_API int b2_dien_scores_fwd(const float* h_seq, const float* t, int64_t ld_t, const float* W, const uint8_t* mask,
                              int64_t batch, int L, int H, float* q, float* s, void* stream);
B2_API int b2_dien_scores_bwd(const float* h_seq, const float* t, int64_t ld_t, const float* W, const uint8_t* mask,
                              const float* q, const float* ds, int64_t batch, int L, int H, float* dh_seq,
                              int accumulate, float* dq, float* dt, void* stream);
B2_API int b2_dien_sum_pool_fwd(const float* x, const float* t, int64_t ld_t, int64_t batch, int L, int H, float* out,
                                int64_t ld_out, void* stream);
B2_API int b2_dien_sum_pool_bwd(const float* x, const float* t, int64_t ld_t, const float* g, int64_t ld_g,
                                int64_t batch, int L, int H, float* dx, float* dt, int accumulate, void* stream);

/*
 * LSH over a long behaviour sequence: ETA's SimHash top-k retrieval (model_zoo/LongCTR/ETA/ETA.py) and SDIM's
 * hash-collision pooling (model_zoo/LongCTR/SDIM/SDIM.py).  x is item_feat_emb (B, L + 1, d) row-major fp32: positions
 * [0, L) the history, position L the target; mask (B, L) bytes, non-zero = valid.  Sample b's rotations start at
 * R + b r_stride (r_stride 0: one shared set).  SimHash bit j of a row v is v . R[:, j] > 0 (bit 0 at exactly 0), the
 * projection in fp32 FMA over ascending columns.
 * b2_eta_retrieve_fwd: R (d, bits).  dist_l = popc(code_l ^ code_target), 1 + bits where mask is 0.  Writes the k
 *   smallest, sorted by (distance, position): ties go to the lower position.  topk_emb (B, k, d), topk_mask (B, k)
 *   bytes (mask != 0 at the chosen position) and topk_pos (B, k) int32, all "=".
 * b2_sdim_pool_fwd: R (d, num_hashes, bits).  Bucket h of a row is its bits-bit code under R[:, h, :]; position l
 *   collides in hash h when its bucket equals the target's and mask[l] != 0.  sums (B, num_hashes, d) "=" the sum of the
 *   colliding rows per hash (zero when none), collide (B, L) "=" one bit per hash, out (B, d) "=" the mean over hashes
 *   of sums, each first divided by max(|sum|, 1e-12) when l2norm (F.normalize).
 * b2_eta_assemble_bwd / b2_sdim_assemble_bwd: dx (B, L + 1, d) "=", every row written once.  Row L = dt0 + dt1 + dt2
 *   (each (B, d)).  Rows [L - S, L) add dshort (B, S, d).  ETA adds dlong (B, k, d) at the positions topk_pos.  SDIM
 *   adds, for each hash h position l collides in, (dlong / num_hashes) times the Jacobian of F.normalize at sums[b, h]
 *   when l2norm (1 / max(|s|, 1e-12) below the clamp), dlong (B, d) / num_hashes without.
 * Range: 1 <= d <= B2_LSH_MAX_DIM, 1 <= L <= B2_LSH_MAX_LEN, batch (L + 1) < 2^31, batch >= 0 (0: no launch);
 * ETA 1 <= bits <= B2_ETA_MAX_BITS and 1 <= k <= min(L, B2_LSH_MAX_TOPK); SDIM 1 <= bits <= B2_SDIM_MAX_BITS (a wider
 * bucket is no longer exact as the reference's float code . powers_of_two), 1 <= num_hashes <= B2_SDIM_MAX_HASHES,
 * 1 <= S <= L, and the shared memory a CTA needs within B2_LSH_MAX_SMEM bytes: ETA 4 d bits + 4 k + 4 bits + L + 16,
 * SDIM 4 d num_hashes bits + 4 (256 / d) num_hashes d + 4 num_hashes + 4 L.  Outside the range, or given a NULL
 * pointer, every entry point returns B2_E_INVALID.
 */
#define B2_LSH_MAX_DIM 256
#define B2_LSH_MAX_LEN 4096
#define B2_LSH_MAX_TOPK 256
#define B2_LSH_MAX_SMEM (227 * 1024 - 1024)
#define B2_ETA_MAX_BITS 64
#define B2_SDIM_MAX_BITS 24
#define B2_SDIM_MAX_HASHES 32
B2_API int b2_eta_retrieve_fwd(const float* x, const uint8_t* mask, const float* R, int64_t r_stride, int64_t batch,
                               int L, int d, int bits, int k, float* topk_emb, uint8_t* topk_mask, int32_t* topk_pos,
                               void* stream);
B2_API int b2_sdim_pool_fwd(const float* x, const uint8_t* mask, const float* R, int64_t r_stride, int64_t batch,
                            int L, int d, int num_hashes, int bits, int l2norm, float* out, float* sums,
                            uint32_t* collide, void* stream);
B2_API int b2_eta_assemble_bwd(const float* dt0, const float* dt1, const float* dt2, const float* dshort, int S,
                               const float* dlong, const int32_t* topk_pos, int64_t batch, int L, int d, int k,
                               float* dx, void* stream);
B2_API int b2_sdim_assemble_bwd(const float* dt0, const float* dt1, const float* dt2, const float* dshort, int S,
                                const float* dlong, const float* sums, const uint32_t* collide, int64_t batch, int L,
                                int d, int num_hashes, int l2norm, float* dx, void* stream);

/*
 * MIRRN (model_zoo/LongCTR/MIRRN/MIRRN.py): three SimHash retrievals over a long behaviour sequence and a FilterLayer2
 * block on each.  x is item_feat_emb (B, L + 1, d) row-major fp32: positions [0, L) the history h, position L the
 * target t; mask (B, L) bytes, non-zero = valid.  k = min(topk, L).  The retrieved rows, their filter outputs and
 * their gradients u, y, du (3, B, k, d) hold retrieval q's rows as the contiguous (B k, d) block q.
 * b2_mirrn_retrieve_fwd: queries t, the masked mean of h[:, L - min(16, L):] and the masked mean of all of h (each
 *   hashed from its masked sum: the division by count + 1e-9 keeps every sign).  Bit j of a row is row . R_q[:, j] > 0
 *   in fp32 FMA over ascending columns, R_q = R + q r_stride (r_stride 0: one (d, bits) set for all three, and the
 *   history is hashed once).  dist_l = popc(code_l ^ code_q), 1 + bits where mask is 0.  topk_pos (B, 3, k) int32
 *   "=" per query the k smallest, ties to the lower position, in ascending position order.
 * b2_mirrn_filter_fwd: u[q, b, s] "=" x[b, p] + 0.02 pos_table[L - p] (p = topk_pos[b, q, s]; pos_table (pos_rows, d)
 *   with pos_rows > L), y[q, b, s, c] "=" a_c u[q, b, s, c] + b_c sum_r htab[(s - r) mod k] u[q, b, r, c], with
 *   (a_c, b_c) = cw_q[n, j, j, 0:2], c = n (d / 4) + j, cw_q the (4, d / 4, d / 4, 2) complex_weight of block q, htab
 *   (k) the first column of the filter's circulant.  LN(u + dropout(y)) is b2_bst_addnorm_fwd on each block q.
 * b2_mirrn_filter_bwd: from dy (the add-norm's da) and dres (its dres; dy itself without dropout): du "=" dres +
 *   a dy - b (H dy); dcw_q[n, j, j, 0] "+=" sum dy u, dcw_q[n, j, j, 1] "+=" sum dy (H u), dpos[L - p] "+=" 0.02 du
 *   (caller zeroes; float atomics: one per CTA and channel for dcw, one per element for dpos).
 * b2_mirrn_mean_fwd / _bwd: out (B, 3, d) "=" the mean of z (3, B, k, d) over the k slots; dz "=" g / k.
 * b2_mirrn_assemble_bwd: dx (B, L + 1, d) "=", every row written once, no atomics.  Row L = dt0 + dt1 + dt2 (each
 *   (B, d)); rows [L - S, L) add dshort (B, S, d); row p adds du[q, b, s] for every (q, s) with topk_pos[b, q, s] = p,
 *   in the order q = 0, 1, 2.
 * Range: d a multiple of 4 in [4, B2_LSH_MAX_DIM], 1 <= L <= B2_LSH_MAX_LEN, 1 <= k <= min(L, B2_LSH_MAX_TOPK),
 * 1 <= bits <= B2_MIRRN_MAX_BITS, batch (L + 1) < 2^31, batch >= 0 (0: no launch), 1 <= S <= L, and shared memory
 * within B2_LSH_MAX_SMEM bytes: retrieval 4 nsets d bits + 8 (256 / d) d + 8 d + 12 (bits + 2) + 24 + 3 L (nsets 1 or
 * 3), filter forward 4 k d + 8 k, backward 8 k d + 8 k + 8 (256 / d) d.  Outside the range, or given a NULL pointer,
 * every entry point returns B2_E_INVALID.
 */
#define B2_MIRRN_MAX_BITS 64
B2_API int b2_mirrn_retrieve_fwd(const float* x, const uint8_t* mask, const float* R, int64_t r_stride, int64_t batch,
                                 int L, int d, int bits, int k, int32_t* topk_pos, void* stream);
B2_API int b2_mirrn_filter_fwd(const float* x, const int32_t* topk_pos, const float* pos_table, int pos_rows,
                               const float* cw0, const float* cw1, const float* cw2, const float* htab, int64_t batch,
                               int L, int d, int k, float* u, float* y, void* stream);
B2_API int b2_mirrn_filter_bwd(const float* dy, const float* dres, const float* u, const int32_t* topk_pos,
                               int pos_rows, const float* cw0, const float* cw1, const float* cw2, const float* htab,
                               int64_t batch, int L, int d, int k, float* du, float* dcw0, float* dcw1, float* dcw2,
                               float* dpos, void* stream);
B2_API int b2_mirrn_mean_fwd(const float* z, int64_t batch, int d, int k, float* out, void* stream);
B2_API int b2_mirrn_mean_bwd(const float* g, int64_t batch, int d, int k, float* dz, void* stream);
B2_API int b2_mirrn_assemble_bwd(const float* dt0, const float* dt1, const float* dt2, const float* dshort, int S,
                                 const float* du, const int32_t* topk_pos, int64_t batch, int L, int d, int k,
                                 float* dx, void* stream);

/*
 * LongCTR input (model_zoo/LongCTR/longctr_dataloader.py, BatchCollator): the triple (batch_dict, item_dict, mask)
 * built on the device from a store of user histories and item features held in HBM.
 * b2_longctr_collate: batch (rows, row_stride) int64 or int32 (batch_dtype B2_I64 | B2_I32), the columns col_user,
 *   col_item and col_seq_len holding each sample's user_index u, item_index t and seq_len.  The histories are CSR:
 *   offsets (num_users + 1) int64, hist the flat int32 item ids, user u's history hist[offsets[u], offsets[u + 1]).
 *   item_info (num_items, num_cols) row-major int32.  With n = min(seq_len, len(history of u)) and k = min(n, L),
 *   slots [0, L) hold keras pad_sequences(maxlen = L, value = 0, padding = truncating = p) of the first n history
 *   items: the last k, right-aligned (B2_LONGCTR_PAD_PRE), or the first k, left-aligned (B2_LONGCTR_PAD_POST), 0
 *   elsewhere; slot L holds t.  mask (rows, L) fp32 "=" (id > 0) over slots [0, L); items (num_cols, rows (L + 1))
 *   int64 "=", items[c, b (L + 1) + l] = item_info[id, c] (positional: a padding slot copies row 0).  One launch.
 *   The caller guarantees 0 <= u < num_users, 0 <= t < num_items, seq_len >= 0 and every history id in
 *   [0, num_items); these are not checked on the device.
 * Range: 0 <= rows < 2^31 (0: no launch), 0 <= L <= B2_LONGCTR_MAX_LEN, 1 <= num_cols <= B2_LONGCTR_MAX_COLS, the
 * three columns inside a row, num_users, num_items >= 1, mask may be NULL when L = 0.  Outside the range, or given a
 * NULL pointer, returns B2_E_INVALID.
 */
#define B2_LONGCTR_PAD_PRE 0
#define B2_LONGCTR_PAD_POST 1
#define B2_LONGCTR_MAX_LEN (1 << 20)
#define B2_LONGCTR_MAX_COLS 64
B2_API int b2_longctr_collate(const void* batch, int batch_dtype, int64_t rows, int64_t row_stride, int col_user,
                              int col_item, int col_seq_len, const int64_t* offsets, const int32_t* hist,
                              int64_t num_users, const int32_t* item_info, int64_t num_items, int num_cols, int L,
                              int padding, float* mask, int64_t* items, void* stream);

/*
 * SIM / TWIN: learned-score top-k retrieval over a long behaviour sequence, SIM's soft-search GSU
 * (model_zoo/LongCTR/SIM/SIM.py) and TWIN's MultiHeadTopKAttention (model_zoo/LongCTR/TWIN/TWIN.py).  x is
 * item_feat_emb (B, L + 1, d) row-major fp32: positions [0, L) the history, position L the target; mask (B, L) bytes,
 * non-zero = valid.  Scores are fp32 FMA dot products over ascending columns.  The selection keeps the k largest
 * scores, sorted by (score desc, position asc): ties go to the lower position, and -0.0 ties with +0.0.
 * b2_sim_retrieve_fwd: u (B, d) = W_b^T W_a t.  qk (B, L) "=" (u . x_l) mask_l (masked positions score 0),
 *   pooled (B, d) "=" sum_l qk_l x_l, and the k best: topk_emb (B, k, d), topk_mask (B, k) bytes (mask != 0 at the
 *   chosen position) and topk_pos (B, k) int32.
 * b2_sim_gsu_bwd: dqk (B, L) "=" (dpooled . x_l) mask_l, du (B, d) "=" sum_l dqk_l x_l.
 * b2_sim_assemble_bwd: dx (B, L + 1, d) "=", every row written once.  Row L = dt0 + dt1 + dt2 + dt3 (each (B, d)).
 *   Rows [0, L): dshort (B, S, d) on rows [L - S, L), dlong (B, k, d) at the positions topk_pos, and
 *   qk_l dpooled + dqk_l u.
 * b2_twin_topk_fwd: q (B, heads d) = t W_M^T of b2_mhta_pack (the 1 / sqrt(head_dim) scale folded in).
 *   score_hl = q_h . x_l, exactly -1e9 where masked; per head the k best, a softmax over them, p (B, heads d) "="
 *   sum_s a_hs x_{pos_hs}, stats (B, heads, 2) "=" {the largest chosen score, sum of exp(score - it)} and
 *   topk_pos (B, heads, k) "=" the chosen positions.  All chosen masked: the weights are uniform over the k.
 * b2_twin_topk_bwd: from dp (B, heads d) and the forward's q, p, stats and topk_pos: dq (B, heads d) "=" and
 *   dx (B, L + 1, d) "=", every row written once.  ds_hs = a_hs (dp_h . x_l - dp_h . p_h) (0 where masked),
 *   dq_h = sum_s ds_hs x_l, dx_l = sum over the heads that chose l of (a_hs dp_h + ds_hs q_h), plus dshort on rows
 *   [L - S, L); row L = dt0 + dt1 + dq W_M (W_M (heads d, d) the forward's packed weight).
 * Range: 1 <= d <= B2_TOPK_MAX_DIM, 1 <= L <= B2_TOPK_MAX_LEN, 1 <= k <= min(L, B2_TOPK_MAX_K), batch (L + 1) < 2^31,
 * batch >= 0 (0: no launch), 1 <= S <= L; TWIN 1 <= heads <= B2_MHTA_MAX_HEADS with heads d <= B2_MHTA_MAX_WIDTH; the
 * dynamic shared memory a CTA needs within B2_TOPK_MAX_SMEM bytes (G = 256 / d column groups): SIM forward
 * 8 L + 4 d + 4 G d + 4 k, SIM backward 4 L + 4 d + 4 G d, TWIN forward 4 L + 4 d + 8 k + 4 G d, TWIN backward
 * 4 ceil(heads L / 2) + 12 heads d + 12 heads k + 4 heads.  Outside the range, or given a NULL pointer, every entry
 * point returns B2_E_INVALID.
 */
#define B2_TOPK_MAX_DIM 256
#define B2_TOPK_MAX_LEN 4096
#define B2_TOPK_MAX_K 256
#define B2_TOPK_MAX_SMEM (220 * 1024)
B2_API int b2_sim_retrieve_fwd(const float* x, const uint8_t* mask, const float* u, int64_t batch, int L, int d,
                               int k, float* qk, float* pooled, float* topk_emb, uint8_t* topk_mask,
                               int32_t* topk_pos, void* stream);
B2_API int b2_sim_gsu_bwd(const float* x, const uint8_t* mask, const float* dpooled, int64_t batch, int L, int d,
                          float* dqk, float* du, void* stream);
B2_API int b2_sim_assemble_bwd(const float* dt0, const float* dt1, const float* dt2, const float* dt3,
                               const float* dshort, int S, const float* dlong, const int32_t* topk_pos,
                               const float* qk, const float* dqk, const float* u, const float* dpooled, int64_t batch,
                               int L, int d, int k, float* dx, void* stream);
B2_API int b2_twin_topk_fwd(const float* q, const float* x, const uint8_t* mask, int64_t batch, int L, int d,
                            int heads, int k, float* p, float* stats, int32_t* topk_pos, void* stream);
B2_API int b2_twin_topk_bwd(const float* q, const float* x, const uint8_t* mask, const float* p, const float* stats,
                            const int32_t* topk_pos, const float* dp, const float* WM, const float* dt0,
                            const float* dt1, const float* dshort, int S, int64_t batch, int L, int d, int heads,
                            int k, float* dq, float* dx, void* stream);

/*
 * WuKong's layer (model_zoo/WuKong/src/WuKong.py, WuKongLayer) on x (B, F, D) with rank k, lcb + fmb = Fo output
 * fields:
 *   fm   = LN_fk(flatten(x (x^T Y)))                 Y = proj_Y (F, k); LN over F k, always affine
 *   z    = cat(FMB_MLP(fm).view(B, fmb, D), x W_lcb^T over the field axis) + R,   R = x (F == Fo) or the projection
 *          x W_res^T + b_res over the field axis
 *   out  = LN_D(z) per (b, field) (optional, one LayerNorm(D) for all fields)
 * Layouts, row-major fp32 (fp = F rounded up to a multiple of 4; pad columns are zero where written "="):
 *   X    (B, F, D)    [b, f, d]: the embedding (layout 0)
 *   X'   (B D, fp)    [b, d, f]: a layer's input (layout 1); X'_{i+1} is written at fpo = Fo rounded up to 4
 *   Ws   (N, fp)      [W_lcb; W_res] zero-padded, N = lcb (+ Fo with a projection); bs (N) = [0; b_res]
 *   C    (B D, N)     = X' Ws^T + bs (the caller's GEMM): columns [LCB out | projection]
 *   fm   (B, F k)     the FMB MLP's input; mlp (B, fmb D) its output, [b, j, d]
 *   flat (B, Fo D)    [b, f, d]: the last layer's output (out_layout 0), what the model's fc reads
 * Range: 1 <= F, Fo <= B2_WUKONG_MAX_FIELDS, 1 <= D <= B2_WUKONG_MAX_DIM, 1 <= k <= B2_WUKONG_MAX_RANK,
 * F k <= B2_WUKONG_MAX_FM_WIDTH, lcb, fmb >= 1, batch >= 0 (0: no launch) with every (B, row) tensor below 2^31
 * elements.  X' and a 16-byte aligned X with D % 4 == 0 stage through float4 loads, anything else through scalar
 * ones.  Outside the range, or given a NULL pointer, every entry point returns B2_E_INVALID.  An aux pointer (optional,
 * row pitch ld) receives the GEMM operand copy of the tensor written beside it: its bf16 rounding (aux_dtype B2_BF16)
 * or its 3xTF32 small part (B2_F32).
 * b2_wukong_fm_fwd:  fm "=" (+ fm_aux) from X (layout 0) or X' (layout 1); ln_mean, ln_rstd (B) "="; layout 0 may
 *   also write X'_0 "=" (xp_out, + xp_aux).
 * b2_wukong_fm_bwd:  from g = d fm, recomputing fm: gx "=" (accumulate 0) or "+=" in the input's layout (layout 0
 *   adds gxp, the gradient of X'_0, transposed); gY, dgamma, dbeta (F k) "+=" (caller zeroes): a per-CTA sum, then
 *   one float atomic per element and CTA.
 * b2_wukong_out_fwd: out "=" as X'_{i+1} (out_layout 1) or flat (out_layout 0) (+ out_aux); res_mode 1 reads the
 *   residual from X' (xp), 2 from C's projection columns; ln_mean, ln_rstd (B Fo) "=" with LayerNorm (gamma != NULL).
 * b2_wukong_out_bwd: from g in out's layout (g_layout): g_mlp (B, fmb D) "=", dC (B D, N) "=" (+ dc_aux); res_mode 1:
 *   gxp (B D, fp) "=" or "+=" (accumulate); res_mode 2: dbias (Fo) "+="; dgamma, dbeta (D) "+=" (caller zeroes).
 * b2_wukong_pack:    Ws "=" and, with W_res, bs "=".
 * b2_wukong_unpack:  gW_lcb (lcb, F) and, when gW_res != NULL, gW_res (Fo, F) "=" from dWs (N, fp).
 */
#define B2_WUKONG_MAX_FIELDS 128
#define B2_WUKONG_MAX_DIM 128
#define B2_WUKONG_MAX_RANK 32
#define B2_WUKONG_MAX_FM_WIDTH 1024
B2_API int b2_wukong_fm_fwd(const float* x, int layout, int64_t batch, int fields, int D, int k, const float* Y,
                            const float* gamma, const float* beta, float eps, float* fm_out, void* fm_aux,
                            int aux_dtype, int64_t ld_aux, float* xp_out, void* xp_aux, int64_t ld_xp_aux,
                            float* ln_mean, float* ln_rstd, void* stream);
B2_API int b2_wukong_fm_bwd(const float* x, int layout, int64_t batch, int fields, int D, int k, const float* Y,
                            const float* gamma, const float* ln_mean, const float* ln_rstd, const float* g,
                            const float* gxp, float* gx, int accumulate, float* gY, float* dgamma, float* dbeta,
                            void* stream);
B2_API int b2_wukong_out_fwd(const float* mlp_out, const float* C, const float* xp, int64_t batch, int fields, int D,
                             int lcb, int fmb, int res_mode, const float* gamma, const float* beta, float eps,
                             int out_layout, float* out, void* out_aux, int aux_dtype, int64_t ld_aux, float* ln_mean,
                             float* ln_rstd, void* stream);
B2_API int b2_wukong_out_bwd(const float* mlp_out, const float* C, const float* xp, int64_t batch, int fields, int D,
                             int lcb, int fmb, int res_mode, const float* gamma, const float* ln_mean,
                             const float* ln_rstd, int g_layout, const float* g, float* g_mlp, float* dC,
                             void* dc_aux, int aux_dtype, int64_t ld_aux, float* gxp, int accumulate, float* dbias,
                             float* dgamma, float* dbeta, void* stream);
B2_API int b2_wukong_pack(const float* W_lcb, const float* W_res, const float* b_res, int fields, int lcb,
                          int out_fields, float* Ws, float* bs, void* stream);
B2_API int b2_wukong_unpack(const float* dWs, int fields, int lcb, int out_fields, float* gW_lcb, float* gW_res,
                            void* stream);

/*
 * FinalNet (model_zoo/FinalNet/src/FinalNet.py).  One FactorizedInteraction layer of a FinalBlock on the caller's
 * GEMM output h = x W^T + b (B, 2 half), row-major fp32:
 *   h2 = h[:, :half], h1 = h[:, half:]
 *   z   = [h2, h1 h2] (residual B2_FINALNET_CONCAT, n = 2 half)  |  h2 + h1 h2 (B2_FINALNET_SUM, n = half)
 *   out = dropout(act(BatchNorm1d(z))) (B, n), each stage optional: gamma == NULL is no batch norm, act a B2_ACT_*
 *         code, drop_rng == NULL no dropout (the Philox mask of element (b, c) of out, as the MLP chain's).
 * Batch norm: eps, momentum as nn.BatchNorm1d; training normalises with the batch's biased variance, updates
 *   running_mean / running_var (unbiased variance) and num_batches (int64) in place, and refuses batch 1; eval
 *   normalises with the running statistics.  mean, rstd (n) "=" are what the backward reads.  stats_ws (fp64): 4 n
 *   doubles, the forward's column sums and, at stats_ws + 2 n, the backward's; a training forward clears all 4 n.
 * Range: 1 <= n <= B2_FINALNET_MAX_WIDTH, batch >= 0 (0: no launch), batch * 2 half < 2^31.  half % 4 == 0 with
 *   16-byte aligned rows runs the float4 path, anything else the scalar one.  Outside the range, or given a NULL
 *   pointer, every entry point returns B2_E_INVALID.  An aux pointer (optional, row pitch ld_aux) receives the GEMM
 *   operand copy of the tensor written beside it: its bf16 rounding (aux_dtype B2_BF16) or 3xTF32 small part (B2_F32).
 * b2_finalnet_fi_fwd: out "=" (+ out_aux); with batch norm in training a zero fill, a statistics pass and the apply
 *   pass, else the apply pass alone.
 * b2_finalnet_fi_bwd: from g = d out (B, n): dh (B, 2 half) "=" (+ dh_aux); dbias (2 half) "+=" (caller zeroes);
 *   with batch norm dgamma, dbeta (n) "=", from the sums at stats_ws (2 n doubles; zero_ws clears them first, which
 *   a training forward has already done).  training selects the batch-statistics backward.
 * FeatureGating (gate_residual "concat") of e (B, F, D) with W (F, F), bias (F):
 *   g = W e + bias over the field axis, out (B, 2 F D) = [e, e * g] flattened.
 *   Range: 1 <= F <= B2_FINALNET_MAX_FIELDS, 1 <= D <= B2_FINALNET_MAX_DIM, F D <= B2_FINALNET_MAX_GATE_WIDTH.
 * b2_finalnet_gate_fwd: out "=" (+ out_aux).
 * b2_finalnet_gate_bwd: from g = d out: de (B, F, D) "=" (accumulate 0) or "+="; dW, db "+=" (caller zeroes).
 * b2_finalnet_loss: the two-block loss of logits y1, y2 (B) and labels (B), batch >= 1, in one launch:
 *   y_pred = sigmoid((y1 + y2) / 2), loss "=" mean_b [BCE(y_pred, y) + BCE(sigmoid(y1), p) + BCE(sigmoid(y2), p)]
 *   with p = y_pred held constant; g1, g2 "=" d loss / d y1, y2.  Log terms clamped at -100 (b2_logit_bce_fwd).
 */
#define B2_FINALNET_CONCAT 0
#define B2_FINALNET_SUM 1
#define B2_FINALNET_MAX_WIDTH 1024
#define B2_FINALNET_MAX_FIELDS 128
#define B2_FINALNET_MAX_DIM 128
#define B2_FINALNET_MAX_GATE_WIDTH 8192
B2_API int b2_finalnet_fi_fwd(const float* h, int64_t batch, int half, int residual, const float* gamma,
                              const float* beta, float eps, float momentum, int training, float* running_mean,
                              float* running_var, int64_t* num_batches, double* stats_ws, int act,
                              const int64_t* drop_rng, int64_t drop_layer, uint32_t drop_thresh, float drop_scale,
                              float* out, void* out_aux, int aux_dtype, int64_t ld_aux, float* mean, float* rstd,
                              void* stream);
B2_API int b2_finalnet_fi_bwd(const float* h, int64_t batch, int half, int residual, const float* gamma,
                              const float* beta, const float* mean, const float* rstd, int training, double* stats_ws,
                              int zero_ws, int act, const int64_t* drop_rng, int64_t drop_layer, uint32_t drop_thresh,
                              float drop_scale, const float* g, float* dh, void* dh_aux, int aux_dtype, int64_t ld_aux,
                              float* dbias, float* dgamma, float* dbeta, void* stream);
B2_API int b2_finalnet_gate_fwd(const float* e, int64_t batch, int fields, int dim, const float* W, const float* bias,
                                float* out, void* out_aux, int aux_dtype, int64_t ld_aux, void* stream);
B2_API int b2_finalnet_gate_bwd(const float* e, int64_t batch, int fields, int dim, const float* W, const float* bias,
                                const float* g, float* de, int accumulate, float* dW, float* db, void* stream);
B2_API int b2_finalnet_loss(const float* y1, const float* y2, const float* label, int64_t batch, float* loss,
                            float* y_pred, float* g1, float* g2, void* stream);

/*
 * MultiHeadTargetAttention (layers/attentions/target_attention.py:95-172 with ScaledDotProductAttention,
 * dot_product_attention.py:32-58): one query, the target t (B, d), per sample over its history x (B, L, d).
 * With use_qkvo, W_q, W_k, W_v (A, d) and W_o (d, A), A = H*hd; W_?,h is head h's hd rows of W_q, W_k, W_v,
 * W_o,h head h's hd columns of W_o, and s = 1/sqrt(hd) (1 without use_scale).  The layer is linear in x but
 * for the softmax, so the projections fold into the query and output GEMMs and x is never projected:
 *   score_hl = q'_h . x_l,  q' = t W_M^T,  M_h = s W_q,h^T W_k,h (d x d)
 *   out = p W_N^T,  p_h = sum_l a_hl x_l,  N_h = W_v,h^T W_o,h^T (d x d)
 * All row-major fp32:
 *   W_M (H*d, d) K-major, the GEMM1 weight:  W_M[h*d + j, i] = M_h[i, j]
 *   W_N (d, H*d) K-major, the GEMM2 weight:  W_N[j, h*d + i] = N_h[i, j]
 *   q' (B, H*d), p (B, H*d): head h at columns h*d .. h*d + d - 1
 *   stats (B, H, 2): {m_h, l_h}, the softmax's max score and sum of exp(score - m_h) over the L positions.
 *     Not the log-sum-exp m_h + log l_h: with every position masked, m_h = -1e9 and fp32 spacing there (64)
 *     swallows log L.
 * Sliced form (use_qkvo False; no weights, no GEMMs): q = t, head h reads columns [h*hd, (h+1)*hd) of t and
 * x, score_hl = scale * q_h . x_l, and p (B, d) is the layer's output.
 * The row kernels take the per-head width `width` (d folded, hd sliced), `x_step`, head h's first column of
 * x (0 folded, hd sliced) and `scale` (1 folded: s is in W_M).  q and p have row pitch heads*width.
 * Masking: mask (B, L) bytes, 0 = masked, or NULL (no masking).  A masked score is exactly -1e9 after the
 * scale (masked_fill(mask == 0, -1e9)); the softmax runs over all L positions, so a row with every position
 * masked gets a_hl = 1/L: p is the mean of all L history rows and each of them receives dp_h / L.
 * Range: heads <= B2_MHTA_MAX_HEADS; heads*width <= B2_MHTA_MAX_WIDTH (one row's q', p, dp, dq' in one
 * warp's registers and shared memory); d <= B2_MHTA_MAX_WIDTH; batch*L within int32.  The pack and unpack
 * need heads*d <= B2_MHTA_MAX_WIDTH.  Outside the range every entry point returns B2_E_INVALID.
 * Saved for the backward: t, x, the mask, q', p, stats and the packed W_M, W_N of the forward; the backward
 * recomputes a_hl = exp(score_hl - m_h) / l_h and uses sum_l a_hl (dp_h . x_l) = dp_h . p_h, so it reads x
 * once and writes dx once:
 *   ds_hl = a_hl (dp_h . x_l - dp_h . p_h) (0 where masked),  dx_l = sum_h (a_hl dp_h + scale ds_hl q_h),
 *   dq_h = scale sum_l ds_hl x_l
 * (the sums over h and the columns of q_h, dp_h as they map onto x: all heads onto all d folded, head h onto
 * its own hd sliced).
 * b2_mhta_pack:   W_M, W_N "=" from W_q, W_k, W_v, W_o; one launch.
 * b2_mhta_fwd:    p, stats "=" from q, x, mask; p_aux (optional, row pitch ld_aux) receives p's GEMM operand
 *   copy: its bf16 rounding (aux_dtype B2_BF16) or its 3xTF32 small part (B2_F32).
 * b2_mhta_bwd:    dq "=" (+ dq_aux as above), dx (B, L, d) "=" from q, x, mask, p, stats and dp.
 * b2_mhta_unpack: gWq, gWk, gWv (A, d) and gWo (d, A) "=" from dW_M (H*d, d) and dW_N (d, H*d):
 *   gW_q,h = s W_k,h dM_h^T,  gW_k,h = s W_q,h dM_h,  gW_v,h = W_o,h^T dN_h^T,  gW_o,h = dN_h^T W_v,h^T.
 */
#define B2_MHTA_MAX_WIDTH 1024
#define B2_MHTA_MAX_HEADS 32
B2_API int b2_mhta_pack(const float* Wq, const float* Wk, const float* Wv, const float* Wo, int d, int heads,
                        int head_dim, float scale, float* WM, float* WN, void* stream);
B2_API int b2_mhta_fwd(const float* q, const float* x, const uint8_t* mask, int64_t batch, int L, int d, int heads,
                       int width, int x_step, float scale, float* p, float* stats, void* p_aux, int aux_dtype,
                       int64_t ld_aux, void* stream);
B2_API int b2_mhta_bwd(const float* q, const float* x, const uint8_t* mask, const float* p, const float* stats,
                       const float* dp, int64_t batch, int L, int d, int heads, int width, int x_step, float scale,
                       float* dq, float* dx, void* dq_aux, int aux_dtype, int64_t ld_aux, void* stream);
B2_API int b2_mhta_unpack(const float* Wq, const float* Wk, const float* Wv, const float* Wo, const float* dWM,
                          const float* dWN, int d, int heads, int head_dim, float scale, float* gWq, float* gWk,
                          float* gWv, float* gWo, void* stream);

/*
 * One CompressedInteractionNet layer (layers/interactions/compressed_interaction_net.py:70-73)
 * without the (B, F*H, D) Hadamard tensor:
 *   out[b,h',d] = bias[h'] + sum_{f,m} w[h', f*H + m] * x0[b,f,d] * xk[b,m,d]
 * x0 (B,F,D), xk (B,H,D), w (H', F*H) = Conv1d weight with kernel_size 1, out (B,H',D); H' <= 32.
 * b2_cin_bwd: g (B,H',D) -> gx0 (B,F,D) ("=" or "+=" with accumulate_x0), gxk (B,H,D) "=",
 * gw (H', F*H) "=" (H <= 64).  The bias gradient is the plain sum of g over (b,d).
 */
B2_API int b2_cin_fwd(const float* x0, const float* xk, const float* w, const float* bias, int64_t batch,
                      int F, int H, int HO, int D, float* out, void* stream);
B2_API int b2_cin_bwd(const float* x0, const float* xk, const float* w, const float* g, int64_t batch, int F,
                      int H, int HO, int D, float* gx0, int accumulate_x0, float* gxk, float* gw,
                      void* stream);

/*
 * Dice (layers/activations.py:37,49-50): p = sigmoid(BatchNorm1d(affine=False, eps, momentum)(x));
 * out = p*x + alpha*(1-p)*x on x (M, C).  training != 0: batch statistics over the M rows (and
 * running_mean/var updated in place like nn.BatchNorm1d, unbiased variance); else running stats.
 * mean/rstd (C) are outputs saved for the backward; stats_ws is a device workspace of 3*C doubles.
 * b2_dice_bwd: gx (M,C) "=", galpha (C) "=" (stats_ws is clobbered).
 */
B2_API int b2_dice_fwd(const float* x, const float* alpha, int64_t M, int C, float eps, float momentum,
                       int training, float* running_mean, float* running_var, float* mean, float* rstd,
                       double* stats_ws, float* out, void* stream);
B2_API int b2_dice_bwd(const float* x, const float* gout, const float* alpha, const float* mean,
                       const float* rstd, int64_t M, int C, int training, double* stats_ws, float* gx,
                       float* galpha, void* stream);
/*
 * DIN_Attention glue (layers/attentions/target_attention.py:79-92).
 * b2_din_input_fwd: out ((B*L), 4d) = [t, h, t-h, t*h] with t = target (B,d) broadcast over L, h = hist (B,L,d).
 * b2_din_input_bwd: from gin ((B*L),4d): gtarget (B,d) "=", ghist (B,L,d) "=" or "+=" (accumulate_hist).
 * b2_din_wsum_fwd:  out (B,d) = sum_l w[b,l]*mask[b,l]*hist[b,l,:]  (mask uint8 or NULL)   (:85-86,91)
 * b2_din_wsum_bwd:  gw (B,L) = mask * <gout[b], hist[b,l]>;  ghist (B,L,d) = w*mask*gout[b].
 */
B2_API int b2_din_input_fwd(const float* target, const float* hist, int64_t B, int L, int d, float* out,
                            void* stream);
B2_API int b2_din_input_bwd(const float* target, const float* hist, const float* gin, int64_t B, int L, int d,
                            float* gtarget, float* ghist, int accumulate_hist, void* stream);
B2_API int b2_din_wsum_fwd(const float* w, const unsigned char* mask, const float* hist, int64_t B, int L,
                           int d, float* out, void* stream);
B2_API int b2_din_wsum_bwd(const float* w, const unsigned char* mask, const float* hist, const float* gout,
                           int64_t B, int L, int d, float* gw, float* ghist, void* stream);
/* use_softmax = True branch of DIN_Attention (target_attention.py:85-90), one launch each way:
 *   p = softmax_L( w * mask + (-1e9) * (1 - mask) )   (mask (B,L) uint8 or NULL)
 *   bwd: gw = p * (g - sum_l g p) * mask */
B2_API int b2_din_softmax_fwd(const float* w, const unsigned char* mask, int64_t B, int L, float* p, void* stream);
B2_API int b2_din_softmax_bwd(const float* p, const float* g, const unsigned char* mask, int64_t B, int L,
                              float* gw, void* stream);

/*
 * Dense layer with fused epilogue; the GEMM behind MLP_Block
 * (layers/blocks/mlp_block.py:74-85,96), CrossNetV2 (cross_net.py:126-129) and
 * the 1x1 Conv1d of CIN (compressed_interaction_net.py:72).
 *   C[m,n] = epi( sum_k A(m,k) * B(k,n) + bias[n] )
 * A element (m,k) at a[m*a_rs + k*a_cs]; B element (k,n) at b[k*b_rs + n*b_cs];
 * C row-major with leading dimension ldc.
 *   act     B2_ACT_*
 *   mul,add optional (M,N) row-major (ld = ldc): C = add + mul * (acc + bias)
 *           (CrossNetV2: mul = x_0, add = x_i).  NULL = absent.
 *   beta_accumulate != 0: C += result (used for gradient accumulation).
 * math: B2_F32 = fp32 FMA (parity path); B2_BF16 = operands rounded to bf16,
 * fp32 accumulate, on wgmma tensor cores when shapes allow.
 */
B2_API int b2_gemm_f32(const float* a, int64_t a_rs, int64_t a_cs, const float* b, int64_t b_rs,
                int64_t b_cs, float* c, int64_t ldc, int64_t M, int64_t N, int64_t K,
                const float* bias, int act, const float* mul, const float* add,
                int beta_accumulate, void* stream);

/*
 * The tensor-core contraction:  C[m,n] = epi( sum_k A(m,k) * B(n,k) ), computed by a TMA-fed wgmma
 * kernel with the accumulators in registers.
 * Operand layouts (TMA loads either as it lies and the kernel re-lays it out in shared memory, so
 * no transpose pass in global memory is ever needed):
 *   a_mn_major == 0:  A in memory (M, K), k contiguous, leading dimension lda   ("K-major")
 *   a_mn_major != 0:  A in memory (K, M), m contiguous, leading dimension lda   ("MN-major")
 *   likewise b_mn_major for B: (N, K) or (K, N).
 * This covers the three contractions of nn.Linear (mlp_block.py:74, autograd of F.linear) on the
 * tensors as they lie in memory:  Y = X W^T (both K-major);  dX = dZ W (B = W MN-major);
 * dW = dZ^T X (A = dZ and B = X MN-major).
 * Epilogue, in this order:  v = acc + bias[n];  c_pre = v (optional: CrossNetV2 keeps W x_i + b for its
 * backward);  v = add + mul * v;  v = act(v);
 *   v = act_bwd'(ybwd[m,n]) * v   (ybwd = the activation OUTPUT whose backward is fused: the dgrad
 *                                  GEMM of layer i+1 emits dZ_i directly; threshold_backward /
 *                                  sigmoid_backward of the reference's autograd);
 *   C = v (+ C if beta_accumulate);  c_small = v - tf32_trunc(v) (the consumer's 3xTF32 operand);
 *   colsum[n] = sum_m v  (bias gradient; the call zeroes colsum first).
 * mul, add, ybwd, c_small share C's leading dimension.
 * fp32 operands: a_small == b_small == NULL is single-pass TF32 (operand mantissas truncated to 10 bits);
 * both non-NULL is error-compensated 3xTF32 (fp32-class accuracy).  The pointers act as a mode flag: their
 * contents are NOT read (the kernel derives the small parts of A and B itself); only their TMA alignment is
 * checked.  B2_GEMM_X3_INLINE selects 3xTF32 without them.
 * Operands must be TMA-addressable (16-byte aligned base, 16-byte row pitch); otherwise B2_E_UNSUPPORTED
 * is returned and the caller uses b2_gemm_f32.
 * elem_dtype == B2_BF16 (BASELINE configs[1] "bf16"): a and b hold bf16 (row pitch a multiple of 16
 * bytes, i.e. leading dimensions % 8 == 0), one pass of wgmma .bf16 with fp32 accumulation;
 * C stays fp32 and c_small, if given, receives C rounded to bf16 (leading dimension ld_aux) — the
 * next contraction's operand.  b2_to_bf16 makes that operand for tensors no epilogue produced.
 */
typedef struct b2_gemm_desc {
  const void* a;          /* fp32, or bf16 when elem_dtype == B2_BF16 */
  const void* b;
  const float* a_small;
  const float* b_small;
  float* c;
  void* c_small;          /* fp32 small part of C; bf16 copy of C when elem_dtype == B2_BF16 */
  float* c_pre;
  const float* bias;
  const float* mul;
  const float* add;
  const float* ybwd;
  float* colsum;
  int64_t lda, ldb, ldc;
  int64_t M, N, K;
  int32_t a_mn_major, b_mn_major;
  int32_t act, act_bwd;
  int32_t beta_accumulate;
  int32_t elem_dtype;     /* B2_F32 (wgmma .tf32 passes on fp32) or B2_BF16 (wgmma .bf16, fp32 accumulation) */
  int64_t ld_aux;         /* leading dimension of c_small (0 = ldc) */
  int64_t flags;          /* B2_GEMM_*: the caller vouches an output is already all-zero (skips its memset) */
  /* Dropout (see "Dropout masks" below); drop_rng == NULL (a zeroed descriptor): no mask.  The mask of the
   * (M, N) output is applied after act and before act_bwd:  v = act(v) * keep * drop_scale  in a forward,
   * v = act_bwd'(ybwd) * keep * drop_scale * v  in a dgrad that folds a dropout layer's backward (ybwd is then
   * that layer's DROPPED output; sigmoid's s is recovered as ybwd / drop_scale).  c_small and colsum see the
   * masked value.  A launch with a mask is never split over K. */
  const int64_t* drop_rng; /* device {seed, offset} snapshot of the forward (b2_dropout_rng_take) */
  int64_t drop_layer;     /* the mask's counter offset: snapshot offset + drop_layer */
  uint32_t drop_thresh;   /* keep iff the element's Philox word < drop_thresh */
  float drop_scale;       /* 1 / (1 - p) */
} b2_gemm_desc;
#define B2_GEMM_C_IS_ZERO 1      /* split-K accumulates into C with red.global: C needs no clearing */
#define B2_GEMM_COLSUM_IS_ZERO 2
#define B2_GEMM_X3_INLINE 4      /* 3xTF32 from the fp32 operands alone: the small parts are made in shared memory */
#define B2_GEMM_BACKFILL 8       /* runs beside a chain of launches on another stream (a wgrad next to the dgrads): a
                                    linear epilogue is split over K into short CTAs (b2_gemm_plan.splits reports it) */
B2_API int b2_gemm_tc_ex(const b2_gemm_desc* desc, void* stream);
/* The launch plan b2_gemm_tc_ex would use for `desc` (pure host arithmetic: no device call, no stream): lets a
   host-only test check that every plan fits the SM (<= 227 KB of shared memory).  stages: k-blocks in flight in
   the operand ring; cstages: the same ring (loaded and converted tiles share a stage); grid: one CTA per tile
   and K split. */
typedef struct b2_gemm_plan {
  int32_t bn, splits, stages, cstages, grid, threads, tiles_m, tiles_n, passes, kb_per_split;
  int64_t smem_bytes;
} b2_gemm_plan;
B2_API int b2_gemm_tc_plan(const b2_gemm_desc* desc, b2_gemm_plan* plan);
B2_API int b2_to_bf16(const float* x, int64_t rows, int64_t cols, int64_t ld_in, void* out, int64_t ld_out,
                      void* stream);
/* small[i] = x[i] - (x[i] with the 13 low mantissa bits cleared). */
B2_API int b2_split_tf32(const float* x, float* small, int64_t n, void* stream);

/*
 * One-pass operand preparation for the K-major tensor-core GEMMs over x (R, C):
 *   v = act'(y) * x when y != NULL (y = activation OUTPUT; fuses the activation backward);
 *   act == B2_PREP_MUL: v = x * y
 *   out (R,C) = v, out_small = 3xTF32 small part, outT (C,R) = v^T, outT_small, colsum[c] = sum_r v[r,c]
 * Every output may be NULL, but outT_small needs outT.  One pass where an activation backward, a transpose,
 * a 3xTF32 split and a column sum would each read x again.
 * drop_rng != NULL: x is the gradient of a dropout layer's output and y (if any) that DROPPED output:
 *   v = act'(y) * keep * drop_scale * x  with the mask of (R, C) at counter offset snapshot offset + drop_layer
 *   (not with B2_PREP_MUL).  drop_rng == NULL: no mask, the other drop arguments are ignored.
 */
B2_API int b2_prep_operand(const float* x, const float* y, int act, int64_t R, int64_t C, float* out,
                           float* out_small, float* outT, float* outT_small, float* colsum,
                           const int64_t* drop_rng, int64_t drop_layer, uint32_t drop_thresh, float drop_scale,
                           void* stream);
/*
 * The N = 1 output head of MLP_Block (Linear(K, 1), mlp_block.py:82): warp-per-row GEMV forward,
 * y[m] = act(<x[m,:], w> + b); and one fused backward: gz = act'(y)*gy, gx[m,:] = gz[m]*w (gx may
 * be NULL), gw (K) = sum_m gz[m]*x[m,:], gb (1) = sum_m gz[m]  ("=" semantics).
 * The backward takes K <= B2_HEAD_MAX_K: it stages 2 * K floats of partial sums in shared memory, and
 * 2 * 28672 * 4 B = 224 KB, with the kernel's static part, stays within the 227 KB per block of sm_90.
 * A wider Linear(K, 1) runs as a general GEMM.
 */
#define B2_HEAD_MAX_K 28672
B2_API int b2_head_fwd(const float* x, const float* w, const float* b, int64_t M, int K, int act, float* y,
                       void* stream);
B2_API int b2_head_bwd(const float* x, const float* w, const float* y, const float* gy, int64_t M, int K,
                       int act, float* gx, float* gw, float* gb, void* stream);
/* Same, fused with the activation backward of the layer that PRODUCED x (x is that layer's
 * activation output, mlp_block.py:78-80): gx <- prev_act'(x) * gx, gx_small = its 3xTF32 small part
 * (or NULL), gb_prev (K) = sum_m gx[m,:] = that layer's bias gradient (or NULL).  grads_zeroed != 0: the
 * caller vouches gw, gb and gb_prev are already all-zero (a gradient arena cleared by the optimizer pass).
 * prev_drop_rng != NULL: that layer ends on dropout and x is its dropped output; its (M, K) mask multiplies gx
 * before prev_act' (gx <- prev_act'(x) * keep * prev_drop_scale * gx), as in b2_gemm_desc. */
B2_API int b2_head_bwd_ex(const float* x, const float* w, const float* y, const float* gy, int64_t M, int K,
                          int act, float* gx, float* gw, float* gb, int prev_act, float* gx_small,
                          float* gb_prev, int grads_zeroed, const int64_t* prev_drop_rng, int64_t prev_drop_layer,
                          uint32_t prev_drop_thresh, float prev_drop_scale, void* stream);

/*
 * Dropout masks (nn.Dropout of MLP_Block, mlp_block.py:80: y = x * keep / (1 - p), keep ~ Bernoulli(1 - p)).
 * The mask is a pure function of a device {seed, offset} pair (int64 each) and the element:
 *   i = m * N + n  (the element of the (M, N) layer output, 64-bit);  off = snapshot offset + layer;
 *   r = Philox4x32-10(counter = {lo32(i >> 2), hi32(i >> 2), lo32(off), hi32(off)}, key = {lo32(seed), hi32(seed)});
 *   keep  <=>  r[i & 3] < thresh,  thresh = min(round((1 - p) * 2^32), 2^32 - 1);  scale = fp32(1 / (1 - p)).
 * A kept element is x * scale (one fp32 multiply), a dropped one is 0.
 * b2_dropout_rng_take: snapshot = state, then state.offset += n_layers (one single-thread launch per forward of
 *   a chain with n_layers dropout layers, which use offsets snapshot.offset + 0 .. n_layers - 1): no two
 *   (forward, layer, element group) share a counter, and a CUDA graph replay draws fresh masks.
 * b2_dropout_apply: y = keep ? x * scale : 0 over (M, N) with leading dimension ld (x and y; y may be x).
 */
B2_API int b2_dropout_rng_take(int64_t* state, int64_t* snapshot, int n_layers, void* stream);
B2_API int b2_dropout_apply(const float* x, float* y, int64_t M, int64_t N, int64_t ld, const int64_t* snapshot,
                            int64_t layer, uint32_t thresh, float scale, void* stream);

/*
 * Final glue of DeepFM.forward + BaseModel.add_loss (model_zoo/DeepFM/DeepFM_torch/
 * src/DeepFM.py:84-86, fuxictr/pytorch/models/rank_model.py:120-131):
 *   logit = sum of nterms per-sample terms; y_pred = sigmoid(logit);
 *   loss  = mean_b BCE(y_pred, y) with torch's log clamp at -100.
 * terms: device array... passed as up to 4 pointers (NULL = absent).
 * Outputs: y_pred (B), loss (1, "=" semantics via two-stage reduction in ws),
 * glogit (B) = (y_pred - y) / B  (NULL to skip).
 */
B2_API int b2_logit_bce_fwd(const float* t0, const float* t1, const float* t2, const float* t3,
                     const float* label, int64_t batch, float* y_pred, float* loss,
                     float* glogit, void* stream);

/*
 * Dense optimizer step over a flat fp32 arena, semantics of
 * nn.utils.clip_grad_norm_(params, max_norm) followed by torch.optim.Adam
 * (defaults betas=(0.9,0.999), eps=1e-8, weight_decay=0, amsgrad=False) as
 * called by BaseModel.train_step (rank_model.py:321-322).
 *   b2_sumsq: out[0] += sum g^2 over n elements (caller zeroes out).
 *   b2_adam_step: clip_coef = min(1, max_norm / (sqrt(sumsq[0]) + 1e-6));
 *                 g' = g*clip_coef; m = b1*m + (1-b1)*g'; v = b2*v + (1-b2)*g'^2;
 *                 p -= (lr/bc1) * m / (sqrt(v)/sqrt(bc2) + eps), with
 *                 bc1 = 1-b1^step, bc2 = 1-b2^step, step read from step_dev[0]
 *                 (device int64, already incremented by the caller).
 *   If zero_grad != 0 the gradient arena is zeroed in the same pass.
 *   b2_adam_sched writes sched[step] = {lr/(1-b1^step), 1/sqrt(1-b2^step)}; b2_adam_step_sched is
 *   b2_adam_step reading those two scalars from the table (shared with the lazy row-wise kernels).
 * Constants, as torch forms them from Python floats: every Adam entry point (and b2_lazy_adam_step,
 * b2_lazy_materialize) takes lr, beta1 and beta2 as double; 1-b1, b2 and 1-b2 are computed in double and
 * rounded to fp32 once, bc1 and bc2 come from pow of the double betas, and the step size is fl32(lr/bc1).
 * eps and max_norm are fp32, as torch applies them.
 * A NaN norm (a NaN gradient) is where these kernels leave torch: torch's clip coefficient is then NaN and
 * every parameter becomes NaN, here fminf(NaN, 1) = 1 and the step runs unclipped.  b2_adam_untouched runs
 * before the norm exists, so no pass could follow torch there.  An infinite norm gives clip_coef = 0, as in
 * torch.
 */
B2_API int b2_sumsq(const float* g, int64_t n, float* out, void* stream);
B2_API int b2_adam_step(float* p, float* g, float* m, float* v, int64_t n, const float* sumsq,
                 float max_norm, double lr, double beta1, double beta2, float eps,
                 const int64_t* step_dev, int zero_grad, void* stream);
/* The same two passes reading G only where a batch wrote it: flags[k] (b2_touch) covers elements
 * [16k, 16k + 16) of the first n_flagged elements (n_flagged % 4 == 0, <= n); the elements after
 * n_flagged have no flags and run as above.  An unflagged granule holds only zeros: b2_sumsq_ex skips
 * it (each thread keeps its elements, so the block partials equal b2_sumsq's), b2_adam_step_ex applies
 * g = 0 without loading or storing G.  A flagged granule is updated as b2_adam_step does, and with
 * zero_grad != 0 its flag is cleared together with its gradient.  flags == NULL is the plain form. */
B2_API int b2_sumsq_ex(const float* g, int64_t n, float* out, const uint8_t* flags, int64_t n_flagged,
                       void* stream);
B2_API int b2_adam_step_ex(float* p, float* g, float* m, float* v, int64_t n, const float* sumsq,
                           float max_norm, double lr, double beta1, double beta2, float eps,
                           const int64_t* step_dev, int zero_grad, uint8_t* flags, int64_t n_flagged,
                           void* stream);
/* The table pass of b2_adam_step_ex (zero_grad = 1, n_flagged = n) split in two launches, for a step whose
 * flags are final before its gradients exist (every granule the backward will write is flagged first):
 *   b2_adam_untouched  every UNFLAGGED granule gets the g = 0 update of step *step_dev + 1 (the optimizer
 *                      counts the step later); P, M, V only, never G or the flags.  At most max_ctas CTAs of
 *                      1024 threads (one per SM), persistent: it is meant to run beside the forward and backward.
 *   b2_adam_touched    every FLAGGED granule is updated as b2_adam_step_ex does (step *step_dev), its gradient
 *                      zeroed and its flag cleared; an unflagged granule costs one flag read.
 * Together they leave P, M, V, G and the flags bit-identical to b2_adam_step_ex.  n % 4 == 0. */
B2_API int b2_adam_untouched(float* p, float* m, float* v, int64_t n, const uint8_t* flags, double lr, double beta1,
                             double beta2, float eps, const int64_t* step_dev, int max_ctas, void* stream);
B2_API int b2_adam_touched(float* p, float* g, float* m, float* v, int64_t n, const float* sumsq, float max_norm,
                           double lr, double beta1, double beta2, float eps, const int64_t* step_dev, uint8_t* flags,
                           void* stream);
B2_API int b2_adam_sched(const int64_t* step_dev, double lr, double beta1, double beta2, float* sched,
                         int64_t sched_len, void* stream);
B2_API int b2_adam_step_sched(float* p, float* g, float* m, float* v, int64_t n, const float* sumsq,
                              float max_norm, double beta1, double beta2, float eps, const int64_t* step_dev,
                              const float* sched, int zero_grad, void* stream);

/*
 * Device-resident evaluation (SURVEY.md 8f row 3).  BaseModel.evaluate
 * (fuxictr/pytorch/models/rank_model.py:350-381) moves y_pred / y_true to the host after every
 * batch and calls sklearn's log_loss / roc_auc_score on float64 copies (fuxictr/metrics.py:45-48);
 * these entry points compute the same two numbers from fp32 device arrays of the whole split.
 *   b2_logloss_sum: sum[0] += sum_i -[y_i log(clip(p_i)) + (1-y_i) log(clip(1-p_i))], fp64,
 *                   clip to [eps, 1-eps] with eps = DBL_EPSILON (sklearn clips the widened float64
 *                   array); the caller zeroes sum and divides by n.
 *   b2_auc: result (device, 5 x u64, zeroed inside) = {n_neg, n_pos, n_nan, n_badlabel, 2U} with
 *           U = #(neg < pos) + 0.5 #(neg == pos) over all (pos, neg) pairs, exact in integers;
 *           AUC = 2U / (2 n_pos n_neg).  Labels must be exactly 0 or 1 (others are counted in
 *           n_badlabel and skipped; sklearn raises); NaN scores are counted in n_nan (sklearn
 *           raises).  workspace: b2_auc_workspace_bytes(n) bytes, 256-byte aligned.
 *   b2_sort_u32: ascending stable LSD radix sort (the building block of b2_auc), same workspace.
 */
B2_API int b2_logloss_sum(const float* y_pred, const float* y_true, int64_t n, double* sum, void* stream);
B2_API int b2_auc_workspace_bytes(int64_t n, int64_t* bytes);
B2_API int b2_auc(const float* y_pred, const float* y_true, int64_t n, void* workspace, int64_t workspace_bytes,
                  uint64_t* result, void* stream);
B2_API int b2_sort_u32(uint32_t* keys, int64_t n, void* workspace, int64_t workspace_bytes, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* FUXICTR_B200_H_ */

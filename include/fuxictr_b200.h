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
 */
B2_API int b2_embed_gather_fwd(const b2_field* fields, int nfields, int64_t batch, int idx_dtype,
                        int elem_dtype, float* mean_count, int32_t* status, void* stream);
/* Same, with the first `hot_rows` rows of every table staged once per CTA in shared memory and served
 * from there (north_star "shared-memory staging of hot rows"): FuxiCTR's tokenizer numbers ids by
 * descending frequency, so the small ids are the hot ones.  Applies when every field is one slot of one
 * common dim (% 4) and the staging area fits 44 KB per CTA; otherwise identical to b2_embed_gather_fwd.
 * The result is bit-identical either way. */
B2_API int b2_embed_gather_hot_fwd(const b2_field* fields, int nfields, int64_t batch, int idx_dtype,
                                   int elem_dtype, float* mean_count, int32_t* status, int hot_rows,
                                   void* stream);

/*
 * Backward of the fused gather: dense-gradient scatter-add with warp-level
 * aggregation of duplicate rows.  Replaces F x aten::embedding_dense_backward
 * (autograd of feature_embedding.py:285,288).  In each descriptor `table` is the
 * (vocab, dim) f32 GRADIENT buffer (accumulated into: the caller zeroes it when it
 * wants "=" semantics), `out` is the incoming gradient laid out exactly like the
 * forward output; rows whose index equals padding_idx receive no gradient
 * (nn.Embedding(padding_idx)).  mean_count is the buffer the forward filled
 * (NULL when no field uses B2_POOL_MEAN).
 */
B2_API int b2_embed_scatter_bwd(const b2_field* fields, int nfields, int64_t batch, int idx_dtype,
                         int elem_dtype, const float* mean_count, void* stream);

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
 * gbias[0] += sum_b gout[b]. `table` fields point at the (vocab,1) gradient buffers. */
B2_API int b2_lr_bwd(const b2_field* fields, int nfields, int64_t batch, int idx_dtype,
              const float* gout, float* gbias, void* stream);


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
 */
typedef struct b2_lazy_ctx {
  const int32_t* last_step; /* [total rows] optimizer step each row is current for */
  const float* sched;       /* float2[sched_len]: {lr/(1-b1^t), 1/sqrt(1-b2^t)} per step t */
  const int64_t* step_dev;  /* device scalar: optimizer steps completed so far */
  int32_t* mark;            /* [total rows] scratch: step at which the row was last enqueued */
  int32_t* worklist;        /* [capacity] global row ids touched this step */
  int32_t* counter;         /* device scalar: worklist length */
  int64_t delta_m, delta_v; /* element offsets from a parameter to its Adam moments (arena layout) */
  float w1, beta2, w2, eps; /* 1-beta1, beta2, 1-beta2, eps */
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
 */
B2_API int b2_front_bwd(const b2_field* emb_fields, const b2_field* lr_fields, int nfields, int64_t batch,
                        int idx_dtype, int want_fm, const float* emb_saved, const float* gx,
                        const float* sums, const float* glogit, float* gbias,
                        const b2_lazy_ctx* lazy /* non-NULL: enqueue every touched row once */, void* stream);
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
                             const int64_t* step_dev, const float* sumsq, float max_norm, float beta1,
                             float beta2, float eps, void* stream);
B2_API int b2_lazy_materialize(const b2_lazy_table* tables_dev, int ntables, int64_t total_rows,
                               int64_t delta_m, int64_t delta_v, int32_t* last_step, const float* sched,
                               const int64_t* step_dev, float beta1, float beta2, float eps, void* stream);

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
 * b2_peer_bcast: one launch copies `nbytes` (multiple of 4, 16-byte aligned buffers) from src into
 * peer_dst[p] for every p < world (P2P stores): the batch-matrix exchange.
 */
B2_API int b2_shard_push(const b2_field* emb_fields, const b2_field* lr_fields, int nfields,
                         int64_t batch_local, int world, int rank, const void* const* peer_ids,
                         int idx_dtype, int64_t ids_stride, float* const* peer_emb,
                         float* const* peer_lrw, int32_t* status, int32_t* owned, int32_t* owned_count,
                         int32_t owned_capacity, void* stream);
B2_API int b2_shard_pull(const b2_field* emb_fields, const b2_field* lr_fields, int nfields,
                         int64_t batch_local, int world, int rank, const float* const* peer_gemb,
                         const float* const* peer_glogit, float scale, const int32_t* owned,
                         const int32_t* owned_count, int32_t owned_capacity, void* stream);
B2_API int b2_peer_bcast(const void* src, int64_t nbytes, void* const* peer_dst, int world, void* stream);
/* The id exchange, compressed: `count` contiguous ids of dtype idx_dtype (B2_F64 truncates like .long())
 * are narrowed to int32 and stored into peer_dst[p] (16-byte aligned) for every p < world. */
B2_API int b2_peer_bcast_ids(const void* src, int idx_dtype, int64_t count, int32_t* const* peer_dst, int world,
                             void* stream);
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
 * Tensor-core dense layer: same contract as b2_gemm_f32 for the K-major case
 *   C[m,n] = epi( sum_k A[m,k] * B[n,k] + bias[n] ),  A (M,K) ld=lda, B (N,K) ld=ldb, fp32,
 * computed by a TMA-fed wgmma .tf32 kernel with the accumulators in registers.
 *   a_small == b_small == NULL : single-pass TF32 (operand mantissas truncated to 10 bits).
 *   a_small, b_small given      : error-compensated 3xTF32 (fp32-class accuracy).  The pointers act as a
 *                                 mode flag: their contents are NOT read (the kernel derives the small
 *                                 parts of A and B itself); only their TMA alignment is checked.
 * Operands must be TMA-addressable (16-byte aligned base, ld % 4 == 0): b2_gemm_tc_supported()
 * says whether they are; otherwise B2_E_UNSUPPORTED is returned and the caller uses b2_gemm_f32.
 */
B2_API int b2_gemm_tc_supported(const float* a, int64_t lda, const float* b, int64_t ldb, int64_t M,
                                int64_t N, int64_t K);
B2_API int b2_gemm_tc(const float* a, int64_t lda, const float* b, int64_t ldb, float* c, int64_t ldc,
                      int64_t M, int64_t N, int64_t K, const float* bias, int act, const float* mul,
                      const float* add, int beta_accumulate, const float* a_small,
                      const float* b_small, void* stream);

/*
 * The general tensor-core contraction:  C[m,n] = epi( sum_k A(m,k) * B(n,k) ).
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
 * mul, add, ybwd, c_small share C's leading dimension.  a_small/b_small: both non-NULL selects 3xTF32
 * (contents not read, see b2_gemm_tc; B2_GEMM_X3_INLINE selects it without them), both NULL single-pass TF32.
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
} b2_gemm_desc;
#define B2_GEMM_C_IS_ZERO 1      /* split-K accumulates into C with red.global: C needs no clearing */
#define B2_GEMM_COLSUM_IS_ZERO 2
#define B2_GEMM_X3_INLINE 4      /* 3xTF32 from the fp32 operands alone: the small parts are made in shared memory */
B2_API int b2_gemm_tc_ex(const b2_gemm_desc* desc, void* stream);
/* The launch plan b2_gemm_tc_ex would use for `desc` (pure host arithmetic: no device call, no stream): lets a
   host-only test check that every plan fits the SM (<= 227 KB of shared memory).  stages: raw TMA tiles in
   flight; cstages: converted (swizzled, split) tiles in flight; grid: one CTA per tile and K split. */
typedef struct b2_gemm_plan {
  int32_t bn, splits, stages, cstages, grid, threads, tiles_m, tiles_n, passes, kb_per_split;
  int64_t smem_bytes;
} b2_gemm_plan;
B2_API int b2_gemm_tc_plan(const b2_gemm_desc* desc, b2_gemm_plan* plan);
B2_API int b2_to_bf16(const float* x, int64_t rows, int64_t cols, int64_t ld_in, void* out, int64_t ld_out,
                      void* stream);
/* small[i] = x[i] - (x[i] with the 13 low mantissa bits cleared). */
B2_API int b2_split_tf32(const float* x, float* small, int64_t n, void* stream);
/* out (cols, rows; ld_out) = in (rows, cols; ld_in)^T; if out_small != NULL it also receives the
 * 3xTF32 small part of the transposed values. */
B2_API int b2_transpose_f32(const float* in, int64_t rows, int64_t cols, int64_t ld_in, float* out,
                            int64_t ld_out, float* out_small, void* stream);

/*
 * One-pass operand preparation for the K-major tensor-core GEMMs over x (R, C):
 *   v = act'(y) * x when y != NULL (y = activation OUTPUT; fuses the activation backward);
 *   act == B2_PREP_MUL: v = x * y
 *   out (R,C) = v, out_small = 3xTF32 small part, outT (C,R) = v^T, outT_small, colsum[c] = sum_r v[r,c]
 * Every output may be NULL.  Replaces b2_act_bwd + b2_transpose_f32 + b2_split_tf32 + b2_colsum.
 */
B2_API int b2_prep_operand(const float* x, const float* y, int act, int64_t R, int64_t C, float* out,
                           float* out_small, float* outT, float* outT_small, float* colsum, void* stream);
/*
 * The N = 1 output head of MLP_Block (Linear(K, 1), mlp_block.py:82): warp-per-row GEMV forward,
 * y[m] = act(<x[m,:], w> + b); and one fused backward: gz = act'(y)*gy, gx[m,:] = gz[m]*w (gx may
 * be NULL), gw (K) = sum_m gz[m]*x[m,:], gb (1) = sum_m gz[m]  ("=" semantics).
 */
B2_API int b2_head_fwd(const float* x, const float* w, const float* b, int64_t M, int K, int act, float* y,
                       void* stream);
B2_API int b2_head_bwd(const float* x, const float* w, const float* y, const float* gy, int64_t M, int K,
                       int act, float* gx, float* gw, float* gb, void* stream);
/* Same, fused with the activation backward of the layer that PRODUCED x (x is that layer's
 * activation output, mlp_block.py:78-80): gx <- prev_act'(x) * gx, gx_small = its 3xTF32 small part
 * (or NULL), gb_prev (K) = sum_m gx[m,:] = that layer's bias gradient (or NULL).  grads_zeroed != 0: the
 * caller vouches gw, gb and gb_prev are already all-zero (a gradient arena cleared by the optimizer pass). */
B2_API int b2_head_bwd_ex(const float* x, const float* w, const float* y, const float* gy, int64_t M, int K,
                          int act, float* gx, float* gw, float* gb, int prev_act, float* gx_small,
                          float* gb_prev, int grads_zeroed, void* stream);
/* Elementwise helpers used by the dense backward.
 * b2_act_bwd: gx = gy * act'(y) where y is the activation OUTPUT (relu, sigmoid). */
B2_API int b2_act_bwd(const float* y, const float* gy, float* gx, int64_t n, int act, void* stream);
/* b2_colsum: out[n] (+)= sum_m x[m*ld + n]  (bias gradients). */
B2_API int b2_colsum(const float* x, int64_t M, int64_t N, int64_t ld, float* out, int accumulate,
              void* stream);

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
 */
B2_API int b2_sumsq(const float* g, int64_t n, float* out, void* stream);
B2_API int b2_adam_step(float* p, float* g, float* m, float* v, int64_t n, const float* sumsq,
                 float max_norm, float lr, float beta1, float beta2, float eps,
                 const int64_t* step_dev, int zero_grad, void* stream);
B2_API int b2_adam_sched(const int64_t* step_dev, float lr, float beta1, float beta2, float* sched,
                         int64_t sched_len, void* stream);
B2_API int b2_adam_step_sched(float* p, float* g, float* m, float* v, int64_t n, const float* sumsq,
                              float max_norm, float beta1, float beta2, float eps, const int64_t* step_dev,
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

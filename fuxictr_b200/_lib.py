"""ctypes binding of libfuxictr_b200.so (the C-ABI declared in include/fuxictr_b200.h).

This is the *only* place Python touches the native library.  Arguments are raw device
pointers (``tensor.data_ptr()``), sizes and the caller's CUDA stream handle; no torch
type crosses the boundary.  A missing library is a hard error: there is no CPU or eager
fallback behind these calls.
"""
import ctypes
import os

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libfuxictr_b200.so")

# dtype / mode codes (mirror include/fuxictr_b200.h)
B2_F32, B2_BF16, B2_F64, B2_I64, B2_I32 = 0, 1, 2, 3, 4
B2_POOL_NONE, B2_POOL_SUM, B2_POOL_MEAN = 0, 1, 2
B2_ACT_NONE, B2_ACT_RELU, B2_ACT_SIGMOID = 0, 1, 2
B2_ACT_LEAKY_RELU = 4
B2_PREP_MUL = 3
B2_GEMM_C_IS_ZERO, B2_GEMM_COLSUM_IS_ZERO, B2_GEMM_X3_INLINE, B2_GEMM_BACKFILL = 1, 2, 4, 8
B2_MAX_FIELDS = 128
B2_CROSSMIX_MAX_RANK, B2_CROSSMIX_MAX_COLS = 64, 256
B2_MHTA_MAX_WIDTH, B2_MHTA_MAX_HEADS = 1024, 32
B2_HEAD_MAX_K = 28672
B2_MASKNET_MAX_WIDTH = 1024
B2_AUTOINT_MAX_FIELDS, B2_AUTOINT_MAX_DIM = 64, 64
B2_WUKONG_MAX_FIELDS, B2_WUKONG_MAX_DIM, B2_WUKONG_MAX_RANK, B2_WUKONG_MAX_FM_WIDTH = 128, 128, 32, 1024
B2_FINALNET_CONCAT, B2_FINALNET_SUM = 0, 1
B2_FINALNET_MAX_WIDTH, B2_FINALNET_MAX_FIELDS, B2_FINALNET_MAX_DIM, B2_FINALNET_MAX_GATE_WIDTH = 1024, 128, 128, 8192
B2_BST_MAX_LEN, B2_BST_MAX_DIM, B2_BST_MAX_HEAD_DIM, B2_BST_MAX_HEADS, B2_BST_MAX_PARTS = 256, 512, 64, 16, 8
B2_BST_POOL_MEAN, B2_BST_POOL_SUM, B2_BST_POOL_TARGET = 0, 1, 2
(B2_TRANSACT_MAX_LEN, B2_TRANSACT_MAX_DIM, B2_TRANSACT_MAX_HEAD_DIM, B2_TRANSACT_MAX_HEADS,
 B2_TRANSACT_MAX_PARTS) = 256, 512, 256, 16, 8
B2_DIEN_MAX_DIM, B2_DIEN_MAX_LEN = 64, 1024
B2_DIEN_GRU, B2_DIEN_AUGRU, B2_DIEN_AGRU = 0, 1, 2
B2_LSH_MAX_DIM, B2_LSH_MAX_LEN, B2_LSH_MAX_TOPK, B2_LSH_MAX_SMEM = 256, 4096, 256, 227 * 1024 - 1024
B2_ETA_MAX_BITS, B2_SDIM_MAX_BITS, B2_SDIM_MAX_HASHES = 64, 24, 32
B2_MIRRN_MAX_BITS = 64
B2_LONGCTR_PAD_PRE, B2_LONGCTR_PAD_POST, B2_LONGCTR_MAX_LEN, B2_LONGCTR_MAX_COLS = 0, 1, 1 << 20, 64
B2_TOPK_MAX_DIM, B2_TOPK_MAX_LEN, B2_TOPK_MAX_K, B2_TOPK_MAX_SMEM = 256, 4096, 256, 220 * 1024
FM_PRODUCT_SUM, FM_BI_INTERACTION, FM_INNER_PRODUCT = 0, 1, 2

c_void_p, c_int, c_int32, c_int64, c_float, c_double = (ctypes.c_void_p, ctypes.c_int, ctypes.c_int32,
                                                        ctypes.c_int64, ctypes.c_float, ctypes.c_double)


class b2_lazy_ctx(ctypes.Structure):
    """struct b2_lazy_ctx of include/fuxictr_b200.h."""
    _fields_ = [
        ("last_step", ctypes.c_void_p), ("sched", ctypes.c_void_p), ("step_dev", ctypes.c_void_p),
        ("mark", ctypes.c_void_p), ("worklist", ctypes.c_void_p), ("counter", ctypes.c_void_p),
        ("delta_m", ctypes.c_int64), ("delta_v", ctypes.c_int64),
        ("w1", ctypes.c_float), ("beta2", ctypes.c_float), ("w2", ctypes.c_float), ("eps", ctypes.c_float),
        ("worklist_capacity", ctypes.c_int32), ("pad_", ctypes.c_int32),
        ("grow_emb", ctypes.c_int64 * 128), ("grow_lr", ctypes.c_int64 * 128),
    ]


class b2_lazy_table(ctypes.Structure):
    """struct b2_lazy_table of include/fuxictr_b200.h (32 bytes)."""
    _fields_ = [("param", ctypes.c_void_p), ("rows", ctypes.c_int64), ("grow_base", ctypes.c_int64),
                ("dim", ctypes.c_int32), ("pad_", ctypes.c_int32)]


class b2_field(ctypes.Structure):
    """struct b2_field of include/fuxictr_b200.h (64 bytes)."""
    _fields_ = [
        ("table", c_void_p), ("idx", c_void_p), ("out", c_void_p),
        ("vocab", c_int64), ("idx_stride", c_int64), ("out_stride", c_int64),
        ("dim", c_int32), ("seq_len", c_int32), ("pool", c_int32), ("padding_idx", c_int32),
    ]


class b2_touch(ctypes.Structure):
    """struct b2_touch of include/fuxictr_b200.h (24 bytes)."""
    _fields_ = [("flags", c_void_p), ("base", c_void_p), ("n", c_int64)]


_FIELD_P = ctypes.POINTER(b2_field)


class b2_gemm_desc(ctypes.Structure):
    """struct b2_gemm_desc of include/fuxictr_b200.h."""
    _fields_ = [
        ("a", c_void_p), ("b", c_void_p), ("a_small", c_void_p), ("b_small", c_void_p),
        ("c", c_void_p), ("c_small", c_void_p), ("c_pre", c_void_p), ("bias", c_void_p), ("mul", c_void_p), ("add", c_void_p),
        ("ybwd", c_void_p), ("colsum", c_void_p),
        ("lda", c_int64), ("ldb", c_int64), ("ldc", c_int64), ("M", c_int64), ("N", c_int64), ("K", c_int64),
        ("a_mn_major", c_int32), ("b_mn_major", c_int32), ("act", c_int32), ("act_bwd", c_int32),
        ("beta_accumulate", c_int32), ("elem_dtype", c_int32), ("ld_aux", c_int64),
        ("flags", c_int64),
        ("drop_rng", c_void_p), ("drop_layer", c_int64), ("drop_thresh", ctypes.c_uint32), ("drop_scale", c_float),
    ]

class b2_gemm_plan(ctypes.Structure):
    """struct b2_gemm_plan of include/fuxictr_b200.h."""
    _fields_ = [(k, c_int32) for k in ("bn", "splits", "stages", "cstages", "grid", "threads", "tiles_m", "tiles_n",
                                       "passes", "kb_per_split")] + \
               [("smem_bytes", c_int64)]


# name -> (restype, argtypes); every symbol the header declares must appear here
# (tests/test_abi.py cross-checks this table against the header text).
SIGNATURES = {
    "b2_version": (ctypes.c_char_p, []),
    "b2_last_error": (ctypes.c_char_p, []),
    "b2_device_cc": (c_int, [c_int]),
    "b2_set_l2_fetch_granularity": (c_int, [c_int]),
    "b2_embed_gather_fwd": (c_int, [_FIELD_P, c_int, c_int64, c_int, c_int, c_void_p, c_void_p, c_int, c_void_p]),
    "b2_embed_scatter_bwd": (c_int, [_FIELD_P, c_int, c_int64, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "b2_lr_fwd": (c_int, [_FIELD_P, c_int, c_int64, c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    "b2_lr_bwd": (c_int, [_FIELD_P, c_int, c_int64, c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    "b2_front_fwd": (c_int, [_FIELD_P, _FIELD_P, c_int, c_int64, c_int, c_int, c_void_p, c_void_p, c_void_p,
                             c_void_p, c_void_p, c_void_p, c_void_p]),
    "b2_front_bwd": (c_int, [_FIELD_P, _FIELD_P, c_int, c_int64, c_int, c_int, c_void_p, c_void_p, c_void_p,
                             c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "b2_lazy_sumsq": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_int, c_int64, c_void_p, c_void_p]),
    "b2_lazy_adam_step": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_int, c_int64, c_int64, c_int64, c_void_p,
                                  c_void_p, c_void_p, c_void_p, c_float, c_double, c_double, c_float, c_void_p]),
    "b2_lazy_materialize": (c_int, [c_void_p, c_int, c_int64, c_int64, c_int64, c_void_p, c_void_p, c_void_p,
                                    c_double, c_double, c_float, c_void_p]),
    "b2_adam_sched": (c_int, [c_void_p, c_double, c_double, c_double, c_void_p, c_int64, c_void_p]),
    "b2_adam_step_sched": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_void_p, c_float, c_double,
                                   c_double, c_float, c_void_p, c_void_p, c_int, c_void_p]),
    "b2_shard_push": (c_int, [_FIELD_P, _FIELD_P, c_int, c_int64, c_int, c_int, c_void_p, c_int, c_int64,
                              c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int32, c_void_p, c_void_p,
                              c_void_p]),
    "b2_shard_pull": (c_int, [_FIELD_P, _FIELD_P, c_int, c_int64, c_int, c_int, c_void_p, c_void_p, c_float,
                              c_void_p, c_void_p, c_int32, c_void_p, c_void_p, c_void_p]),
    "b2_shard_publish_ids": (c_int, [c_void_p, c_int, c_int64, c_void_p, _FIELD_P, _FIELD_P, c_int, c_int, c_int,
                                     c_void_p, c_void_p]),
    "b2_shard_publish_rows": (c_int, [c_void_p, c_int, c_int64, c_int64, c_int64, c_void_p, _FIELD_P, _FIELD_P, c_int,
                                      c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "b2_shard_lookup": (c_int, [_FIELD_P, _FIELD_P, c_int, c_int64, c_int, c_int, c_void_p, c_int64, c_void_p, c_void_p,
                                c_void_p, c_void_p, c_void_p, c_void_p]),
    "b2_front_reduce": (c_int, [c_void_p, c_void_p, c_void_p, c_int64, c_int, c_int, c_int, c_void_p, c_void_p,
                                c_void_p]),
    "b2_front_gprep": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int, c_int, c_int, c_void_p,
                               c_void_p, c_void_p, c_int, c_void_p]),
    "b2_fm_fwd": (c_int, [c_void_p, c_int64, c_int, c_int, c_int, c_void_p, c_void_p]),
    "b2_fm_bwd": (c_int, [c_void_p, c_void_p, c_int64, c_int, c_int, c_int, c_void_p, c_void_p]),
    "b2_crossnet_fwd": (c_int, [c_void_p, c_void_p, c_void_p, c_int64, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "b2_crossnet_bwd": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int, c_int,
                                c_void_p, c_void_p, c_void_p, c_void_p]),
    "b2_crossmix_pack": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "b2_crossmix_fwd": (c_int, [c_void_p, c_void_p, c_int64, c_int, c_int, c_void_p, c_void_p, c_int, c_int64,
                                c_void_p]),
    "b2_crossmix_bwd": (c_int, [c_void_p, c_void_p, c_void_p, c_int64, c_int, c_int, c_void_p, c_void_p, c_int,
                                c_int64, c_void_p, c_void_p]),
    "b2_crossmix_unpack": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p,
                                   c_void_p]),
    "b2_gdcn_pack": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_void_p]),
    "b2_gdcn_fwd": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int, c_void_p, c_void_p, c_int,
                            c_int64, c_void_p]),
    "b2_gdcn_bwd": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int, c_void_p, c_void_p, c_int,
                            c_int64, c_void_p, c_void_p, c_void_p]),
    "b2_gdcn_unpack": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p]),
    "b2_fs_gate_fwd": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int64, c_int, c_void_p, c_void_p,
                               c_void_p, c_void_p, c_int, c_int64, c_void_p]),
    "b2_fs_gate_bwd": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_int64, c_int,
                               c_void_p, c_void_p, c_void_p, c_void_p]),
    "b2_agg_pack": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "b2_agg_fwd": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int, c_void_p, c_void_p]),
    "b2_agg_bwd": (c_int, [c_void_p, c_void_p, c_void_p, c_int64, c_int, c_void_p, c_void_p, c_void_p, c_int,
                           c_int64, c_void_p, c_void_p, c_void_p, c_void_p]),
    "b2_agg_unpack": (c_int, [c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "b2_field_ln_fwd": (c_int, [c_void_p, c_int64, c_int, c_int, c_void_p, c_void_p, c_int64, c_float, c_void_p,
                                c_void_p, c_void_p, c_void_p]),
    "b2_field_ln_bwd": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int, c_int, c_void_p, c_int64,
                                c_void_p, c_int, c_void_p, c_void_p, c_void_p]),
    "b2_mask_row_fwd": (c_int, [c_void_p, c_int64, c_int, c_void_p, c_void_p, c_float, c_int, c_void_p, c_int64,
                                ctypes.c_uint32, c_float, c_void_p, c_int64, c_void_p, c_int, c_int64, c_void_p,
                                c_void_p, c_void_p]),
    "b2_mask_row_bwd": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_int64,
                                ctypes.c_uint32, c_float, c_void_p, c_int64, c_int64, c_int, c_void_p, c_void_p, c_int,
                                c_int64, c_void_p, c_void_p, c_void_p]),
    "b2_mask_mul": (c_int, [c_void_p, c_void_p, c_int64, c_void_p, c_int, c_void_p]),
    "b2_autoint_pack": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p]),
    "b2_autoint_fwd": (c_int, [c_void_p, c_void_p, c_int64, c_int, c_int, c_int, c_int, c_int, c_float, c_void_p,
                               c_void_p, c_float, c_void_p, c_int64, ctypes.c_uint32, c_float, c_void_p, c_void_p,
                               c_int, c_int64, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "b2_autoint_bwd": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                               c_int64, c_int, c_int, c_int, c_int, c_int, c_float, c_void_p, c_void_p, c_int64,
                               ctypes.c_uint32, c_float, c_void_p, c_void_p, c_int, c_int64, c_void_p, c_void_p,
                               c_void_p, c_void_p]),
    "b2_autoint_unpack": (c_int, [c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "b2_wukong_fm_fwd": (c_int, [c_void_p, c_int, c_int64, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_float,
                                 c_void_p, c_void_p, c_int, c_int64, c_void_p, c_void_p, c_int64, c_void_p, c_void_p,
                                 c_void_p]),
    "b2_wukong_fm_bwd": (c_int, [c_void_p, c_int, c_int64, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p,
                                 c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    "b2_wukong_out_fwd": (c_int, [c_void_p, c_void_p, c_void_p, c_int64, c_int, c_int, c_int, c_int, c_int, c_void_p,
                                  c_void_p, c_float, c_int, c_void_p, c_void_p, c_int, c_int64, c_void_p, c_void_p,
                                  c_void_p]),
    "b2_wukong_out_bwd": (c_int, [c_void_p, c_void_p, c_void_p, c_int64, c_int, c_int, c_int, c_int, c_int, c_void_p,
                                  c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int64,
                                  c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    "b2_wukong_pack": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "b2_wukong_unpack": (c_int, [c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "b2_finalnet_fi_fwd": (c_int, [c_void_p, c_int64, c_int, c_int, c_void_p, c_void_p, c_float, c_float, c_int,
                                   c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_int64, ctypes.c_uint32,
                                   c_float, c_void_p, c_void_p, c_int, c_int64, c_void_p, c_void_p, c_void_p]),
    "b2_finalnet_fi_bwd": (c_int, [c_void_p, c_int64, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_int,
                                   c_void_p, c_int, c_int, c_void_p, c_int64, ctypes.c_uint32, c_float, c_void_p,
                                   c_void_p, c_void_p, c_int, c_int64, c_void_p, c_void_p, c_void_p, c_void_p]),
    "b2_finalnet_gate_fwd": (c_int, [c_void_p, c_int64, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_int,
                                     c_int64, c_void_p]),
    "b2_finalnet_gate_bwd": (c_int, [c_void_p, c_int64, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_int,
                                     c_void_p, c_void_p, c_void_p]),
    "b2_finalnet_loss": (c_int, [c_void_p, c_void_p, c_void_p, c_int64, c_void_p, c_void_p, c_void_p, c_void_p,
                                 c_void_p]),
    "b2_bst_tokens_fwd": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_int64, c_int, c_int,
                                  c_void_p, c_void_p, c_int, c_int64, c_void_p]),
    "b2_bst_tokens_bwd": (c_int, [c_void_p, c_void_p, c_int64, c_int, c_int, c_int, c_int, c_void_p, c_void_p,
                                  c_void_p, c_void_p]),
    "b2_bst_attn_fwd": (c_int, [c_void_p, c_void_p, c_int64, c_int, c_int, c_int, c_int, c_float, c_void_p, c_int64,
                                ctypes.c_uint32, c_float, c_void_p, c_void_p, c_int, c_int64, c_void_p, c_void_p,
                                c_void_p]),
    "b2_bst_attn_bwd": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int, c_int,
                                c_int, c_int, c_float, c_void_p, c_int64, ctypes.c_uint32, c_float, c_void_p, c_void_p,
                                c_int, c_int64, c_void_p]),
    "b2_bst_addnorm_fwd": (c_int, [c_void_p, c_void_p, c_int64, c_int, c_void_p, c_void_p, c_float, c_void_p, c_int64,
                                   ctypes.c_uint32, c_float, c_void_p, c_void_p, c_int, c_int64, c_void_p, c_void_p,
                                   c_void_p]),
    "b2_bst_addnorm_bwd": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int, c_void_p, c_void_p,
                                   c_void_p, c_void_p, c_int64, ctypes.c_uint32, c_float, c_void_p, c_void_p, c_int,
                                   c_int64, c_void_p, c_void_p, c_void_p, c_void_p]),
    "b2_bst_pool_fwd": (c_int, [c_void_p, c_void_p, c_int64, c_int, c_int, c_int, c_void_p, c_int64, c_void_p]),
    "b2_bst_pool_bwd": (c_int, [c_void_p, c_int64, c_void_p, c_int64, c_int, c_int, c_int, c_void_p, c_void_p]),
    "b2_transact_tokens_fwd": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_int, c_void_p, c_int, c_int64,
                                       c_int64, c_int, c_int, c_void_p, c_void_p, c_int, c_int64, c_void_p, c_void_p]),
    "b2_transact_tokens_bwd": (c_int, [c_void_p, c_int64, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "b2_transact_attn_fwd": (c_int, [c_void_p, c_void_p, c_int64, c_int, c_int, c_int, c_float, c_void_p, c_int64,
                                     ctypes.c_uint32, c_float, c_void_p, c_void_p, c_int, c_int64, c_void_p, c_void_p,
                                     c_void_p]),
    "b2_transact_attn_bwd": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int, c_int,
                                     c_int, c_float, c_void_p, c_int64, ctypes.c_uint32, c_float, c_void_p, c_void_p,
                                     c_void_p, c_int, c_int64, c_void_p]),
    "b2_transact_out_fwd": (c_int, [c_void_p, c_void_p, c_int64, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p,
                                    c_void_p, c_int, c_int64, c_void_p]),
    "b2_transact_out_bwd": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int, c_int, c_int, c_void_p,
                                    c_void_p]),
    "b2_gru_fwd": (c_int, [c_void_p, c_int64, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int,
                           c_int64, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "b2_gru_bwd": (c_int, [c_void_p, c_int64, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int,
                           c_int64, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p,
                           c_void_p, c_void_p, c_void_p, c_void_p]),
    "b2_dien_scores_fwd": (c_int, [c_void_p, c_void_p, c_int64, c_void_p, c_void_p, c_int64, c_int, c_int, c_void_p,
                                   c_void_p, c_void_p]),
    "b2_dien_scores_bwd": (c_int, [c_void_p, c_void_p, c_int64, c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int,
                                   c_int, c_void_p, c_int, c_void_p, c_void_p, c_void_p]),
    "b2_dien_sum_pool_fwd": (c_int, [c_void_p, c_void_p, c_int64, c_int64, c_int, c_int, c_void_p, c_int64, c_void_p]),
    "b2_dien_sum_pool_bwd": (c_int, [c_void_p, c_void_p, c_int64, c_void_p, c_int64, c_int64, c_int, c_int, c_void_p,
                                     c_void_p, c_int, c_void_p]),
    "b2_eta_retrieve_fwd": (c_int, [c_void_p, c_void_p, c_void_p, c_int64, c_int64, c_int, c_int, c_int, c_int,
                                    c_void_p, c_void_p, c_void_p, c_void_p]),
    "b2_sdim_pool_fwd": (c_int, [c_void_p, c_void_p, c_void_p, c_int64, c_int64, c_int, c_int, c_int, c_int, c_int,
                                 c_void_p, c_void_p, c_void_p, c_void_p]),
    "b2_eta_assemble_bwd": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_int64, c_int,
                                    c_int, c_int, c_void_p, c_void_p]),
    "b2_sdim_assemble_bwd": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p,
                                     c_int64, c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
    "b2_mirrn_retrieve_fwd": (c_int, [c_void_p, c_void_p, c_void_p, c_int64, c_int64, c_int, c_int, c_int, c_int,
                                      c_void_p, c_void_p]),
    "b2_mirrn_filter_fwd": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p,
                                    c_int64, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "b2_mirrn_filter_bwd": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p,
                                    c_void_p, c_int64, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p,
                                    c_void_p, c_void_p]),
    "b2_mirrn_mean_fwd": (c_int, [c_void_p, c_int64, c_int, c_int, c_void_p, c_void_p]),
    "b2_mirrn_mean_bwd": (c_int, [c_void_p, c_int64, c_int, c_int, c_void_p, c_void_p]),
    "b2_mirrn_assemble_bwd": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_int64,
                                      c_int, c_int, c_int, c_void_p, c_void_p]),
    "b2_longctr_collate": (c_int, [c_void_p, c_int, c_int64, c_int64, c_int, c_int, c_int, c_void_p, c_void_p,
                                   c_int64, c_void_p, c_int64, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "b2_sim_retrieve_fwd": (c_int, [c_void_p, c_void_p, c_void_p, c_int64, c_int, c_int, c_int, c_void_p, c_void_p,
                                    c_void_p, c_void_p, c_void_p, c_void_p]),
    "b2_sim_gsu_bwd": (c_int, [c_void_p, c_void_p, c_void_p, c_int64, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "b2_sim_assemble_bwd": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p,
                                    c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int, c_int, c_int, c_void_p,
                                    c_void_p]),
    "b2_twin_topk_fwd": (c_int, [c_void_p, c_void_p, c_void_p, c_int64, c_int, c_int, c_int, c_int, c_void_p, c_void_p,
                                 c_void_p, c_void_p]),
    "b2_twin_topk_bwd": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                 c_void_p, c_void_p, c_void_p, c_int, c_int64, c_int, c_int, c_int, c_int, c_void_p,
                                 c_void_p, c_void_p]),
    "b2_mhta_pack":(c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_float, c_void_p,
                             c_void_p, c_void_p]),
    "b2_mhta_fwd": (c_int, [c_void_p, c_void_p, c_void_p, c_int64, c_int, c_int, c_int, c_int, c_int, c_float,
                            c_void_p, c_void_p, c_void_p, c_int, c_int64, c_void_p]),
    "b2_mhta_bwd": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int, c_int, c_int,
                            c_int, c_int, c_float, c_void_p, c_void_p, c_void_p, c_int, c_int64, c_void_p]),
    "b2_mhta_unpack": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int,
                               c_float, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "b2_cin_fwd": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int, c_int, c_int, c_int, c_void_p,
                           c_void_p]),
    "b2_cin_bwd": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int, c_int, c_int, c_int, c_void_p,
                           c_int, c_void_p, c_void_p, c_void_p]),
    "b2_dice_fwd": (c_int, [c_void_p, c_void_p, c_int64, c_int, c_float, c_float, c_int, c_void_p, c_void_p,
                            c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "b2_dice_bwd": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int, c_int, c_void_p,
                            c_void_p, c_void_p, c_void_p]),
    "b2_din_input_fwd": (c_int, [c_void_p, c_void_p, c_int64, c_int, c_int, c_void_p, c_void_p]),
    "b2_din_input_bwd": (c_int, [c_void_p, c_void_p, c_void_p, c_int64, c_int, c_int, c_void_p, c_void_p, c_int,
                                 c_void_p]),
    "b2_din_wsum_fwd": (c_int, [c_void_p, c_void_p, c_void_p, c_int64, c_int, c_int, c_void_p, c_void_p]),
    "b2_din_wsum_bwd": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int, c_int, c_void_p, c_void_p,
                                c_void_p]),
    "b2_din_softmax_fwd": (c_int, [c_void_p, c_void_p, c_int64, c_int, c_void_p, c_void_p]),
    "b2_din_softmax_bwd": (c_int, [c_void_p, c_void_p, c_void_p, c_int64, c_int, c_void_p, c_void_p]),
    "b2_gemm_f32": (c_int, [c_void_p, c_int64, c_int64, c_void_p, c_int64, c_int64, c_void_p, c_int64,
                            c_int64, c_int64, c_int64, c_void_p, c_int, c_void_p, c_void_p, c_int, c_void_p]),
    "b2_gemm_tc_ex": (c_int, [c_void_p, c_void_p]),
    "b2_gemm_tc_plan": (c_int, [c_void_p, c_void_p]),
    "b2_to_bf16": (c_int, [c_void_p, c_int64, c_int64, c_int64, c_void_p, c_int64, c_void_p]),
    "b2_split_tf32": (c_int, [c_void_p, c_void_p, c_int64, c_void_p]),
    "b2_prep_operand": (c_int, [c_void_p, c_void_p, c_int, c_int64, c_int64, c_void_p, c_void_p, c_void_p, c_void_p,
                                c_void_p, c_void_p, c_int64, ctypes.c_uint32, c_float, c_void_p]),
    "b2_head_fwd": (c_int, [c_void_p, c_void_p, c_void_p, c_int64, c_int, c_int, c_void_p, c_void_p]),
    "b2_head_bwd": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int, c_int, c_void_p, c_void_p,
                            c_void_p, c_void_p]),
    "b2_head_bwd_ex": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int, c_int, c_void_p, c_void_p,
                               c_void_p, c_int, c_void_p, c_void_p, c_int, c_void_p, c_int64, ctypes.c_uint32, c_float,
                               c_void_p]),
    "b2_dropout_rng_take": (c_int, [c_void_p, c_void_p, c_int, c_void_p]),
    "b2_dropout_apply": (c_int, [c_void_p, c_void_p, c_int64, c_int64, c_int64, c_void_p, c_int64, ctypes.c_uint32,
                                 c_float, c_void_p]),
    "b2_logit_bce_fwd": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int64,
                                 c_void_p, c_void_p, c_void_p, c_void_p]),
    "b2_sumsq": (c_int, [c_void_p, c_int64, c_void_p, c_void_p]),
    "b2_adam_step": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_void_p, c_float, c_double,
                             c_double, c_double, c_float, c_void_p, c_int, c_void_p]),
    "b2_sumsq_ex": (c_int, [c_void_p, c_int64, c_void_p, c_void_p, c_int64, c_void_p]),
    "b2_adam_step_ex": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_void_p, c_float, c_double,
                                c_double, c_double, c_float, c_void_p, c_int, c_void_p, c_int64, c_void_p]),
    "b2_adam_untouched": (c_int, [c_void_p, c_void_p, c_void_p, c_int64, c_void_p, c_double, c_double, c_double,
                                  c_float, c_void_p, c_int, c_void_p]),
    "b2_adam_touched": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_void_p, c_float, c_double,
                                c_double, c_double, c_float, c_void_p, c_void_p, c_void_p]),
    "b2_table_mark": (c_int, [_FIELD_P, _FIELD_P, c_int, c_int64, c_int, c_void_p, c_void_p]),
    "b2_logloss_sum": (c_int, [c_void_p, c_void_p, c_int64, c_void_p, c_void_p]),
    "b2_auc_workspace_bytes": (c_int, [c_int64, ctypes.POINTER(c_int64)]),
    "b2_auc": (c_int, [c_void_p, c_void_p, c_int64, c_void_p, c_int64, c_void_p, c_void_p]),
    "b2_sort_u32": (c_int, [c_void_p, c_int64, c_void_p, c_int64, c_void_p]),
}

_lib = None


class B2Error(RuntimeError):
    """A C-ABI call returned a negative status (message from b2_last_error())."""


def load():
    """dlopen the in-tree library; raises (never falls back) when it is absent."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            "fuxictr_b200: %s is missing. Build it with `python -m fuxictr_b200.build` "
            "(needs nvcc); there is no CPU fallback for the H100 hot path." % LIB_PATH)
    lib = ctypes.CDLL(LIB_PATH)
    for name, (restype, argtypes) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError here == header/library mismatch: fail loudly
        fn.restype = restype
        fn.argtypes = argtypes
    _lib = lib
    gran = os.environ.get("B2_L2_FETCH", "")
    if gran:      # diagnostic override of cudaLimitMaxL2FetchGranularity (see b2_set_l2_fetch_granularity)
        rc = lib.b2_set_l2_fetch_granularity(int(gran))
        if rc != 0 and lib.b2_device_cc(0) > 0:
            raise B2Error("b2_set_l2_fetch_granularity(%s): %s" % (gran, lib.b2_last_error().decode()))
    return lib


def call(name, *args):
    """Invoke an int-returning entry point and raise B2Error on failure."""
    lib = load()
    rc = getattr(lib, name)(*args)
    if rc != 0:
        raise B2Error("%s failed (%d): %s" % (name, rc, lib.b2_last_error().decode()))


def version():
    return load().b2_version().decode()

"""ctypes binding of libmultimae_b200.so (the C ABI declared in include/multimae_b200.h).

The library is the product: there is no Python/CPU fallback.  `lib()` raises if the shared object is missing
or was built for a different ABI version.
"""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libmultimae_b200.so")

c_void_p = ctypes.c_void_p
c_int = ctypes.c_int
c_i64 = ctypes.c_int64
c_float = ctypes.c_float


class GemmEpilogue(ctypes.Structure):
    _fields_ = [
        ("alpha", c_float),
        ("act", c_int),
        ("accumulate", c_int),
        ("reserved", c_int),
        ("bias", c_void_p),
        ("residual", c_void_p),
        ("dgelu_z", c_void_p),
        ("preact_bf16", c_void_p),
        ("out_f32", c_void_p),
        ("out_bf16", c_void_p),
        ("ld_residual", c_i64),
        ("ld_dgelu_z", c_i64),
        ("ld_preact", c_i64),
        ("ld_out_f32", c_i64),
        ("ld_out_bf16", c_i64),
    ]


MAX_TASKS = 8
c_float_p = c_void_p  # device pointers travel as integers
POS_MODES = {"bicubic": 0, "bilinear": 1}     # MMAE_POS_BICUBIC / MMAE_POS_BILINEAR


class EmbedLayout(ctypes.Structure):
    _fields_ = [
        ("num_tasks", c_int),
        ("grid_h", c_int * MAX_TASKS), ("grid_w", c_int * MAX_TASKS),
        ("tok_offset", c_int * (MAX_TASKS + 1)),
        ("k_offset", c_int * (MAX_TASKS + 1)),
        ("patch", c_int * MAX_TASKS), ("channels", c_int * MAX_TASKS),
        ("is_semseg", c_int * MAX_TASKS), ("num_classes", c_int * MAX_TASKS),
    ]


class EmbedInputs(ctypes.Structure):
    _fields_ = [("data", c_void_p * MAX_TASKS), ("class_emb", c_void_p * MAX_TASKS)]


class EmbedParams(ctypes.Structure):
    _fields_ = [("weight", c_void_p * MAX_TASKS), ("bias", c_void_p * MAX_TASKS), ("pos", c_void_p * MAX_TASKS),
                ("global_tokens", c_void_p)]


class EmbedGrads(ctypes.Structure):
    _fields_ = [("weight", c_void_p * MAX_TASKS), ("bias", c_void_p * MAX_TASKS), ("class_emb", c_void_p * MAX_TASKS),
                ("global_tokens", c_void_p)]


BLOCK_FIELDS = ["norm1_w", "norm1_b", "qkv_w", "qkv_b", "proj_w", "proj_b", "norm2_w", "norm2_b", "fc1_w", "fc1_b",
                "fc2_w", "fc2_b"]


class BlockParams(ctypes.Structure):
    _fields_ = [(n, c_void_p) for n in BLOCK_FIELDS]


class BlockGrads(ctypes.Structure):
    _fields_ = [(n, c_void_p) for n in BLOCK_FIELDS]


class BlockDropout(ctypes.Structure):
    _fields_ = [("attn_p", c_float), ("proj_p", c_float), ("mlp_p", c_float), ("seed", c_void_p), ("prev_mlp_p", c_float),
                ("prev_seed", c_void_p)]


class DecoderIndex(ctypes.Structure):
    _fields_ = [("batch", c_int), ("dim", c_int), ("num_visible", c_int), ("num_global", c_int),
                ("num_queries", c_int), ("total_tokens", c_int), ("num_tasks", c_int), ("own_task", c_int),
                ("query_mode", c_int), ("tok_offset", c_int * (MAX_TASKS + 1)), ("ids_keep", c_void_p), ("ids_restore", c_void_p)]


HEAD_TAIL_FIELDS = ["context_norm_w", "context_norm_b", "query_norm_w", "query_norm_b", "out_norm_w", "out_norm_b",
                    "q_w", "q_b", "kv_w", "kv_b", "proj_w", "proj_b", "fc1_w", "fc1_b", "fc2_w", "fc2_b"]


class DecHeadParams(ctypes.Structure):
    _fields_ = ([("proj_context_w", c_void_p), ("proj_context_b", c_void_p), ("mask_token", c_void_p),
                 ("pos", c_void_p), ("task_emb", c_void_p * MAX_TASKS)] + [(n, c_void_p) for n in HEAD_TAIL_FIELDS])


class DecHeadGrads(ctypes.Structure):
    _fields_ = ([("proj_context_w", c_void_p), ("proj_context_b", c_void_p), ("mask_token", c_void_p),
                 ("task_emb", c_void_p * MAX_TASKS)] + [(n, c_void_p) for n in HEAD_TAIL_FIELDS])


class CtxProjParams(ctypes.Structure):
    _fields_ = [("num", c_int), ("dim", c_int * MAX_TASKS), ("weight", c_void_p * MAX_TASKS), ("bias", c_void_p * MAX_TASKS)]


class CtxProjGrads(ctypes.Structure):
    _fields_ = [("weight", c_void_p * MAX_TASKS)]


class AdamwSegment(ctypes.Structure):
    _fields_ = [("param", c_void_p), ("grad", c_void_p), ("exp_avg", c_void_p), ("exp_avg_sq", c_void_p),
                ("mirror_bf16", c_void_p), ("n", c_i64), ("group", c_int), ("reserved", c_int)]


class MmaeError(RuntimeError):
    pass


_lib = None

# name -> (restype, argtypes); every symbol of include/multimae_b200.h appears here
SIGNATURES = {
    "mmae_abi_version": (c_int, []),
    "mmae_last_error": (ctypes.c_char_p, []),
    "mmae_launch_count": (c_i64, []),
    "mmae_profile_gemm": (c_int, [c_int]),
    "mmae_profile_gemm_read": (c_int, [ctypes.POINTER(ctypes.c_double), ctypes.POINTER(ctypes.c_double),
                                       ctypes.POINTER(c_i64)]),
    "mmae_profile_gemm_dump": (c_i64, [ctypes.c_char_p, c_i64]),
    "mmae_gemm_set_variant": (c_int, [c_int]),
    "mmae_gemm_set_tma_store": (c_int, [c_int]),
    "mmae_set_pdl": (c_int, [c_int]),
    "mmae_set_wgrad_stream": (c_int, [c_int]),
    "mmae_gemm_bf16": (c_int, [c_void_p, c_i64, c_int, c_void_p, c_i64, c_int, c_int, c_int, c_int, c_int,
                               ctypes.POINTER(GemmEpilogue), c_void_p]),
    "mmae_cast_f32_to_bf16": (c_int, [c_void_p, c_void_p, c_i64, c_void_p]),
    "mmae_cast_colsum_f32": (c_int, [c_void_p, c_i64, c_void_p, c_i64, c_void_p, c_int, c_int, c_void_p]),
    "mmae_colsum_bf16": (c_int, [c_void_p, c_i64, c_void_p, c_int, c_int, c_void_p]),
    "mmae_gelu_bf16": (c_int, [c_void_p, c_void_p, c_i64, c_int, c_void_p]),
    "mmae_dgelu_colsum_bf16": (c_int, [c_void_p, c_void_p, c_i64, c_void_p, c_int, c_int, c_void_p]),
    "mmae_set_fuse_gelu": (c_int, [c_int]),
    "mmae_add_bf16_f32": (c_int, [c_void_p, c_void_p, c_void_p, c_i64, c_void_p]),
    "mmae_transpose_bf16": (c_int, [c_void_p, c_i64, c_void_p, c_i64, c_int, c_int, c_void_p]),
    "mmae_layernorm_forward": (c_int, [c_void_p, c_i64, c_void_p, c_void_p, c_void_p, c_i64, c_void_p, c_i64,
                                       c_void_p, c_void_p, c_int, c_int, c_float, c_void_p]),
    "mmae_add_layernorm_forward": (c_int, [c_void_p, c_i64, c_void_p, c_i64, c_void_p, c_i64, c_void_p, c_void_p, c_void_p,
                                           c_i64, c_void_p, c_void_p, c_int, c_int, c_float, c_void_p]),
    "mmae_layernorm_backward": (c_int, [c_void_p, c_int, c_i64, c_void_p, c_i64, c_void_p, c_void_p, c_void_p,
                                        c_void_p, c_i64, c_void_p, c_i64, c_void_p, c_void_p, c_int, c_int, c_void_p]),
    "mmae_layernorm_backward_ex": (c_int, [c_void_p, c_int, c_i64, c_void_p, c_i64, c_void_p, c_void_p, c_void_p,
                                           c_void_p, c_i64, c_void_p, c_i64, c_void_p, c_void_p, c_void_p, c_i64, c_void_p,
                                           c_int, c_int, c_void_p]),
    "mmae_set_sm_budget": (c_int, [c_int]),
    "mmae_attention_set_tc": (c_int, [c_int]),
    "mmae_attention_forward": (c_int, [c_void_p, c_i64, c_void_p, c_i64, c_void_p, c_i64, c_void_p, c_i64, c_void_p,
                                       c_int, c_int, c_int, c_int, c_int, c_float, c_float, c_void_p, c_void_p]),
    "mmae_attention_backward": (c_int, [c_void_p, c_i64, c_void_p, c_i64, c_void_p, c_i64, c_void_p, c_i64, c_void_p,
                                        c_i64, c_void_p, c_void_p, c_void_p, c_i64, c_void_p, c_i64, c_void_p, c_i64,
                                        c_int, c_int, c_int, c_int, c_int, c_float, c_float, c_void_p, c_void_p]),
    "mmae_dropout_keep_mask": (c_int, [c_void_p, c_int, c_i64, c_int, c_float, c_void_p, c_void_p]),
    "mmae_sample_masks": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, ctypes.POINTER(c_int), c_int, c_void_p,
                                  c_void_p, c_void_p, c_void_p]),
    "mmae_embed_saved_bytes": (c_i64, [ctypes.POINTER(EmbedLayout), c_int, c_int, c_int]),
    "mmae_embed_workspace_bytes": (c_i64, [ctypes.POINTER(EmbedLayout), c_int, c_int, c_int]),
    "mmae_embed_forward": (c_int, [ctypes.POINTER(EmbedLayout), ctypes.POINTER(EmbedInputs), ctypes.POINTER(EmbedParams),
                                   c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    "mmae_embed_backward": (c_int, [ctypes.POINTER(EmbedLayout), ctypes.POINTER(EmbedInputs),
                                    ctypes.POINTER(EmbedParams), ctypes.POINTER(EmbedGrads), c_void_p, c_int, c_int,
                                    c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    "mmae_pos_resample_forward": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
    "mmae_pos_resample_backward": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
    "mmae_embed_pos_backward": (c_int, [ctypes.POINTER(EmbedLayout), c_void_p, c_int, c_int, c_int, c_int, c_void_p,
                                        ctypes.POINTER(c_void_p), c_void_p]),
    "mmae_block_saved_bytes": (c_i64, [c_int] * 5),
    "mmae_block_workspace_bytes": (c_i64, [c_int] * 5),
    "mmae_block_forward": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int,
                                   c_float, c_void_p, c_void_p, c_void_p, ctypes.POINTER(BlockDropout),
                                   ctypes.POINTER(BlockParams), c_void_p, c_void_p, c_void_p]),
    "mmae_block_saved_x_mid": (c_void_p, [c_void_p, c_int, c_int, c_int, c_int, c_int]),
    "mmae_block_backward": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int,
                                    c_int, c_int, c_void_p, c_void_p, c_void_p, ctypes.POINTER(BlockDropout),
                                    ctypes.POINTER(BlockParams), ctypes.POINTER(BlockGrads), c_void_p, c_void_p, c_void_p]),
    "mmae_dechead_saved_bytes": (c_i64, [ctypes.POINTER(DecoderIndex), c_int, c_int, c_int]),
    "mmae_dechead_workspace_bytes": (c_i64, [ctypes.POINTER(DecoderIndex), c_int, c_int, c_int]),
    "mmae_dechead_forward": (c_int, [c_void_p, c_int, ctypes.POINTER(DecoderIndex), c_int, c_int, c_float,
                                     ctypes.POINTER(DecHeadParams), c_void_p, c_void_p, c_void_p, c_void_p]),
    "mmae_dechead_backward": (c_int, [c_void_p, c_int, ctypes.POINTER(DecoderIndex), c_int, c_int,
                                      ctypes.POINTER(DecHeadParams), ctypes.POINTER(DecHeadGrads), c_void_p, c_void_p,
                                      c_void_p, c_void_p, c_void_p]),
    "mmae_ctxproj_saved_bytes": (c_i64, [c_int] * 3),
    "mmae_ctxproj_forward": (c_int, [c_void_p, c_int, c_int, ctypes.POINTER(CtxProjParams), c_void_p, c_void_p, c_void_p]),
    "mmae_ctxproj_backward": (c_int, [c_int, c_int, ctypes.POINTER(CtxProjParams), ctypes.POINTER(CtxProjGrads), c_void_p,
                                      c_void_p, c_void_p, c_void_p]),
    "mmae_dechead_forward_ctx": (c_int, [c_void_p, c_i64, ctypes.POINTER(DecoderIndex), c_int, c_int, c_float,
                                         ctypes.POINTER(DecHeadParams), c_void_p, c_void_p, c_void_p, c_void_p]),
    "mmae_dechead_backward_ctx": (c_int, [ctypes.POINTER(DecoderIndex), c_int, c_int, ctypes.POINTER(DecHeadParams),
                                          ctypes.POINTER(DecHeadGrads), c_void_p, c_void_p, c_i64, c_void_p, c_void_p,
                                          c_void_p]),
    "mmae_dectail_saved_bytes": (c_i64, [c_int] * 6),
    "mmae_dectail_workspace_bytes": (c_i64, [c_int] * 6),
    "mmae_dectail_forward": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p,
                                     c_void_p, c_void_p, c_void_p]),
    "mmae_dectail_backward": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p,
                                      c_void_p, c_void_p, c_void_p, c_void_p]),
    "mmae_masked_loss_forward": (c_int, [c_int, c_int, c_float, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int,
                                         c_int, c_void_p, c_void_p, c_void_p]),
    "mmae_masked_loss_backward": (c_int, [c_int, c_int, c_float, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int,
                                          c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    "mmae_grad_unscale_norm": (c_int, [c_void_p, c_i64, c_void_p, c_float, c_float, c_void_p, c_void_p, c_void_p]),
    "mmae_weight_mirror_register": (c_int, [c_void_p, c_void_p, c_i64]),
    "mmae_adamw_step": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_i64, c_float, c_float, c_float, c_float,
                                c_float, c_int, c_void_p, c_void_p, c_void_p]),
    "mmae_ema_update": (c_int, [ctypes.POINTER(c_void_p), ctypes.POINTER(c_void_p), ctypes.POINTER(c_i64), c_int, c_float,
                                c_float, c_void_p]),
    "mmae_adamw_step_groups": (c_int, [ctypes.POINTER(AdamwSegment), c_int, ctypes.POINTER(ctypes.c_double),
                                       ctypes.POINTER(ctypes.c_double), c_int, ctypes.c_double, ctypes.c_double,
                                       ctypes.c_double, c_void_p, c_void_p, c_void_p]),
    "mmae_augment_batch": (c_int, [c_void_p, c_void_p, c_i64, c_int, c_int, ctypes.POINTER(c_int), c_int, c_i64, c_void_p,
                                   c_i64, ctypes.POINTER(c_void_p), ctypes.POINTER(c_float), ctypes.POINTER(c_float),
                                   c_void_p]),
    "mmae_cls_augment_batch": (c_int, [c_void_p, c_void_p, c_i64, c_int, c_int, c_i64, c_int, ctypes.POINTER(c_int),
                                       c_void_p, c_i64, c_void_p, ctypes.POINTER(c_float), ctypes.POINTER(c_float),
                                       c_void_p]),
    "mmae_unpatchify": (c_int, [c_void_p, c_i64, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p]),
    "mmae_unpatchify_bf16": (c_int, [c_void_p, c_i64, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p]),
    "mmae_patchify_bf16": (c_int, [c_void_p, c_void_p, c_i64, c_int, c_int, c_int, c_int, c_int, c_void_p]),
    "mmae_patchify": (c_int, [c_void_p, c_void_p, c_i64, c_int, c_int, c_int, c_int, c_int, c_void_p]),
    "mmae_clshead_saved_bytes": (c_i64, [c_int] * 4),
    "mmae_clshead_workspace_bytes": (c_i64, [c_int] * 4),
    "mmae_clshead_forward": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_float, c_void_p, c_void_p, c_void_p,
                                     c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "mmae_clshead_backward": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p,
                                      c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "mmae_convnext_proj_saved_bytes": (c_i64, [c_int] * 4),
    "mmae_convnext_proj_workspace_bytes": (c_i64, [c_int] * 4),
    "mmae_convnext_proj_forward": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, ctypes.POINTER(c_int), c_int,
                                           c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "mmae_convnext_proj_backward": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, ctypes.POINTER(c_int), c_int,
                                            c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "mmae_convnext_block_saved_bytes": (c_i64, [c_int] * 5),
    "mmae_convnext_block_workspace_bytes": (c_i64, [c_int] * 5),
    "mmae_convnext_block_forward": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_float,
                                            ctypes.POINTER(c_void_p), c_void_p, c_void_p, c_void_p]),
    "mmae_convnext_block_backward": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int,
                                             ctypes.POINTER(c_void_p), ctypes.POINTER(c_void_p), c_void_p, c_void_p,
                                             c_void_p]),
    "mmae_convnext_tail_saved_bytes": (c_i64, [c_int] * 6),
    "mmae_convnext_tail_workspace_bytes": (c_i64, [c_int] * 6),
    "mmae_convnext_tail_forward": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p,
                                           c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "mmae_convnext_tail_backward": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p,
                                            c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "mmae_segmenter_proj_saved_bytes": (c_i64, [c_int] * 4),
    "mmae_segmenter_proj_workspace_bytes": (c_i64, [c_int] * 4),
    "mmae_segmenter_proj_forward": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, ctypes.POINTER(c_int), c_int, c_int,
                                            c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "mmae_segmenter_proj_backward": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, ctypes.POINTER(c_int), c_int, c_int,
                                             c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "mmae_segmenter_mask_workspace_bytes": (c_i64, [c_int] * 3),
    "mmae_segmenter_mask_forward": (c_int, [c_void_p] * 6 + [c_float, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p,
                                                             c_void_p]),
    "mmae_segmenter_mask_backward": (c_int, [c_void_p] * 8 + [c_int, c_int, c_int, c_int] + [c_void_p] * 6),
    "mmae_segmenter_tail_saved_bytes": (c_i64, [c_int] * 5),
    "mmae_segmenter_tail_workspace_bytes": (c_i64, [c_int] * 5),
    "mmae_segmenter_tail_forward": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_float, c_float,
                                            ctypes.POINTER(c_void_p), c_void_p, c_void_p, c_void_p, c_void_p]),
    "mmae_segmenter_tail_backward": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int,
                                             ctypes.POINTER(c_void_p), ctypes.POINTER(c_void_p), c_void_p, c_void_p, c_void_p]),
    # ---- fp32 tier (fp32_output_adapters)
    "mmae_linear_f32_workspace_bytes": (c_i64, [c_int] * 3),
    "mmae_linear_f32_forward": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p]),
    "mmae_linear_f32_backward": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int,
                                         c_void_p, c_void_p]),
    "mmae_gelu_f32": (c_int, [c_void_p, c_void_p, c_i64, c_int, c_void_p]),
    "mmae_attention_f32_forward": (c_int, [c_void_p, c_i64, c_void_p, c_i64, c_void_p, c_i64, c_void_p, c_i64, c_void_p,
                                           c_int, c_int, c_int, c_int, c_int, c_float, c_void_p]),
    "mmae_attention_f32_backward": (c_int, [c_void_p, c_i64, c_void_p, c_i64, c_void_p, c_i64, c_void_p, c_i64, c_void_p,
                                            c_i64, c_void_p, c_void_p, c_void_p, c_i64, c_void_p, c_i64, c_void_p, c_i64,
                                            c_int, c_int, c_int, c_int, c_int, c_float, c_void_p]),
    "mmae_block_f32_saved_bytes": (c_i64, [c_int] * 5),
    "mmae_block_f32_workspace_bytes": (c_i64, [c_int] * 5),
    "mmae_block_f32_forward": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_float, c_void_p, c_void_p,
                                       ctypes.POINTER(BlockParams), c_void_p, c_void_p, c_void_p]),
    "mmae_block_f32_backward": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p,
                                        ctypes.POINTER(BlockParams), ctypes.POINTER(BlockGrads), c_void_p, c_void_p,
                                        c_void_p]),
    "mmae_dechead_f32_saved_bytes": (c_i64, [ctypes.POINTER(DecoderIndex), c_int, c_int, c_int]),
    "mmae_dechead_f32_workspace_bytes": (c_i64, [ctypes.POINTER(DecoderIndex), c_int, c_int, c_int]),
    "mmae_dechead_f32_forward": (c_int, [c_void_p, c_int, ctypes.POINTER(DecoderIndex), c_int, c_int, c_float,
                                         ctypes.POINTER(DecHeadParams), c_void_p, c_void_p, c_void_p, c_void_p]),
    "mmae_dechead_f32_backward": (c_int, [c_void_p, c_int, ctypes.POINTER(DecoderIndex), c_int, c_int,
                                          ctypes.POINTER(DecHeadParams), ctypes.POINTER(DecHeadGrads), c_void_p, c_void_p,
                                          c_void_p, c_void_p, c_void_p]),
    "mmae_dectail_f32_workspace_bytes": (c_i64, [c_int] * 6),
    "mmae_dectail_f32_forward": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p,
                                         c_void_p, c_void_p]),
    "mmae_dectail_f32_backward": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p,
                                          c_void_p, c_void_p, c_void_p, c_void_p]),
    "mmae_standardize_depth_set_variant": (c_int, [c_int]),
    "mmae_standardize_depth": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_float, c_void_p, c_void_p]),
}

ABI_VERSION = 17


def lib():
    """Load (once) and return the ctypes handle.  Fails loudly when the CUDA library is not built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise MmaeError(
            "multimae_b200: %s is missing - build it with `python -m multimae_b200.build` "
            "(there is no CPU fallback)" % LIB_PATH)
    handle = ctypes.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(handle, name)  # AttributeError if the symbol is not exported
        fn.restype = res
        fn.argtypes = args
    ver = handle.mmae_abi_version()
    if ver != ABI_VERSION:
        raise MmaeError("multimae_b200: ABI version mismatch (library %d, binding %d)" % (ver, ABI_VERSION))
    _lib = handle
    return _lib


def check(rc, what=""):
    if rc != 0:
        msg = lib().mmae_last_error()
        raise MmaeError("%s failed (rc=%d): %s" % (what or "mmae call", rc, (msg or b"").decode()))


def ptr(t):
    """Device pointer of a torch tensor (or None)."""
    return None if t is None else t.data_ptr()


def current_stream():
    import torch
    return torch.cuda.current_stream().cuda_stream

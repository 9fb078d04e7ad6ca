"""ctypes binding of libvitb200.so (include/vitb200.h).  No torch, no numpy-side compute: this module only
marshals pointers and sizes across the C-ABI.  There is NO CPU fallback: if the library is missing it is an
ImportError-style failure, and every entry point fails loudly when no H100 is visible."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("VB_LIB_PATH") or os.path.join(_HERE, "libvitb200.so")   # VB_LIB_PATH: developer A/B builds

KIND = {"vit": 0, "deepvit": 1, "cait": 2, "crossvit": 3, "parallel_vit": 4, "patch_merger_vit": 5, "t2t_vit": 6, "cct": 7, "levit": 8,
        "cvt": 9, "twins_svt": 10, "crossformer": 11, "nest": 12, "regionvit": 13, "ats_vit": 14,
        "small_dataset_vit": 15, "mobilevit": 16, "scalable_vit": 17, "pit": 18, "mae": 19, "simmim": 20, "mpp": 21}
PRECISION = {"fp32": 0, "float32": 0, "bf16": 1, "bfloat16": 1}
MEM_HOST, MEM_DEVICE = 0, 1
ABI_VERSION = 7                     # VB_ABI_VERSION of include/vitb200.h this binding is written against


class VbConfig(C.Structure):
    _fields_ = [(n, C.c_int32) for n in (
        "struct_size", "kind", "precision", "image_h", "image_w", "patch_h", "patch_w", "channels", "num_classes",
        "dim", "depth", "heads", "dim_head", "mlp_dim", "pool", "cls_depth", "max_batch",
        "sm_dim", "lg_dim",
        "sm_patch_size", "sm_enc_depth", "sm_enc_heads", "sm_enc_mlp_dim", "sm_enc_dim_head",
        "lg_patch_size", "lg_enc_depth", "lg_enc_heads", "lg_enc_mlp_dim", "lg_enc_dim_head",
        "cross_attn_depth", "cross_attn_heads", "cross_attn_dim_head", "cross_depth", "parallel_branches",
        "patch_merge_layer_index", "patch_merge_num_tokens",
        "t2t_num_layers", "t2t_k0", "t2t_s0", "t2t_k1", "t2t_s1", "t2t_k2", "t2t_s2", "t2t_k3", "t2t_s3",
        "cct_conv_layers", "cct_kernel", "cct_stride", "cct_pool_kernel", "cct_pool_stride", "cct_pos_emb")]


CONFIG_SIZE_ABI7 = VbConfig.cct_conv_layers.offset   # VB_CONFIG_SIZE_ABI7: the struct before the CCT fields were appended
CCT_POS = {"sine": 0, "learnable": 1, "none": 2}     # VB_CCT_POS_*
LEVIT_MAX_STAGES = 8                                # VB_LEVIT_MAX_STAGES


class VbLevitConfig(C.Structure):
    _fields_ = [("struct_size", C.c_int32), ("stages", C.c_int32), ("dims", C.c_int32 * LEVIT_MAX_STAGES),
                ("depths", C.c_int32 * LEVIT_MAX_STAGES), ("heads", C.c_int32 * LEVIT_MAX_STAGES), ("dim_key", C.c_int32),
                ("dim_value", C.c_int32), ("mlp_mult", C.c_int32), ("num_distill_classes", C.c_int32)]


CVT_STAGES = 3                                      # VB_CVT_STAGES


class VbCvtConfig(C.Structure):
    _fields_ = [("struct_size", C.c_int32)] + [(n, C.c_int32 * CVT_STAGES) for n in (
        "emb_dim", "emb_kernel", "emb_stride", "proj_kernel", "kv_proj_stride", "heads", "depth", "mlp_mult")]


TWINS_STAGES = 4                                    # VB_TWINS_STAGES


class VbTwinsSvtConfig(C.Structure):
    _fields_ = [("struct_size", C.c_int32)] + [(n, C.c_int32 * TWINS_STAGES) for n in (
        "emb_dim", "patch_size", "local_patch_size", "global_k", "depth")] + [("peg_kernel_size", C.c_int32)]


CROSSFORMER_STAGES, CROSSFORMER_MAX_KERNELS = 4, 4  # VB_CROSSFORMER_STAGES, VB_CROSSFORMER_MAX_KERNELS


class VbCrossformerConfig(C.Structure):
    _fields_ = [("struct_size", C.c_int32)] + [(n, C.c_int32 * CROSSFORMER_STAGES) for n in (
        "dim", "depth", "global_wsz", "local_wsz", "stride", "n_kernels")] + [
        ("kernels", (C.c_int32 * CROSSFORMER_MAX_KERNELS) * CROSSFORMER_STAGES)]


NEST_MAX_LEVELS = 8                                  # VB_NEST_MAX_LEVELS


class VbNestConfig(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("struct_size", "patch_size", "dim", "heads", "num_hierarchies", "levels")] + [
        ("block_repeats", C.c_int32 * NEST_MAX_LEVELS), ("mlp_mult", C.c_int32), ("seq_len", C.c_int32)]


REGIONVIT_STAGES = 4                                 # VB_REGIONVIT_STAGES


class VbRegionvitConfig(C.Structure):
    _fields_ = [("struct_size", C.c_int32), ("dims", C.c_int32 * REGIONVIT_STAGES), ("depth", C.c_int32 * REGIONVIT_STAGES)] + [
        (n, C.c_int32) for n in ("window_size", "local_patch_size", "tokenize_local_3_conv", "use_peg", "mlp_mult")]


ATS_MAX_DEPTH = 64                                   # VB_ATS_MAX_DEPTH


class VbAtsVitConfig(C.Structure):
    _fields_ = [("struct_size", C.c_int32), ("max_tokens_per_depth", C.c_int32 * ATS_MAX_DEPTH)]


MOBILEVIT_MV2 = 7                                    # VB_MOBILEVIT_MV2


class VbMobilevitConfig(C.Structure):
    _fields_ = [("struct_size", C.c_int32), ("channels", C.c_int32 * 10), ("last_dim", C.c_int32), ("dims", C.c_int32 * 3),
                ("depths", C.c_int32 * 3), ("kernel_size", C.c_int32), ("ph", C.c_int32), ("pw", C.c_int32)] + \
               [(f, C.c_int32 * MOBILEVIT_MV2) for f in ("mv2_in", "mv2_hidden", "mv2_out", "mv2_stride", "mv2_expand", "mv2_residual")]


SCALABLE_VIT_STAGES = 4                              # VB_SCALABLE_VIT_STAGES


class VbScalableVitConfig(C.Structure):
    _fields_ = ([("struct_size", C.c_int32), ("num_stages", C.c_int32)] +
                [(f, C.c_int32 * SCALABLE_VIT_STAGES) for f in ("dim", "depth", "heads", "ssa_dim_key", "ssa_dim_value", "reduction_factor",
                                                                "iwsa_dim_key", "iwsa_dim_value", "window")] +
                [("ff_expansion_factor", C.c_int32)])


PIT_MAX_STAGES = 8                                   # VB_PIT_MAX_STAGES


class VbPitConfig(C.Structure):
    _fields_ = [("struct_size", C.c_int32), ("stages", C.c_int32), ("depth", C.c_int32 * PIT_MAX_STAGES),
                ("heads", C.c_int32 * PIT_MAX_STAGES)]


MIM_MAX_PATCHES = 4096                               # VB_MIM_MAX_PATCHES


class VbMimConfig(C.Structure):
    _fields_ = [("struct_size", C.c_int32), ("masking_ratio", C.c_double), ("decoder_dim", C.c_int32), ("decoder_depth", C.c_int32),
                ("decoder_heads", C.c_int32), ("decoder_dim_head", C.c_int32)]


class VbMppConfig(VbMimConfig):
    """vb_mpp_config: a vb_mim_config (its struct_size set to this struct's size) followed by MPP's fields."""
    _fields_ = [("mask_prob", C.c_double), ("replace_prob", C.c_double), ("random_patch_prob", C.c_double),
                ("output_channel_bits", C.c_int32)]


class VbError(RuntimeError):
    pass


_f32p = C.POINTER(C.c_float)
_i64p = C.POINTER(C.c_int64)

# name -> (restype, argtypes); must list EVERY symbol include/vitb200.h declares (tests/test_abi.py checks)
SIGNATURES = {
    "vb_abi_version": (C.c_int, []),
    "vb_create": (C.c_int, [C.POINTER(VbConfig), C.c_int, C.POINTER(C.c_void_p)]),
    "vb_create_levit": (C.c_int, [C.POINTER(VbConfig), C.POINTER(VbLevitConfig), C.c_int, C.POINTER(C.c_void_p)]),
    "vb_create_cvt": (C.c_int, [C.POINTER(VbConfig), C.POINTER(VbCvtConfig), C.c_int, C.POINTER(C.c_void_p)]),
    "vb_create_twins_svt": (C.c_int, [C.POINTER(VbConfig), C.POINTER(VbTwinsSvtConfig), C.c_int, C.POINTER(C.c_void_p)]),
    "vb_create_crossformer": (C.c_int, [C.POINTER(VbConfig), C.POINTER(VbCrossformerConfig), C.c_int, C.POINTER(C.c_void_p)]),
    "vb_create_nest": (C.c_int, [C.POINTER(VbConfig), C.POINTER(VbNestConfig), C.c_int, C.POINTER(C.c_void_p)]),
    "vb_create_regionvit": (C.c_int, [C.POINTER(VbConfig), C.POINTER(VbRegionvitConfig), C.c_int, C.POINTER(C.c_void_p)]),
    "vb_create_ats_vit": (C.c_int, [C.POINTER(VbConfig), C.POINTER(VbAtsVitConfig), C.c_int, C.POINTER(C.c_void_p)]),
    "vb_create_mobilevit": (C.c_int, [C.POINTER(VbConfig), C.POINTER(VbMobilevitConfig), C.c_int, C.POINTER(C.c_void_p)]),
    "vb_create_scalable_vit": (C.c_int, [C.POINTER(VbConfig), C.POINTER(VbScalableVitConfig), C.c_int, C.POINTER(C.c_void_p)]),
    "vb_create_pit": (C.c_int, [C.POINTER(VbConfig), C.POINTER(VbPitConfig), C.c_int, C.POINTER(C.c_void_p)]),
    "vb_op_mv2_dwconv": (C.c_int, [C.c_int32, C.c_void_p] + [C.c_int32] * 5 + [C.c_void_p] * 3 + [C.c_int32, _f32p]),
    "vb_op_patch_attention": (C.c_int, [C.c_int32, C.c_void_p] + [C.c_int32] * 8 + [C.c_float, C.c_void_p, C.c_int32, C.c_int32, _f32p]),
    "vb_ats_set_seed": (C.c_int, [C.c_void_p, C.c_uint64]),
    "vb_forward_ats": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p,
                                 C.c_void_p]),
    "vb_ats_last_draws": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]),
    "vb_op_ats_sample": (C.c_int, [C.c_int32, C.c_void_p] + [C.c_int32] * 5 + [C.c_float, C.c_void_p, C.c_int32, C.c_uint64, C.c_uint64] +
                         [C.c_void_p] * 3),
    "vb_op_masked_attention": (C.c_int, [C.c_int32, C.c_void_p] + [C.c_int32] * 5 + [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, _f32p]),
    "vb_op_spt": (C.c_int, [C.c_int32, C.c_void_p] + [C.c_int32] * 5 + [C.c_void_p] * 7),
    "vb_op_lsa_attention": (C.c_int, [C.c_int32, C.c_void_p] + [C.c_int32] * 5 + [C.c_float, C.c_void_p, C.c_int32, C.c_int32, _f32p]),
    "vb_create_mim": (C.c_int, [C.POINTER(VbConfig), C.POINTER(VbMimConfig), C.c_int, C.POINTER(C.c_void_p)]),
    "vb_mim_set_seed": (C.c_int, [C.c_void_p, C.c_uint64]),
    "vb_forward_mim": (C.c_int, [C.c_void_p, C.c_void_p] + [C.c_int32] * 4 + [C.c_void_p] * 4 + [C.c_int32, C.c_void_p]),
    "vb_op_mim_mask": (C.c_int, [C.c_int32, C.c_int32, C.c_int32, C.c_uint64, C.c_uint64, C.c_void_p]),
    "vb_forward_mpp": (C.c_int, [C.c_void_p, C.c_void_p] + [C.c_int32] * 4 + [C.c_void_p] * 4 + [C.c_int32, C.c_void_p]),
    "vb_op_mpp_draws": (C.c_int, [C.c_int32] * 3 + [C.c_double, C.c_double, C.c_uint64, C.c_uint64, C.c_void_p, C.c_void_p]),
    "vb_create_distill": (C.c_int, [C.POINTER(VbConfig), C.c_int, C.POINTER(C.c_void_p)]),
    "vb_forward_distill_loss": (C.c_int, [C.c_void_p, C.c_void_p] + [C.c_int32] * 4 + [C.c_void_p] * 3 +
                                [C.c_int32, C.c_double, C.c_double] + [C.c_void_p] * 4 + [C.c_int32, C.c_void_p]),
    "vb_op_distill_loss": (C.c_int, [C.c_void_p] * 3 + [C.c_int32, C.c_int32, C.c_double, C.c_double, C.c_void_p]),
    "vb_set_dropout": (C.c_int, [C.c_void_p, C.c_float, C.c_float, C.c_uint64]),
    "vb_forward_train": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p]),
    "vb_op_dropout_mask": (C.c_int, [C.c_uint64, C.c_uint32, C.c_uint32, C.c_int32, C.c_int32, C.c_float, C.c_void_p]),
    "vb_set_weight": (C.c_int, [C.c_void_p, C.c_char_p, C.c_void_p, _i64p, C.c_int32]),
    "vb_num_weights": (C.c_int, [C.c_void_p]),
    "vb_weight_info": (C.c_int, [C.c_void_p, C.c_int32, C.POINTER(C.c_char_p), _i64p, C.POINTER(C.c_int32)]),
    "vb_finalize": (C.c_int, [C.c_void_p]),
    "vb_forward": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p]),
    "vb_forward_tokens": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p]),
    "vb_forward_distill": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p,
                                     C.c_void_p, C.c_int32, C.c_void_p]),
    "vb_embed_rows": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32]),
    "vb_forward_embed": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p]),
    "vb_forward_head": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p]),
    "vb_to_patch": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p]),
    "vb_patch_to_emb": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p]),
    "vb_dp_unique_id": (C.c_int, [C.c_void_p]),
    "vb_dp_init": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32]),
    "vb_forward_allgather": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]),
    "vb_last_launch_count": (C.c_int64, [C.c_void_p]),
    "vb_graph_stats": (C.c_int, [C.c_void_p, _i64p, _i64p, _i64p, C.POINTER(C.c_char_p)]),
    "vb_last_attention_path": (C.c_int32, []),
    "vb_profile_enable": (C.c_int, [C.c_void_p, C.c_int32]),
    "vb_profile_read": (C.c_int, [C.c_void_p, C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(C.c_double), _i64p, C.c_int32]),
    "vb_last_error": (C.c_char_p, [C.c_void_p]),
    "vb_destroy": (None, [C.c_void_p]),
    "vb_op_linear": (C.c_int, [C.c_int32] + [C.c_void_p] * 5 + [C.c_int32, C.c_void_p] + [C.c_int32] * 4 + [_f32p]),
    "vb_op_attention": (C.c_int, [C.c_int32, C.c_int32] + [C.c_void_p] * 8 + [C.c_int32] * 6 + [_f32p]),
    "vb_op_layernorm": (C.c_int, [C.c_int32] + [C.c_void_p] * 4 + [C.c_int32] * 3 + [_f32p]),
    "vb_op_patch_merger": (C.c_int, [C.c_int32] + [C.c_void_p] * 5 + [C.c_int32] * 5 + [_f32p]),
    "vb_op_ln_linear": (C.c_int, [C.c_void_p] * 5 + [C.c_int32, C.c_void_p] + [C.c_int32] * 4 + [_f32p]),
    "vb_op_gemm": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p,
                             C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p] + [C.c_int32] * 3 + [C.c_void_p] + [C.c_int32] * 4 + [_f32p]),
    "vb_op_attention_ex": (C.c_int, [C.c_int32, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p] + [C.c_int32] * 3 + [C.c_void_p] * 5 +
                           [C.c_int32] * 6 + [C.c_float, C.c_int32, _f32p]),
    "vb_op_attention_bias": (C.c_int, [C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p,
                                       C.c_void_p] + [C.c_int32] * 6 + [C.c_float, C.c_int32, C.c_int32, _f32p]),
    "vb_op_dwconv": (C.c_int, [C.c_int32, C.c_void_p] + [C.c_int32] * 4 + [C.c_void_p] * 2 + [C.c_int32] * 2 + [C.c_void_p] * 6 +
                     [C.c_int32, _f32p]),
    "vb_op_window_attention": (C.c_int, [C.c_int32, C.c_void_p] + [C.c_int32] * 7 + [C.c_void_p, C.c_int32, C.c_int32, _f32p]),
    "vb_op_window_bias_attention": (C.c_int, [C.c_int32, C.c_void_p] + [C.c_int32] * 8 + [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32,
                                                                                           _f32p]),
    "vb_op_block_attention": (C.c_int, [C.c_int32, C.c_void_p] + [C.c_int32] * 8 + [C.c_void_p, C.c_int32, C.c_int32, _f32p]),
    "vb_op_nest_aggregate": (C.c_int, [C.c_int32, C.c_void_p] + [C.c_int32] * 4 + [C.c_void_p] * 3 + [C.c_int32] * 2 +
                             [C.c_void_p, C.c_void_p, C.c_int32, _f32p]),
    "vb_op_r2l_attention": (C.c_int, [C.c_int32, C.c_void_p] + [C.c_int32] * 8 + [C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_int32,
                                                                                   _f32p]),
    "vb_op_conv2d": (C.c_int, [C.c_int32, C.c_void_p] + [C.c_int32] * 7 + [C.c_void_p] * 2 + [C.c_int32] * 4 + [C.c_void_p] * 2 +
                     [C.c_float, C.c_int32, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_int32, _f32p]),
    "vb_op_cct_pool": (C.c_int, [C.c_int32, C.c_void_p] + [C.c_int32] * 6 + [C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, _f32p]),
    "vb_op_seq_pool": (C.c_int, [C.c_int32, C.c_void_p] + [C.c_int32] * 3 + [C.c_void_p] * 5 + [C.c_int32, _f32p]),
    "vb_op_pool_layernorm": (C.c_int, [C.c_int32, C.c_void_p] + [C.c_int32] * 4 + [C.c_void_p] * 2 + [C.c_int32, C.c_void_p, C.c_int32,
                                                                                                     _f32p]),
    "vb_op_gather_grid": (C.c_int, [C.c_int32, C.c_void_p] + [C.c_int32] * 6 + [C.c_void_p, C.c_int32, C.c_int32, _f32p]),
    "vb_op_softmax_rows": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p] + [C.c_int32] * 4 + [C.c_float, C.c_int32, _f32p]),
}

_lib = None


def load() -> C.CDLL:
    """Load libvitb200.so (building is `python -m vit_tensorflow_b200.build` / __graft_entry__.build())."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise VbError(f"{LIB_PATH} not found: build it with `python -m vit_tensorflow_b200.build` "
                          "(there is no CPU / PyTorch fallback)")
        lib = C.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(lib, name)
            fn.restype = res
            fn.argtypes = args
        if lib.vb_abi_version() != ABI_VERSION:
            raise VbError("libvitb200 ABI version mismatch")
        _lib = lib
    return _lib


ATTENTION_PATHS = {0: None, 1: "flash", 2: "cls", 3: "rows", 4: "mid_fused", 5: "simt"}   # VB_ATTN_PATH_* of include/vitb200.h


def last_attention_path():
    """The attention branch ("flash", "cls", "rows", "mid_fused" or "simt") that served the most recent attention call of this
    thread since the previous last_attention_path() call, or None (vb_last_attention_path; reading it resets it)."""
    return ATTENTION_PATHS[load().vb_last_attention_path()]


def check(rc: int, handle=None):
    if rc != 0:
        msg = load().vb_last_error(handle)
        raise VbError(f"libvitb200 error {rc}: {msg.decode() if msg else '?'}")


def _ptr(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _f32(a):
    return None if a is None else np.ascontiguousarray(a, dtype=np.float32)


# ---------------------------------------------------------------------------- single-operator helpers
def op_linear(a, w, bias=None, scale=None, res=None, gelu=False, precision="bf16", iters=0):
    """out = epi(a @ w); returns (out float32 [M,N], ms per launch or None)."""
    a, w, bias, scale, res = map(_f32, (a, w, bias, scale, res))
    M, K = a.shape
    K2, N = w.shape
    assert K == K2
    out = np.empty((M, N), np.float32)
    ms = C.c_float(0)
    check(load().vb_op_linear(PRECISION[precision], _ptr(a), _ptr(w), _ptr(bias), _ptr(scale), _ptr(res), int(bool(gelu)),
                              _ptr(out), M, N, K, iters, C.byref(ms)))
    return out, (ms.value if iters > 0 else None)


def op_attention(q, k, v, heads, variant=0, mix_a=None, mix_b=None, ln_gamma=None, ln_beta=None, precision="bf16", iters=0):
    q, k, v, mix_a, mix_b, ln_gamma, ln_beta = map(_f32, (q, k, v, mix_a, mix_b, ln_gamma, ln_beta))
    B, nq, inner = q.shape
    nk = k.shape[1]
    out = np.empty_like(q)
    ms = C.c_float(0)
    check(load().vb_op_attention(PRECISION[precision], variant, _ptr(q), _ptr(k), _ptr(v), _ptr(mix_a), _ptr(mix_b),
                                 _ptr(ln_gamma), _ptr(ln_beta), _ptr(out), B, nq, nk, heads, inner // heads, iters, C.byref(ms)))
    return out, (ms.value if iters > 0 else None)


def op_layernorm(x, gamma, beta, precision="bf16", iters=0):
    x, gamma, beta = map(_f32, (x, gamma, beta))
    M, D = x.shape
    out = np.empty_like(x)
    ms = C.c_float(0)
    check(load().vb_op_layernorm(PRECISION[precision], _ptr(x), _ptr(gamma), _ptr(beta), _ptr(out), M, D, iters, C.byref(ms)))
    return out, (ms.value if iters > 0 else None)


def op_ln_linear(x, gamma, beta, w, bias=None, gelu=False, iters=0):
    """out = act(LayerNorm(x) @ w + bias) through the LayerNorm-folded wgmma GEMM (bf16 engine); returns (out, ms)."""
    x, gamma, beta, w, bias = map(_f32, (x, gamma, beta, w, bias))
    M, K = x.shape
    N = w.shape[1]
    out = np.empty((M, N), np.float32)
    ms = C.c_float(0)
    check(load().vb_op_ln_linear(_ptr(x), _ptr(gamma), _ptr(beta), _ptr(w), _ptr(bias), int(bool(gelu)), _ptr(out), M, N, K, iters,
                                 C.byref(ms)))
    return out, (ms.value if iters > 0 else None)


def op_gemm(a, wt, N, K, out, bias=None, scale=None, gelu=False, res=None, out_off=0, out_f32=False, ln_stats=None, ln_c1=None,
            want_stats=False, iters=0, silu=False):
    """The bf16 wgmma GEMM in the engine's operand layouts (vb_op_gemm): a [M, lda], wt K-major [b_rows, ldw] (b_rows < N: the
    missing rows read as zero), out [M, ldc] initial contents (columns [out_off, out_off + N) are written); res: None, a
    separate [M, ldr] array, or the string "out" for the in-place residual; silu: the SiLU epilogue instead of GELU.  Returns (out
    [M, ldc], stats [N/64, M, 2] or None, ms per launch or None)."""
    a, wt, bias, scale, ln_stats, ln_c1 = map(_f32, (a, wt, bias, scale, ln_stats, ln_c1))
    out = np.array(out, dtype=np.float32, order="C", copy=True)
    M, lda = a.shape
    b_rows, ldw = wt.shape
    ldc = out.shape[1]
    if isinstance(res, str):
        assert res == "out"
        res_p, ldr = _ptr(out), ldc
    else:
        res = _f32(res)
        res_p, ldr = _ptr(res), (0 if res is None else res.shape[1])
    stats = np.empty((N // 64, M, 2), np.float32) if want_stats else None
    ms = C.c_float(0)
    act = 3 if silu else int(bool(gelu))                 # Act: ACT_SILU = 3, ACT_GELU = 1
    check(load().vb_op_gemm(_ptr(a), lda, _ptr(wt), ldw, b_rows, _ptr(bias), _ptr(scale), act, res_p, ldr, _ptr(ln_stats),
                            _ptr(ln_c1), _ptr(out), ldc, out_off, int(bool(out_f32)), _ptr(stats), M, N, K, iters, C.byref(ms)))
    return out, stats, (ms.value if iters > 0 else None)


def op_attention_ex(q, heads, dh, out, kv=None, k_off=0, v_off=0, variant=0, mix_a=None, mix_b=None, ln_gamma=None,
                    ln_beta=None, scale=0.0, precision="bf16", iters=0):
    """Attention in the engine's layouts (vb_op_attention_ex): q [B, nq, ldq]; kv None (k, v at columns k_off / v_off of the q rows)
    or [B, nk, ldkv]; out [B, nq, ldo] initial contents, returned whole.  scale <= 0: dh^-0.5.  Returns (out, ms or None)."""
    q, kv, mix_a, mix_b, ln_gamma, ln_beta = map(_f32, (q, kv, mix_a, mix_b, ln_gamma, ln_beta))
    out = np.array(out, dtype=np.float32, order="C", copy=True)
    B, nq, ldq = q.shape
    nk = nq if kv is None else kv.shape[1]
    ldkv = 0 if kv is None else kv.shape[2]
    ms = C.c_float(0)
    check(load().vb_op_attention_ex(PRECISION[precision], variant, _ptr(q), ldq, _ptr(kv), ldkv, k_off, v_off, _ptr(mix_a), _ptr(mix_b),
                                    _ptr(ln_gamma), _ptr(ln_beta), _ptr(out), out.shape[2], B, nq, nk, heads, dh, float(scale), iters,
                                    C.byref(ms)))
    return out, (ms.value if iters > 0 else None)


def op_attention_bias(q, k, v, pos_bias, heads, dh, fmap, q_step, scale, out, gelu_out=True, precision="bf16", iters=0):
    """LeViT attention (vb_op_attention_bias): q [B, nq, ldq], k / v [B, fmap^2, ld], pos_bias the Embedding table [fmap^2, heads],
    out [B, nq, ldo] initial contents, returned whole.  Returns (out, ms or None)."""
    q, k, v, pos_bias = map(_f32, (q, k, v, pos_bias))
    out = np.array(out, dtype=np.float32, order="C", copy=True)
    B = q.shape[0]
    ms = C.c_float(0)
    check(load().vb_op_attention_bias(PRECISION[precision], _ptr(q), q.shape[2], _ptr(k), k.shape[2], _ptr(v), v.shape[2], _ptr(pos_bias),
                                      _ptr(out), out.shape[2], B, heads, dh, fmap, q_step, float(scale), int(bool(gelu_out)), iters,
                                      C.byref(ms)))
    return out, (ms.value if iters > 0 else None)


def op_dwconv(x, ln_gamma, ln_beta, wq, bn_q, wkv, bn_kv, kv_stride, precision="bf16", iters=0):
    """CvT's depthwise q / k|v projections (vb_op_dwconv): x [B, H, W, C], the depthwise kernels [k, k, 1, C], the
    BatchNormalizations [4, C] (gamma, beta, moving_mean, moving_variance).  Returns (q [B, H, W, C], kv [B, ceil(H/s),
    ceil(W/s), C], ms or None)."""
    x, ln_gamma, ln_beta, wq, bn_q, wkv, bn_kv = map(_f32, (x, ln_gamma, ln_beta, wq, bn_q, wkv, bn_kv))
    B, H, W, Cc = x.shape
    k = wq.shape[0]
    q = np.empty((B, H, W, Cc), np.float32)
    kv = np.empty((B, -(-H // kv_stride), -(-W // kv_stride), Cc), np.float32)
    ms = C.c_float(0)
    check(load().vb_op_dwconv(PRECISION[precision], _ptr(x), B, H, W, Cc, _ptr(ln_gamma), _ptr(ln_beta), k, kv_stride, _ptr(wq),
                              _ptr(bn_q), _ptr(wkv), _ptr(bn_kv), _ptr(q), _ptr(kv), iters, C.byref(ms)))
    return q, kv, (ms.value if iters > 0 else None)


def op_window_attention(qkv, H, W, p, heads, dh, precision="bf16", iters=0):
    """Twins-SVT's local attention (vb_op_window_attention): qkv [B*H*W, ld] fused q|k|v rows of a pixel-major map.  Returns
    (out [B*H*W, heads*dh] pixel-major, ms or None)."""
    qkv = _f32(qkv)
    rows, ld = qkv.shape
    B = rows // (H * W)
    out = np.zeros((rows, heads * dh), np.float32)
    ms = C.c_float(0)
    check(load().vb_op_window_attention(PRECISION[precision], _ptr(qkv), ld, B, H, W, p, heads, dh, _ptr(out), heads * dh, iters,
                                        C.byref(ms)))
    return out, (ms.value if iters > 0 else None)


def op_window_bias_attention(qkv, H, W, wsz, is_long, heads, dh, table, precision="bf16", iters=0):
    """CrossFormer's attention (vb_op_window_bias_attention): qkv [B*H*W, ld] fused q|k|v rows of a pixel-major map, table the
    (2 wsz - 1)^2 window table.  Returns (out [B*H*W, heads*dh] pixel-major, ms or None)."""
    qkv, table = _f32(qkv), _f32(table)
    rows, ld = qkv.shape
    B = rows // (H * W)
    out = np.zeros((rows, heads * dh), np.float32)
    ms = C.c_float(0)
    check(load().vb_op_window_bias_attention(PRECISION[precision], _ptr(qkv), ld, B, H, W, wsz, int(bool(is_long)), heads, dh, _ptr(table),
                                             _ptr(out), heads * dh, iters, C.byref(ms)))
    return out, (ms.value if iters > 0 else None)


def op_block_attention(qkv, H, W, bh, bw, heads, dh, precision="bf16", iters=0):
    """NesT's block attention (vb_op_block_attention): qkv [B*H*W, ld] fused q|k|v rows of a pixel-major map, attention within
    each bh x bw block.  Returns (out [B*H*W, heads*dh] pixel-major, ms or None)."""
    qkv = _f32(qkv)
    rows, ld = qkv.shape
    B = rows // (H * W)
    out = np.zeros((rows, heads * dh), np.float32)
    ms = C.c_float(0)
    check(load().vb_op_block_attention(PRECISION[precision], _ptr(qkv), ld, B, H, W, bh, bw, heads, dh, _ptr(out), heads * dh, iters,
                                       C.byref(ms)))
    return out, (ms.value if iters > 0 else None)


def op_mv2_dwconv(x, w, bn, stride, precision="bf16", iters=0):
    """MobileViT's MV2 depthwise step (vb_op_mv2_dwconv): x [B, H, W, C], the depthwise kernel [3, 3, 1, C], the BatchNormalization
    [4, C] (gamma, beta, moving_mean, moving_variance).  Returns (out [B, ceil(H/s), ceil(W/s), Cp] with Cp = C (fp32) or C rounded
    up to a multiple of 64 (bf16), ms or None)."""
    x, w, bn = map(_f32, (x, w, bn))
    B, H, W, Cc = x.shape
    cp = Cc if PRECISION[precision] == 0 else -(-Cc // 64) * 64
    out = np.empty((B, -(-H // stride), -(-W // stride), cp), np.float32)
    ms = C.c_float(0)
    check(load().vb_op_mv2_dwconv(PRECISION[precision], _ptr(x), B, H, W, Cc, stride, _ptr(w), _ptr(bn), _ptr(out), iters, C.byref(ms)))
    return out, (ms.value if iters > 0 else None)


def op_patch_attention(qkv, H, W, ph, pw, heads, dh, scale=0.0, precision="bf16", iters=0):
    """MobileViT's attention (vb_op_patch_attention): qkv [B*H*W, ld] fused q|k|v rows of a pixel-major map; the pixels of one
    patch position (y % ph, x % pw) attend together.  Returns (out [B*H*W, heads*dh] pixel-major, ms or None)."""
    qkv = _f32(qkv)
    rows, ld = qkv.shape
    B = rows // (H * W)
    out = np.zeros((rows, heads * dh), np.float32)
    ms = C.c_float(0)
    check(load().vb_op_patch_attention(PRECISION[precision], _ptr(qkv), ld, B, H, W, ph, pw, heads, dh, float(scale), _ptr(out), heads * dh,
                                       iters, C.byref(ms)))
    return out, (ms.value if iters > 0 else None)


def op_nest_aggregate(x, gamma, beta, pos=None, bh=1, bw=1, precision="bf16", iters=0):
    """NesT's aggregation tail (vb_op_nest_aggregate): x [B, H, W, C] -> LayerNorm (eps 1e-5) -> MaxPool2D(3, 2, SAME) -> + pos
    [bh * bw] per in-block position.  Returns (out [B, ceil(H/2), ceil(W/2), C], stats [ceil(C/64), rows, 2] of the bf16 rows
    (None in fp32), ms or None)."""
    x, gamma, beta = map(_f32, (x, gamma, beta))
    B, H, W, Cc = x.shape
    Ho, Wo = -(-H // 2), -(-W // 2)
    out = np.empty((B, Ho, Wo, Cc), np.float32)
    bf = PRECISION[precision] == PRECISION["bf16"]
    stats = np.zeros((-(-Cc // 64), B * Ho * Wo, 2), np.float32) if bf else None
    pos = _f32(pos)
    ms = C.c_float(0)
    check(load().vb_op_nest_aggregate(PRECISION[precision], _ptr(x), B, H, W, Cc, _ptr(gamma), _ptr(beta), _ptr(pos), bh, bw, _ptr(out),
                                      _ptr(stats) if stats is not None else None, iters, C.byref(ms)))
    return out, stats, (ms.value if iters > 0 else None)


ACT = {"none": 0, "gelu": 1, "hswish": 2, "silu": 3}   # Act of csrc/common.h


def op_conv2d(x, kernel, bias=None, stride=1, valid=False, image=False, HW=None, cin=None, off=0, ln_gamma=None, ln_beta=None,
              ln_eps=1e-5, gelu_in=False, act="none", res=None, want_stats=False, precision="bf16", iters=0):
    """A Conv2D as the engine runs it (vb_op_conv2d): unfold_same, then the GEMM.  x: image=True, an NHWC image [B, H, W, cin];
    else a token map [B*H*W, ld] with HW = (B, H, W) and the channels at columns [off, off + cin).  kernel [k, k, cin, N] (Keras).
    Returns (out [B*oh*ow, N], stats [N/64, rows, 2] of the bf16 rows or None, ms or None)."""
    x, kernel, bias, ln_gamma, ln_beta, res = map(_f32, (x, kernel, bias, ln_gamma, ln_beta, res))
    k, _, kc, N = kernel.shape
    if image:
        B, H, W, ld = x.shape
        cin = ld
    else:
        B, H, W = HW
        ld = x.shape[1]
        cin = kc if cin is None else cin
    oh, ow = ((H - k) // stride + 1, (W - k) // stride + 1) if valid else (-(-H // stride), -(-W // stride))
    rows = B * oh * ow
    out = np.empty((rows, N), np.float32)
    stats = np.zeros((N // 64, rows, 2), np.float32) if want_stats else None
    ms = C.c_float(0)
    check(load().vb_op_conv2d(PRECISION[precision], _ptr(x), int(bool(image)), B, H, W, cin, ld, off, _ptr(kernel), _ptr(bias), N, k,
                              stride, int(bool(valid)), _ptr(ln_gamma), _ptr(ln_beta), float(ln_eps), int(bool(gelu_in)), ACT[act],
                              _ptr(res), 0 if res is None else res.shape[1], _ptr(out), _ptr(stats), iters, C.byref(ms)))
    return out, stats, (ms.value if iters > 0 else None)


def op_cct_pool(x, k, stride, pos=None, rows=None, precision="bf16", iters=0):
    """CCT's ReLU + MaxPool2D(k, stride, SAME) + positions (vb_op_cct_pool): x [B, H, W, C] -> (out [B, rows, C], ms or None);
    rows None: oh * ow."""
    x, pos = _f32(x), _f32(pos)
    B, H, W, Cc = x.shape
    rows = -(-H // stride) * -(-W // stride) if rows is None else rows
    out = np.empty((B, rows, Cc), np.float32)
    ms = C.c_float(0)
    check(load().vb_op_cct_pool(PRECISION[precision], _ptr(x), B, H, W, Cc, k, stride, _ptr(pos), rows, _ptr(out), iters, C.byref(ms)))
    return out, (ms.value if iters > 0 else None)


def op_seq_pool(x, gamma, beta, pw, pb, precision="bf16", iters=0):
    """CCT's sequence pooling (vb_op_seq_pool): x [B, n, D], pw [D], pb scalar -> (z [B, D], ms or None)."""
    x, gamma, beta, pw = map(_f32, (x, gamma, beta, pw))
    pb = np.asarray([pb], np.float32).reshape(1)
    B, n, D = x.shape
    z = np.empty((B, D), np.float32)
    ms = C.c_float(0)
    check(load().vb_op_seq_pool(PRECISION[precision], _ptr(x), B, n, D, _ptr(gamma), _ptr(beta), _ptr(pw), _ptr(pb), _ptr(z), iters,
                                C.byref(ms)))
    return z, (ms.value if iters > 0 else None)


def op_pool_layernorm(x, D, gamma=None, beta=None, mean=False, precision="bf16", iters=0):
    """The heads' pooling (vb_op_pool_layernorm): x [B, n, ldx] -> (z [B, D] = LayerNorm(row 0 or the mean of the rows' first D
    columns), ms or None); gamma / beta None: the pool alone."""
    x, gamma, beta = map(_f32, (x, gamma, beta))
    B, n, ldx = x.shape
    z = np.empty((B, D), np.float32)
    ms = C.c_float(0)
    check(load().vb_op_pool_layernorm(PRECISION[precision], _ptr(x), B, n, ldx, D, _ptr(gamma), _ptr(beta), int(bool(mean)), _ptr(z),
                                      iters, C.byref(ms)))
    return z, (ms.value if iters > 0 else None)


def op_gather_grid(x, B, H, W, C_, step, out, precision="bf16", iters=0):
    """LeViT's strided query gather (vb_op_gather_grid): x [B*H*W, ldi], out [B*ceil(H/step)*ceil(W/step), ldo] initial contents,
    returned whole with the first C_ columns of pixel (step r, step c) in row (r, c)."""
    x = _f32(x)
    out = np.array(out, dtype=np.float32, order="C", copy=True)
    ms = C.c_float(0)
    check(load().vb_op_gather_grid(PRECISION[precision], _ptr(x), x.shape[1], B, H, W, C_, step, _ptr(out), out.shape[1], iters,
                                   C.byref(ms)))
    return out, (ms.value if iters > 0 else None)


def op_r2l_attention(qkv, B, lh, lw, rh, rw, heads, dh, table, window_size, precision="bf16", ldo=None, iters=0):
    """RegionViT's regional-to-local attention (vb_op_r2l_attention): qkv [B*lh*lw + B*rh*rw, ld] fused q|k|v rows, the local map's
    then the region map's, table [(2 ws - 1)^2, heads] (the reference's Embedding).  Returns (out [rows, ldo], ms or None)."""
    qkv, table = _f32(qkv), _f32(table)
    rows, ld = qkv.shape
    ldo = heads * dh if ldo is None else ldo
    out = np.zeros((rows, ldo), np.float32)
    ms = C.c_float(0)
    check(load().vb_op_r2l_attention(PRECISION[precision], _ptr(qkv), ld, B, lh, lw, rh, rw, heads, dh, _ptr(table), window_size, _ptr(out),
                                     ldo, iters, C.byref(ms)))
    return out, (ms.value if iters > 0 else None)


def op_ats_sample(qkv, B, P, heads, dh, scale, rows, K, seed=0, counter=0, precision="bf16"):
    """ATS-ViT's sampling step (vb_op_ats_sample) on fused q|k|v rows [B*P, ld] of images with rows[b] live rows.  Returns
    (sel [B, 1 + min(P - 1, K)], rows_new [B], draws [B, K])."""
    qkv = _f32(qkv)
    rows = np.ascontiguousarray(rows, np.int32)
    Pn = 1 + min(P - 1, K)
    sel, rows_new, draws = np.zeros((B, Pn), np.int32), np.zeros(B, np.int32), np.zeros((B, K), np.int32)
    check(load().vb_op_ats_sample(PRECISION[precision], _ptr(qkv), qkv.shape[1], B, P, heads, dh, scale, _ptr(rows), K, seed, counter,
                                  _ptr(sel), _ptr(rows_new), _ptr(draws)))
    return sel, rows_new, draws


def op_masked_attention(qkv, B, n, heads, dh, nk_img, precision="bf16", iters=0):
    """Attention with a key count per image (vb_op_masked_attention): qkv [B*n, ld] fused q|k|v rows.  Returns (out [B*n, heads*dh],
    ms or None)."""
    qkv = _f32(qkv)
    nk = np.ascontiguousarray(nk_img, np.int32)
    out = np.zeros((B * n, heads * dh), np.float32)
    ms = C.c_float(0)
    check(load().vb_op_masked_attention(PRECISION[precision], _ptr(qkv), qkv.shape[1], B, n, heads, dh, _ptr(nk), _ptr(out), heads * dh,
                                        iters, C.byref(ms)))
    return out, (ms.value if iters > 0 else None)


def op_spt(img, p, gamma, beta, kernel, bias, cls=None, pos=None, precision="bf16"):
    """The small-dataset ViT's SPT plus cls row and positions (vb_op_spt): img [B, H, W, 3] -> [B, 1 + np, dim], row 0 = cls + pos[0],
    row 1 + t = Dense(LayerNorm(shifted patch t)) + pos[1 + t]; cls / pos None: zero."""
    img = _f32(img)
    B, H, W, _ = img.shape
    kernel = _f32(kernel)
    dim = kernel.shape[1]
    rows = 1 + (H // p) * (W // p)
    out = np.zeros((B, rows, dim), np.float32)
    opt = [None if a is None else _f32(a) for a in (cls, pos)]
    check(load().vb_op_spt(PRECISION[precision], _ptr(img), B, H, W, p, dim, _ptr(_f32(gamma)), _ptr(_f32(beta)), _ptr(kernel),
                           _ptr(_f32(bias)), *[None if a is None else _ptr(a) for a in opt], _ptr(out)))
    return out


def op_lsa_attention(qkv, B, n, heads, dh, scale, precision="bf16", iters=0):
    """Locality self-attention (vb_op_lsa_attention) on fused q|k|v rows [B*n, ld]: the diagonal masked, scores times `scale`.
    Returns (out [B*n, heads*dh], ms or None)."""
    qkv = _f32(qkv)
    out = np.zeros((B * n, heads * dh), np.float32)
    ms = C.c_float(0)
    check(load().vb_op_lsa_attention(PRECISION[precision], _ptr(qkv), qkv.shape[1], B, n, heads, dh, scale, _ptr(out), heads * dh, iters,
                                     C.byref(ms)))
    return out, (ms.value if iters > 0 else None)


def op_softmax_rows(s, n, npad, scale, p, iters=0):
    """softmax_rows_bf16 (vb_op_softmax_rows): s [rows, lds] fp32 scores, p [rows, ldp] initial contents; returns (p, ms or None)."""
    s = _f32(s)
    p = np.array(p, dtype=np.float32, order="C", copy=True)
    ms = C.c_float(0)
    check(load().vb_op_softmax_rows(_ptr(s), s.shape[1], _ptr(p), p.shape[1], s.shape[0], n, npad, float(scale), iters, C.byref(ms)))
    return p, (ms.value if iters > 0 else None)


def op_patch_merger(x, gamma, beta, queries, precision="bf16", iters=0):
    """PatchMerger.call (vit_with_patch_merger.py:49-55): x [B, n, D], queries [nt, D] -> [B, nt, D]."""
    x, gamma, beta, queries = map(_f32, (x, gamma, beta, queries))
    B, n, D = x.shape
    nt = queries.shape[0]
    out = np.empty((B, nt, D), np.float32)
    ms = C.c_float(0)
    check(load().vb_op_patch_merger(PRECISION[precision], _ptr(x), _ptr(gamma), _ptr(beta), _ptr(queries), _ptr(out), B, n, D, nt,
                                    iters, C.byref(ms)))
    return out, (ms.value if iters > 0 else None)


def op_mim_mask(B, n, seed=0, counter=0, descending=False):
    """The MAE / SimMIM mask kernel on its own (vb_op_mim_mask): indices int32 [B, n], each image's noise permutation with the
    masked ids first (descending: SimMIM's top_k order, else MAE's argsort order)."""
    out = np.zeros((B, n), np.int32)
    check(load().vb_op_mim_mask(int(bool(descending)), B, n, int(seed) & 0xFFFFFFFFFFFFFFFF, int(counter) & 0xFFFFFFFFFFFFFFFF, _ptr(out)))
    return out


def op_mpp_draws(B, n, k, replace_prob, random_patch_prob, seed=0, counter=0):
    """MPP's draws on their own (vb_op_mpp_draws): (mask_ids int32 [B, k] ascending, source int32 [B, n]: j, the random patch id,
    or -1 for the mask token)."""
    ids, src = np.empty((B, k), np.int32), np.empty((B, n), np.int32)
    check(load().vb_op_mpp_draws(B, n, k, float(replace_prob), float(random_patch_prob), int(seed) & 0xFFFFFFFFFFFFFFFF,
                                 int(counter) & 0xFFFFFFFFFFFFFFFF, _ptr(ids), _ptr(src)))
    return ids, src


def op_distill_loss(student_logits, labels, teacher_logits, temperature, alpha):
    """DistillWrapper's loss kernels on their own (vb_op_distill_loss): float32 [B, K] rows -> the loss float32 [B]."""
    s, y, t = (np.ascontiguousarray(a, dtype=np.float32) for a in (student_logits, labels, teacher_logits))
    if s.ndim != 2 or y.shape != s.shape or t.shape != s.shape:
        raise ValueError(f"op_distill_loss: student_logits, labels and teacher_logits must be [B, K] alike, got {s.shape}, {y.shape}, "
                         f"{t.shape}")
    out = np.empty(s.shape[0], np.float32)
    check(load().vb_op_distill_loss(_ptr(s), _ptr(y), _ptr(t), s.shape[0], s.shape[1], float(temperature), float(alpha), _ptr(out)))
    return out


def op_dropout_mask(seed, draw, site, M, N, rate):
    """The training-mode dropout stream on its own (vb_op_dropout_mask): keep uint8 [M, N] of site `site` at draw `draw`."""
    out = np.zeros((M, N), np.uint8)
    check(load().vb_op_dropout_mask(int(seed) & 0xFFFFFFFFFFFFFFFF, int(draw) & 0xFFFFFFFF, int(site) & 0xFFFFFFFF, M, N, float(rate),
                                    _ptr(out)))
    return out

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
        "cvt": 9, "twins_svt": 10, "crossformer": 11}
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
            want_stats=False, iters=0):
    """The bf16 wgmma GEMM in the engine's operand layouts (vb_op_gemm): a [M, lda], wt K-major [b_rows, ldw] (b_rows < N: the
    missing rows read as zero), out [M, ldc] initial contents (columns [out_off, out_off + N) are written); res: None, a
    separate [M, ldr] array, or the string "out" for the in-place residual.  Returns (out [M, ldc], stats [N/64, M, 2] or None,
    ms per launch or None)."""
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
    check(load().vb_op_gemm(_ptr(a), lda, _ptr(wt), ldw, b_rows, _ptr(bias), _ptr(scale), int(bool(gelu)), res_p, ldr, _ptr(ln_stats),
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

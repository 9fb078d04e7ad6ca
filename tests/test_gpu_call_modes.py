"""GPU parity tests of the wgmma GEMM, the attention kernels and the T2T row softmax in the operand layouts the engine calls
them with (vb_op_gemm, vb_op_attention_ex, vb_op_softmax_rows): strided operands, column-offset and in-place outputs,
fp32 output with zero-filled weight rows, epilogue row statistics feeding a LayerNorm-folded GEMM, fused [q|k|v] rows,
head-padded attention, and batch x heads beyond 65 535.  References are float64 numpy on the same bf16-rounded operands,
with the bounds of test_gpu_ops.py."""
import numpy as np
import pytest

from cases import bf16_round
from test_gpu_ops import (ATTN_BF16_REL, ATTN_BF16_SIGMA, BF16_ATOL, BF16_RTOL, _assert_close_sigma, _attention_ref, _gelu,
                          _ln_linear_ref, _sigma_worst)
from test_gpu_attention_paths import served_by  # noqa: F401 (fixture)

pytestmark = pytest.mark.gpu


def _worst(err, bound, label):
    worst = float((err / bound).max())
    print(f"\n[{label}] max err {float(err.max()):.3e}, worst err / bound {worst:.3f}")
    return worst


def _bf16(rng, shape, scale=1.0):
    return bf16_round((scale * rng.standard_normal(shape)).astype(np.float32))


def _packed(w, ldw, pad=np.nan):
    """Keras [K, N] weight -> the K-major [N, ldw] form the kernel reads, columns [K, ldw) = pad"""
    K, N = w.shape
    wt = np.full((N, ldw), pad, np.float32)
    wt[:, :K] = w.T
    return wt


# ------------------------------------------------------------------------------------------------------------------ GEMM
@pytest.mark.parametrize("epi", ["plain", "bias_gelu_scale_res"])
@pytest.mark.parametrize("M,N,K", [(394, 768, 192), (65, 1152, 384), (8, 256, 200), (130, 192, 64)])
def test_gemm_strided_operands_and_offset_output(lib, M, N, K, epi):
    """lda = K + 24, ldw = K + 40 with NaN in every pad column (a read past K poisons the output), the output written at
    column 16 of a [M, N + 40] buffer whose other columns hold sentinels that must come back bit for bit."""
    from vit_tensorflow_b200 import _lib
    rng = np.random.default_rng(M * 7 + N + K)
    lda, ldw, off, ldc = K + 24, K + 40, 16, N + 40
    a = np.full((M, lda), np.nan, np.float32)
    a[:, :K] = _bf16(rng, (M, K))
    w = _bf16(rng, (K, N), 1 / np.sqrt(K))
    sentinel = _bf16(rng, (M, ldc), 3.0)
    full = epi != "plain"
    bias = rng.standard_normal(N).astype(np.float32) if full else None
    scale = rng.uniform(0.5, 1.5, N).astype(np.float32) if full else None
    res = _bf16(rng, (M, N + 8)) if full else None          # ldr = N + 8
    out, _, _ = _lib.op_gemm(a, _packed(w, ldw), N, K, sentinel, bias=bias, scale=scale, gelu=full, res=res, out_off=off)
    ref = a[:, :K].astype(np.float64) @ w.astype(np.float64)
    if full:
        ref = _gelu(ref + bias) * scale + res[:, :N]
    keep = np.ones(ldc, bool)
    keep[off:off + N] = False
    np.testing.assert_array_equal(out[:, keep], sentinel[:, keep])
    got = out[:, off:off + N]
    assert np.isfinite(got).all()
    assert _worst(np.abs(got - ref), BF16_ATOL + BF16_RTOL * np.abs(ref), f"gemm strided {epi}") <= 1.0


@pytest.mark.parametrize("epi", ["bias_scale_res", "gelu_res", "bias_gelu_scale_res"])
@pytest.mark.parametrize("M,N,K", [(394, 768, 192), (700, 1152, 384), (63, 384, 64), (1, 256, 128)])
def test_gemm_inplace_residual_equals_out_of_place(lib, M, N, K, epi):
    """res == out (every to_out / fc2 + residual, T2T's X += P V): bit-identical to the same residual from a separate buffer."""
    from vit_tensorflow_b200 import _lib
    rng = np.random.default_rng(M + N + K)
    a = _bf16(rng, (M, K))
    wt = _packed(_bf16(rng, (K, N), 1 / np.sqrt(K)), K)
    x = _bf16(rng, (M, N))
    bias = rng.standard_normal(N).astype(np.float32) if "bias" in epi else None
    scale = rng.uniform(0.5, 1.5, N).astype(np.float32) if "scale" in epi else None
    gelu = "gelu" in epi
    sep, _, _ = _lib.op_gemm(a, wt, N, K, np.zeros((M, N), np.float32), bias=bias, scale=scale, gelu=gelu, res=x)
    inp, _, _ = _lib.op_gemm(a, wt, N, K, x, bias=bias, scale=scale, gelu=gelu, res="out")
    np.testing.assert_array_equal(inp, sep)
    ref = a.astype(np.float64) @ wt.T.astype(np.float64)
    if bias is not None:
        ref = ref + bias
    if gelu:
        ref = _gelu(ref)
    if scale is not None:
        ref = ref * scale
    ref = ref + x
    assert _worst(np.abs(inp - ref), BF16_ATOL + BF16_RTOL * np.abs(ref), f"gemm in-place {epi}") <= 1.0


@pytest.mark.parametrize("n,Dp", [(784, 192), (197, 64), (3136, 64), (50, 192)])
def test_gemm_f32_out_with_zero_filled_weight_rows(lib, n, Dp):
    """T2T S = Q K^T (engine.cu layer_t2t): A = Q and the weight = K read out of the fused [q|k|v] rows (lda = ldw = 3 Dp,
    K = Dp), only b_rows = n weight rows exist, N = round_up(n, 64), fp32 output.  Values within fp32 accumulation error of
    the float64 product; columns [n, N) exactly 0 (the TMA zero fill), not the sentinel that was there."""
    from vit_tensorflow_b200 import _lib
    rng = np.random.default_rng(n + Dp)
    N = (n + 63) // 64 * 64
    qkv = _bf16(rng, (n, 3 * Dp))
    kvn = np.concatenate([qkv[:, Dp:], np.full((n, Dp), np.nan, np.float32)], 1)    # K rows at column 0, pitch 3 Dp
    out, _, _ = _lib.op_gemm(qkv, kvn, N, Dp, np.full((n, N), 7.0, np.float32), out_f32=True)
    q64, k64 = qkv[:, :Dp].astype(np.float64), qkv[:, Dp:2 * Dp].astype(np.float64)
    ref = q64 @ k64.T
    bound = Dp * 2.0 ** -23 * (np.abs(q64) @ np.abs(k64).T) + 1e-30
    assert _worst(np.abs(out[:, :n] - ref), bound, "gemm fp32 out") <= 1.0
    assert (out[:, n:] == 0).all()


def _stats_ref(y):
    """float64 (sum, sumsq) over every 64-column chunk of y [M, N] -> [N/64, M, 2] and the bounds' scales"""
    M, N = y.shape
    c = y.astype(np.float64).reshape(M, N // 64, 64).transpose(1, 0, 2)
    return c.sum(-1), (c ** 2).sum(-1), np.abs(c).sum(-1)


@pytest.mark.parametrize("res", [False, True])
@pytest.mark.parametrize("M,N,K", [(394, 768, 192), (700, 1152, 384), (63, 384, 64), (130, 192, 256)])   # 256-, 128-, 128-, 128-wide tiles
def test_gemm_stats_out(lib, M, N, K, res):
    """Epilogue row statistics (stats_out): each (sum, sumsq) equals the float64 sums over its 64 columns of the RETURNED bf16
    output within 1e-5 relative to sum |x| (resp. sum x^2)."""
    from vit_tensorflow_b200 import _lib
    rng = np.random.default_rng(M + 3 * N + K)
    a = _bf16(rng, (M, K))
    wt = _packed(_bf16(rng, (K, N), 1 / np.sqrt(K)), K)
    bias = rng.standard_normal(N).astype(np.float32)
    r = bf16_round(5.0 * rng.standard_normal((M, N)).astype(np.float32) + 20.0) if res else None
    out, st, _ = _lib.op_gemm(a, wt, N, K, np.zeros((M, N), np.float32), bias=bias, res=r, want_stats=True)
    s1, s2, sabs = _stats_ref(out)
    w1 = _worst(np.abs(st[..., 0] - s1), 1e-5 * sabs + 1e-30, "stats_out sum")
    w2 = _worst(np.abs(st[..., 1] - s2), 1e-5 * s2 + 1e-30, "stats_out sumsq")
    assert w1 <= 1.0 and w2 <= 1.0


@pytest.mark.parametrize("rows", ["offset50", "outliers"])
@pytest.mark.parametrize("M,D,N,K1", [(394, 768, 768, 768), (63, 384, 1152, 1536), (130, 192, 256, 384)])
def test_gemm_stats_chain_into_ln_folded_gemm(lib, M, D, N, K1, rows):
    """The engine's chain: X = fc2(h) + X (stats_out) -> the next layer's LayerNorm-folded GEMM reducing (mean, rstd) from those
    epilogue statistics.  Against the float64 LayerNorm of the returned bf16 X followed by the matmul, with
    test_ln_folded_linear's bound; the residual rows have mean 50 (E[x^2] - mu^2 cancels 3.4 digits) and, for 'outliers',
    four channels two orders of magnitude above the rest."""
    from vit_tensorflow_b200 import _lib
    rng = np.random.default_rng(M + D + N)
    x = rng.standard_normal((M, D)).astype(np.float32) + 50.0
    if rows == "outliers":
        cols = rng.choice(D, 4, replace=False)
        x[:, cols] = (100.0 * (50.0 + rng.standard_normal((M, 4)))).astype(np.float32)
    x = bf16_round(x)
    h = _bf16(rng, (M, K1))
    w1 = _bf16(rng, (K1, D), 0.3 / np.sqrt(K1))
    b1 = (0.2 * rng.standard_normal(D)).astype(np.float32)
    X, st, _ = _lib.op_gemm(h, _packed(w1, K1), D, K1, x, bias=b1, res="out", want_stats=True)
    # fold LayerNorm(gamma, beta) into the next Dense as the engine packs it: Wt = bf16(W * gamma), c1 = row sums of Wt,
    # c2 = beta . W + bias
    g = rng.uniform(0.5, 1.5, D).astype(np.float32)
    be = (0.2 * rng.standard_normal(D)).astype(np.float32)
    w2 = (rng.standard_normal((D, N)) / np.sqrt(D)).astype(np.float32)
    b2 = (0.2 * rng.standard_normal(N)).astype(np.float32)
    wt2 = bf16_round((w2 * g[:, None]).T.copy())
    c1 = wt2.astype(np.float64).sum(1).astype(np.float32)
    c2 = (be.astype(np.float64) @ w2.astype(np.float64) + b2).astype(np.float32)
    out, _, _ = _lib.op_gemm(X, wt2, N, D, np.zeros((M, N), np.float32), bias=c2, ln_stats=st, ln_c1=c1)
    ref, y = _ln_linear_ref(X, g, be, w2, b2, False)
    scale = np.sqrt((y ** 2) @ (w2.astype(np.float64) ** 2))
    bound = 2.0 ** -7 * np.abs(ref) + 2.0 ** -6 * scale + 1e-3
    assert _worst(np.abs(out - ref), bound, f"stats chain {rows}") <= 1.0


# ------------------------------------------------------------------------------------------------------------- attention
def _mixes(rng, variant, heads):
    mix_a = rng.standard_normal((heads, heads)).astype(np.float32) if variant else None
    mix_b = rng.standard_normal((heads, heads)).astype(np.float32) if variant == 2 else None
    g = rng.uniform(0.5, 1.5, heads).astype(np.float32) if variant == 1 else None
    b = rng.standard_normal(heads).astype(np.float32) if variant == 1 else None
    return mix_a, mix_b, g, b


def _check_attention(out, ref, precision, variant):
    if precision == "fp32":
        np.testing.assert_allclose(out, ref, rtol=2e-4, atol=2e-4)
    else:
        _assert_close_sigma(out, ref, ATTN_BF16_SIGMA[variant], ATTN_BF16_REL)


def _fused_case(rng, B, n, heads, dh, precision):
    rnd = bf16_round if precision == "bf16" else (lambda t: t)
    inner = heads * dh
    qkv = rnd(rng.standard_normal((B, n, 3 * inner), dtype=np.float32))
    return qkv, qkv[..., :inner], qkv[..., inner:2 * inner], qkv[..., 2 * inner:]


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("n", [197, 258, 577])
def test_attention_fused_qkv_rows_flash(lib, n, precision):
    """Self-attention reading the fused to_qkv output (engine.cu layer_self): q, k, v at columns 0 / inner / 2 inner of the
    same rows, ldq = ldk = ldv = 3 inner, ldo = inner.  bf16 dim_head 64: the flash kernel."""
    from vit_tensorflow_b200 import _lib
    rng = np.random.default_rng(n)
    B, heads, dh = 2, 3, 64
    inner = heads * dh
    qkv, q, k, v = _fused_case(rng, B, n, heads, dh, precision)
    out, _ = _lib.op_attention_ex(qkv, heads, dh, np.zeros((B, n, inner), np.float32), k_off=inner, v_off=2 * inner, precision=precision)
    _check_attention(out, _attention_ref(q, k, v, heads, 0, None, None, None, None), precision, 0)


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("variant", [1, 2])
@pytest.mark.parametrize("heads,dh", [(4, 64), (8, 48), (16, 32)])
def test_attention_fused_qkv_rows_mix(lib, heads, dh, variant, precision):
    """DeepViT re-attention / CaiT talking heads on the fused [q|k|v] rows: heads 8 / 16 take the rows path, heads 4 the
    mid_fused path (attn_generic_mma.cu); fp32 the SIMT kernels."""
    from vit_tensorflow_b200 import _lib
    rng = np.random.default_rng(heads * 10 + variant)
    B, n = 2, 197
    inner = heads * dh
    qkv, q, k, v = _fused_case(rng, B, n, heads, dh, precision)
    ma, mb, g, b = _mixes(rng, variant, heads)
    out, _ = _lib.op_attention_ex(qkv, heads, dh, np.zeros((B, n, inner), np.float32), k_off=inner, v_off=2 * inner, variant=variant,
                                  mix_a=ma, mix_b=mb, ln_gamma=g, ln_beta=b, precision=precision)
    _check_attention(out, _attention_ref(q, k, v, heads, variant, ma, mb, g, b), precision, variant)


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("variant", [0, 2])
@pytest.mark.parametrize("dh", [48, 64])
@pytest.mark.parametrize("nk", [197, 50])
def test_attention_cls_query_over_kv_rows(lib, nk, dh, variant, precision):
    """CaiT class attention / CrossViT cross attention (engine.cu layer_cls, cross_attend): q [B, 1, inner] against the to_kv
    output [B, nk, 2 inner], k at column 0 and v at column inner (ldk = ldv = 2 inner).  dim_head 64 is CrossViT's default
    cross_attn_dim_head."""
    from vit_tensorflow_b200 import _lib
    rng = np.random.default_rng(nk + dh + variant)
    rnd = bf16_round if precision == "bf16" else (lambda t: t)
    B, heads = 3, 8
    inner = heads * dh
    q = rnd(rng.standard_normal((B, 1, inner), dtype=np.float32))
    kv = rnd(rng.standard_normal((B, nk, 2 * inner), dtype=np.float32))
    ma, mb, g, b = _mixes(rng, variant, heads)
    out, _ = _lib.op_attention_ex(q, heads, dh, np.zeros((B, 1, inner), np.float32), kv=kv, k_off=0, v_off=inner, variant=variant,
                                  mix_a=ma, mix_b=mb, precision=precision)
    _check_attention(out, _attention_ref(q, kv[..., :inner], kv[..., inner:], heads, variant, ma, mb, g, b), precision, variant)


def _pad_heads(x, heads, dh, dhp=64):
    """[.., heads*dh] -> [.., heads*dhp], head h's columns d >= dh zero (what the zero-padded to_q / to_kv / to_qkv columns of
    pad_heads_f32 produce)"""
    y = np.zeros(x.shape[:-1] + (heads, dhp), np.float32)
    y[..., :dh] = x.reshape(x.shape[:-1] + (heads, dh))
    return y.reshape(x.shape[:-1] + (heads * dhp,))


@pytest.mark.parametrize("nq", [197, 1])
@pytest.mark.parametrize("dh", [16, 32, 48])
def test_attention_head_padded_scale(lib, dh, nq):
    """bf16 ViT / CrossViT layers with dim_head < 64 (engine.cu make_layer): heads widened to 64 with zeros and run with
    scale = dim_head^-0.5 (flash kernel for nq >= 2 on fused [q|k|v] rows, cls kernel for nq = 1 on [k|v] rows).  Against the
    UNPADDED float64 reference; the padded output columns are exactly 0; without the scale argument the bound must fail
    (the test sees the scale)."""
    from vit_tensorflow_b200 import _lib
    rng = np.random.default_rng(dh + nq)
    B, heads, nk, dhp = 2, 4, 197, 64
    inner, innp = heads * dh, heads * dhp
    q = bf16_round(rng.standard_normal((B, nq, inner), dtype=np.float32))
    k = bf16_round(rng.standard_normal((B, nk, inner), dtype=np.float32))
    v = bf16_round(rng.standard_normal((B, nk, inner), dtype=np.float32))
    ref = _attention_ref(q, k, v, heads, 0, None, None, None, None)
    qp, kp, vp = _pad_heads(q, heads, dh), _pad_heads(k, heads, dh), _pad_heads(v, heads, dh)
    if nq > 1:
        args = dict(q=np.concatenate([qp, kp, vp], -1), k_off=innp, v_off=2 * innp)
    else:
        args = dict(q=qp, kv=np.concatenate([kp, vp], -1), k_off=0, v_off=innp)
    zeros = np.zeros((B, nq, innp), np.float32)
    run = lambda scale: _lib.op_attention_ex(heads=heads, dh=dhp, out=zeros, scale=scale, **args)[0].reshape(B, nq, heads, dhp)
    out = run(dh ** -0.5)
    assert (out[..., dh:] == 0).all()
    _assert_close_sigma(out[..., :dh].reshape(B, nq, inner), ref, ATTN_BF16_SIGMA[0], ATTN_BF16_REL)
    wrong, _ = _sigma_worst(run(0.0)[..., :dh].reshape(B, nq, inner), ref, ATTN_BF16_SIGMA[0], ATTN_BF16_REL)
    print(f"[head-padded, default scale 64^-0.5] worst err / bound {wrong:.1f}")
    assert wrong > 1.0


# B * heads > 65 535 (the gridDim.y / gridDim.z limit) at a few MB: nq = nk = 5
GRID_PATHS = {
    "fp32_generic": dict(precision="fp32", heads=16, dh=16, variants=(0, 1, 2), path="simt"),
    "bf16_simt_dh14": dict(precision="bf16", heads=16, dh=14, variants=(0,), path="simt"),
    "bf16_rows_h8": dict(precision="bf16", heads=8, dh=16, variants=(1, 2), path="rows"),
    "bf16_rows_h16": dict(precision="bf16", heads=16, dh=16, variants=(1, 2), path="rows"),
    "bf16_mid_fused_h4": dict(precision="bf16", heads=4, dh=16, variants=(1, 2), path="mid_fused"),
    "bf16_mid_fused_h1": dict(precision="bf16", heads=1, dh=16, variants=(2,), path="mid_fused"),   # B alone > 65 535 (mid_fused_kernel)
    "bf16_flash": dict(precision="bf16", heads=16, dh=64, variants=(0,), path="flash"),             # controls: flat grids already
    "bf16_cls": dict(precision="bf16", heads=16, dh=16, variants=(0,), nq=1, path="cls"),
}


@pytest.mark.parametrize("path", sorted(GRID_PATHS))
def test_attention_batch_times_heads_beyond_65535(lib, served_by, path):
    """Every attention path at B * heads > 65 535 against the float64 reference, and the last images of the batch equal the
    same images run alone (bit for bit).  The named path must be the one that served the call."""
    from vit_tensorflow_b200 import _lib
    p = GRID_PATHS[path]
    heads, dh, precision = p["heads"], p["dh"], p["precision"]
    B = 65536 // heads + 4
    nq, nk = p.get("nq", 5), 5
    inner = heads * dh
    rng = np.random.default_rng(heads * 100 + dh)
    rnd = bf16_round if precision == "bf16" else (lambda t: t)
    q = rnd(rng.standard_normal((B, nq, inner), dtype=np.float32))
    kv = rnd(rng.standard_normal((B, nk, 2 * inner), dtype=np.float32))
    k, v = kv[..., :inner], kv[..., inner:]
    for variant in p["variants"]:
        ma, mb, g, b = _mixes(rng, variant, heads)
        kw = dict(kv=kv, k_off=0, v_off=inner, variant=variant, mix_a=ma, mix_b=mb, ln_gamma=g, ln_beta=b, precision=precision)
        out, _ = served_by(lambda: _lib.op_attention_ex(q, heads, dh, np.zeros((B, nq, inner), np.float32), **kw), p["path"])
        _check_attention(out, _attention_ref(q, k, v, heads, variant, ma, mb, g, b), precision, variant)
        kw["kv"] = kv[-3:]
        tail, _ = _lib.op_attention_ex(q[-3:], heads, dh, np.zeros((3, nq, inner), np.float32), **kw)
        np.testing.assert_array_equal(out[-3:], tail)


# ------------------------------------------------------------------------------------------------------------ softmax rows
@pytest.mark.parametrize("n", [1, 63, 784, 4096, 4097, 5184])
def test_softmax_rows(lib, n):
    """softmax_rows_bf16 (the T2T attention, engine.cu layer_t2t) with npad = round_up(n, 64): rows of up to 4096 keys in
    registers, longer rows in the three-pass kernel.  Values within bf16 rounding of the float64 softmax, P[:, n:npad]
    exactly 0, columns past npad untouched."""
    from vit_tensorflow_b200 import _lib
    rng = np.random.default_rng(n)
    rows, D = 37, 147
    npad = (n + 63) // 64 * 64
    lds, ldp = npad, npad + 64
    s = np.full((rows, lds), np.nan, np.float32)
    s[:, :n] = (np.sqrt(D) * 2.0 * rng.standard_normal((rows, n))).astype(np.float32)   # q.k of a width-147 head, unscaled
    sentinel = bf16_round(rng.standard_normal((rows, ldp)).astype(np.float32) + 3.0)
    scale = np.float32(1.0 / np.sqrt(np.float32(D)))
    p, _ = _lib.op_softmax_rows(s, n, npad, scale, sentinel)
    z = s[:, :n].astype(np.float64) * np.float64(scale)
    ref = np.exp(z - z.max(-1, keepdims=True))
    ref /= ref.sum(-1, keepdims=True)
    # bf16 rounding is up to half an ulp = 2^-8 relative (just above a power of two) and is reached; the fp32 evaluation
    # underneath (scale * log2(e) rounded, exp2f, 1 / l) adds ~1e-6 relative: 2^-16 leaves room for it and nothing else
    assert _worst(np.abs(p[:, :n] - ref), (2.0 ** -8 + 2.0 ** -16) * ref + 1e-30, f"softmax rows n={n}") <= 1.0
    assert (p[:, n:npad] == 0).all()
    np.testing.assert_array_equal(p[:, npad:], sentinel[:, npad:])

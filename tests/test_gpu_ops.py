"""GPU parity tests of single kernels, through the C-ABI (vb_op_*), against numpy on the same operands.

bf16 kernels are checked against float64 math on the bf16-ROUNDED operands, so the only differences are fp32
accumulation order and the final bf16 rounding of the output: tolerance 2^-8 relative + small absolute.
fp32 kernels must match to fp32 round-off."""
import numpy as np
import pytest
from scipy.special import erf

from cases import bf16_round

pytestmark = pytest.mark.gpu

BF16_RTOL, BF16_ATOL = 2.0 ** -7, 2e-2


def _gelu(x):
    return 0.5 * x * (1 + erf(x / np.sqrt(2.0)))


def _linear_case(lib, M, N, K, bias, scale, res, gelu, precision, seed=0):
    from vit_tensorflow_b200 import _lib
    rng = np.random.default_rng(seed)
    rnd = bf16_round if precision == "bf16" else (lambda x: x)
    a = rnd(rng.standard_normal((M, K), dtype=np.float32))
    w = rnd((rng.standard_normal((K, N)) / np.sqrt(K)).astype(np.float32))
    b = rng.standard_normal(N).astype(np.float32) if bias else None
    s = rng.uniform(0.5, 1.5, N).astype(np.float32) if scale else None
    r = rnd(rng.standard_normal((M, N), dtype=np.float32)) if res else None
    out, _ = _lib.op_linear(a, w, b, s, r, gelu, precision)
    ref = a.astype(np.float64) @ w.astype(np.float64)
    if bias:
        ref = ref + b
    if gelu:
        ref = _gelu(ref)
    if scale:
        ref = ref * s
    if res:
        ref = ref + r
    return out, ref


# M <= 64: the second consumer warpgroup of the 128-row tile has no rows (CaiT class layers, CrossViT cross attention: M = batch)
SMALL_M = [(1, 256, 64), (2, 192, 128), (8, 768, 192), (63, 384, 64), (64, 256, 256), (65, 128, 64), (127, 512, 200)]


@pytest.mark.parametrize("M,N,K", [(128, 256, 64), (128, 128, 64), (256, 512, 768), (394, 768, 768), (100, 64, 8),
                                   (777, 3072, 768), (1000, 384, 384), (130, 1024, 200), (50432, 768, 768)] + SMALL_M)
def test_gemm_bf16_plain(lib, M, N, K):
    out, ref = _linear_case(lib, M, N, K, False, False, False, False, "bf16")
    np.testing.assert_allclose(out, ref, rtol=BF16_RTOL, atol=BF16_ATOL)


@pytest.mark.parametrize("bias,scale,res,gelu", [(1, 0, 0, 0), (1, 0, 0, 1), (1, 0, 1, 0), (1, 1, 1, 0), (0, 0, 1, 0), (1, 1, 1, 1)])
@pytest.mark.parametrize("M,N,K", [(394, 768, 192), (5000, 384, 1536), (641, 2304, 768), (700, 1152, 384)] + SMALL_M)   # 4th: 128-wide tiles
def test_gemm_bf16_epilogues(lib, M, N, K, bias, scale, res, gelu):
    out, ref = _linear_case(lib, M, N, K, bias, scale, res, gelu, "bf16", seed=M + N)
    np.testing.assert_allclose(out, ref, rtol=BF16_RTOL, atol=BF16_ATOL)


def test_gemm_bf16_linearity(lib):
    """Size-independent property at the BASELINE M: GEMM(a1 + a2) == GEMM(a1) + GEMM(a2) up to bf16 rounding,
    and every row of the output is produced (no tile skipped)."""
    from vit_tensorflow_b200 import _lib
    rng = np.random.default_rng(1)
    M, N, K = 50432, 768, 768
    a1 = bf16_round(rng.integers(-4, 5, (M, K)).astype(np.float32))      # small integers: exact in bf16 and fp32
    w = bf16_round(rng.integers(-2, 3, (K, N)).astype(np.float32) / 4)
    out, _ = _lib.op_linear(a1, w, precision="bf16")
    ref = a1.astype(np.float64) @ w.astype(np.float64)                   # exact integers/4 -> compare after bf16 rounding
    np.testing.assert_allclose(out, bf16_round(ref.astype(np.float32)), rtol=0, atol=0)


@pytest.mark.parametrize("M,N,K", [(394, 768, 192), (33, 1000, 192), (200, 100, 77)])
def test_gemm_fp32(lib, M, N, K):
    out, ref = _linear_case(lib, M, N, K, True, True, True, True, "fp32")
    np.testing.assert_allclose(out, ref, rtol=1e-4, atol=1e-4)


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("M,D", [(394, 192), (1000, 768), (77, 1024), (50, 100), (64, 2048)])
def test_layernorm(lib, precision, M, D):
    from vit_tensorflow_b200 import _lib
    rng = np.random.default_rng(D)
    rnd = bf16_round if precision == "bf16" else (lambda x: x)
    x = rnd((rng.standard_normal((M, D)) * 2 + 0.5).astype(np.float32))
    g = rng.uniform(0.5, 1.5, D).astype(np.float32)
    b = rng.standard_normal(D).astype(np.float32)
    out, _ = _lib.op_layernorm(x, g, b, precision)
    x64 = x.astype(np.float64)
    mu = x64.mean(-1, keepdims=True)
    var = ((x64 - mu) ** 2).mean(-1, keepdims=True)
    ref = (x64 - mu) / np.sqrt(var + 1e-3) * g + b
    if precision == "fp32":
        np.testing.assert_allclose(out, ref, rtol=1e-5, atol=1e-5)
    else:
        np.testing.assert_allclose(out, ref, rtol=BF16_RTOL, atol=BF16_ATOL)


def _attention_ref(q, k, v, heads, variant, mix_a, mix_b, g, b):
    B, nq, inner = q.shape
    dh = inner // heads
    sp = lambda t: t.reshape(t.shape[0], t.shape[1], heads, dh).transpose(0, 2, 1, 3).astype(np.float64)
    Q, K, V = sp(q), sp(k), sp(v)
    dots = np.einsum('bhid,bhjd->bhij', Q, K) * dh ** -0.5
    if variant == 2:
        dots = np.einsum('bhij,hg->bgij', dots, mix_a.astype(np.float64))
    dots -= dots.max(-1, keepdims=True)
    attn = np.exp(dots)
    attn /= attn.sum(-1, keepdims=True)
    if variant == 1:
        attn = np.einsum('bhij,hg->bgij', attn, mix_a.astype(np.float64))
        a = attn.transpose(0, 2, 3, 1)
        mu = a.mean(-1, keepdims=True)
        var = ((a - mu) ** 2).mean(-1, keepdims=True)
        attn = ((a - mu) / np.sqrt(var + 1e-3) * g + b).transpose(0, 3, 1, 2)
    if variant == 2:
        attn = np.einsum('bhij,hg->bgij', attn, mix_b.astype(np.float64))
    out = np.einsum('bhij,bhjd->bhid', attn, V)
    return out.transpose(0, 2, 1, 3).reshape(B, nq, inner)


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("variant", [0, 1, 2])
@pytest.mark.parametrize("B,nq,nk,heads,dh", [(2, 197, 197, 3, 64), (3, 17, 17, 4, 16), (2, 1, 197, 4, 48), (1, 577, 577, 2, 64),
                                               (4, 65, 65, 2, 32), (2, 197, 197, 16, 64), (2, 196, 196, 8, 48),
                                               (2, 1, 197, 8, 48), (1, 50, 50, 6, 32),
                                               (3, 257, 257, 2, 64), (2, 258, 300, 1, 64)])   # last two: one / two query rows past a multiple of the item size
def test_attention(lib, precision, variant, B, nq, nk, heads, dh):
    from vit_tensorflow_b200 import _lib
    rng = np.random.default_rng(nq * 7 + variant)
    rnd = bf16_round if precision == "bf16" else (lambda x: x)
    inner = heads * dh
    q = rnd(rng.standard_normal((B, nq, inner), dtype=np.float32))
    k = rnd(rng.standard_normal((B, nk, inner), dtype=np.float32))
    v = rnd(rng.standard_normal((B, nk, inner), dtype=np.float32))
    mix_a = rng.standard_normal((heads, heads)).astype(np.float32) if variant else None
    mix_b = rng.standard_normal((heads, heads)).astype(np.float32) if variant == 2 else None
    g = rng.uniform(0.5, 1.5, heads).astype(np.float32) if variant == 1 else None
    b = rng.standard_normal(heads).astype(np.float32) if variant == 1 else None
    out, _ = _lib.op_attention(q, k, v, heads, variant, mix_a, mix_b, g, b, precision)
    ref = _attention_ref(q, k, v, heads, variant, mix_a, mix_b, g, b)
    if precision == "fp32":
        np.testing.assert_allclose(out, ref, rtol=2e-4, atol=2e-4)
    else:
        # P (and DeepViT's re-attention weights) are rounded to bf16 before the PV product on the tensor-core paths and the
        # output is stored as bf16: both are 2^-9 relative.  The bound is stated against the spread of the output (sigma_out:
        # ~0.07 for plain softmax over N(0,1) scores at n = 577, ~14 for DeepViT's O(1) re-attention weights), not against 1.
        _assert_close_sigma(out, ref, ATTN_BF16_SIGMA[variant], ATTN_BF16_REL)


@pytest.mark.parametrize("variant", [1, 2])
@pytest.mark.parametrize("B,nq,nk,heads,dh", [(2, 130, 130, 8, 64), (1, 64, 256, 16, 32), (3, 65, 65, 8, 16), (2, 5, 37, 16, 48),
                                               (1, 256, 256, 8, 48), (5, 197, 197, 16, 64), (2, 16, 16, 8, 64), (150, 70, 70, 8, 32)])
def test_attention_mix_shapes(lib, variant, B, nq, nk, heads, dh):
    """Head-mixing attention (attn_generic_mma.cu; deepvit.py:79-87, cait.py:121-127) at the edges of its tiling:
    partial 64-row query tiles (nq = 130, 65, 5), a single key block, the 256-key limit, key counts that leave the second
    block of a super-block empty (nk = 16, 37, 70), dim_head 16 / 32 / 48 / 64, more items than CTAs (B = 150 x 2 tiles)."""
    from vit_tensorflow_b200 import _lib
    rng = np.random.default_rng(nq * 31 + nk + variant)
    inner = heads * dh
    q = bf16_round(rng.standard_normal((B, nq, inner), dtype=np.float32))
    k = bf16_round(rng.standard_normal((B, nk, inner), dtype=np.float32))
    v = bf16_round(rng.standard_normal((B, nk, inner), dtype=np.float32))
    mix_a = rng.standard_normal((heads, heads)).astype(np.float32)
    mix_b = rng.standard_normal((heads, heads)).astype(np.float32) if variant == 2 else None
    g = rng.uniform(0.5, 1.5, heads).astype(np.float32) if variant == 1 else None
    b = rng.standard_normal(heads).astype(np.float32) if variant == 1 else None
    out, _ = _lib.op_attention(q, k, v, heads, variant, mix_a, mix_b, g, b, "bf16")
    ref = _attention_ref(q, k, v, heads, variant, mix_a, mix_b, g, b)
    _assert_close_sigma(out, ref, ATTN_BF16_SIGMA[variant], ATTN_BF16_REL)


# bf16 attention bound: |err| <= SIGMA * std(ref) + REL * |ref|  (bf16 operands and probabilities, fp32 accumulation)
ATTN_BF16_SIGMA = {0: 1.5e-2, 1: 1.5e-2, 2: 1.5e-2}
ATTN_BF16_REL = 1.0e-2


def _sigma_worst(out, ref, sigma_frac, rel):
    """max over elements of |out - ref| / (sigma_frac * std(ref) + rel * |ref|), and the max error itself"""
    err = np.abs(out - ref)
    bound = sigma_frac * float(ref.std()) + rel * np.abs(ref)
    return float((err / bound).max()), float(err.max())


def _assert_close_sigma(out, ref, sigma_frac, rel):
    worst, emax = _sigma_worst(out, ref, sigma_frac, rel)
    sig = float(ref.std())
    print(f"\n[attention bf16] max err {emax:.3e}, sigma_out {sig:.3e}, max err / sigma_out {emax / sig:.3e}, "
          f"worst err / bound {worst:.3f}")
    assert worst <= 1.0, f"max err {emax:.4e} at sigma_out {sig:.4e}: {worst:.2f} x the bound"


FLASH_FK = 64      # keys per block of attn_flash.cu (FK)


def _rescale_case(B, n, heads, ramp, dh=64):
    """q, k, v (bf16-rounded) for test_attention_lazy_rescale, and the fraction of rows the construction reaches: the scores
    in the kernel's log2 units (dh^-0.5 * log2(e)) per 64-key block."""
    rng = np.random.default_rng(n + heads)
    inner = heads * dh
    nblk = (n + FLASH_FK - 1) // FLASH_FK
    blk = lambda j: slice(j * FLASH_FK, min((j + 1) * FLASH_FK, n))
    q = rng.standard_normal((B, n, inner), dtype=np.float32)
    k = rng.standard_normal((B, n, inner), dtype=np.float32)
    v = bf16_round(rng.standard_normal((B, n, inner), dtype=np.float32))
    u = np.ones(inner, np.float32)
    if ramp in ("up", "down", "zigzag"):          # geometric: a block's max beats the previous blocks' by ~1.6x
        f = {"up": [1.6 ** j for j in range(nblk)], "down": [1.6 ** (nblk - 1 - j) for j in range(nblk)],
             "zigzag": [(1 + 5 * (j % 2)) * 1.1 ** j for j in range(nblk)]}[ramp]
        for j in range(nblk):
            k[:, blk(j)] *= f[j]
    elif ramp == "ragged_max":   # every query leans on u, the last block's keys on 2u: q.k dh^-0.5 ~ 16 there, ~N(0, 1) elsewhere
        q = u + 0.5 * q
        k[:, blk(nblk - 1)] = 2 * u + 0.5 * k[:, blk(nblk - 1)]
    else:   # "underflow": every query leans on u, block 0 on +8u, block 1 on -8u: q.k dh^-0.5 = +-64 (+-2 of noise)
        q = u + 0.25 * q
        k[:, blk(0)] = 8 * u + 0.25 * k[:, blk(0)]
        k[:, blk(1)] = -8 * u + 0.25 * k[:, blk(1)]
    q, k = bf16_round(q), bf16_round(k)
    sp = lambda t: t.reshape(B, n, heads, dh).transpose(0, 2, 1, 3).astype(np.float64)
    s2 = np.einsum('bhid,bhjd->bhij', sp(q), sp(k)) * dh ** -0.5 * 1.4426950408889634
    bm = np.stack([s2[..., blk(j)].max(-1) for j in range(nblk)], -1)          # [B, h, n, nblk] block row maxima
    run = np.maximum.accumulate(bm, -1)
    full = n // FLASH_FK                                                      # blocks of 64 valid keys
    raised = bm[..., 1:full] > run[..., :full - 1]                            # a full block j > 0 raises the running max: alpha < 1
    arg = s2.argmax(-1)
    reach = {"up": raised.mean(), "down": (arg < FLASH_FK).mean(), "zigzag": raised.any(-1).mean(),
             "ragged_max": (arg >= (nblk - 1) * FLASH_FK).mean(),
             # p of block 1 below 2^-149, the smallest fp32 subnormal: exactly 0 however exp2 is evaluated
             "underflow": (s2[..., blk(1)].max(-1) - s2.max(-1) < -150).mean()}[ramp]
    return q, k, v, float(reach)


@pytest.mark.parametrize("ramp", ["up", "down", "zigzag", "ragged_max", "underflow"])
@pytest.mark.parametrize("B,n,heads", [(2, 577, 2), (3, 197, 3), (1, 300, 1), (3, 191, 3), (2, 129, 2)])
def test_attention_lazy_rescale(lib, B, n, heads, ramp):
    """The flash kernel (attn_flash.cu) streams the keys in blocks of FK = 64 and on every block raises its running row max
    and rescales the running output and row sum by alpha = 2^(m_old - m_new).  N(0,1) scores barely move the max after the
    first block, so the keys are scaled per 64-key block: 'up' makes (almost) every later block raise the max, 'down' keeps
    the first block's max throughout, 'zigzag' alternates.  'ragged_max' puts the row maxima into the last, partial block
    (n % 64 = 1 at n = 577 / 129, 5 at n = 197, 63 at n = 191: valid keys next to masked ones).  'underflow' puts block 1's scores ~180
    log2 units below block 0's, so its probabilities are exactly 0 and it must contribute nothing (and no NaN)."""
    from vit_tensorflow_b200 import _lib
    q, k, v, reach = _rescale_case(B, n, heads, ramp)
    assert reach > (0.99 if ramp in ("ragged_max", "underflow") else 0.9), f"test construction reaches only {reach:.2f} of the rows"
    out, _ = _lib.op_attention(q, k, v, heads, 0, precision="bf16")
    ref = _attention_ref(q, k, v, heads, 0, None, None, None, None)
    assert np.isfinite(out).all()
    _assert_close_sigma(out, ref, 1.5e-2, 1.0e-2)


def _ln_linear_ref(x, g, b, w, bias, gelu):
    x64 = x.astype(np.float64)
    mu = x64.mean(-1, keepdims=True)
    var = ((x64 - mu) ** 2).mean(-1, keepdims=True)
    y = (x64 - mu) / np.sqrt(var + 1e-3) * g + b
    r = y @ w.astype(np.float64)
    if bias is not None:
        r = r + bias
    return _gelu(r) if gelu else r, y


@pytest.mark.parametrize("gelu", [False, True])
@pytest.mark.parametrize("rows", ["normal", "offset50", "outliers"])
@pytest.mark.parametrize("M,N,K", [(394, 768, 768), (1000, 3072, 1024), (130, 192, 384), (515, 1152, 384)])
def test_ln_folded_linear(lib, M, N, K, rows, gelu):
    """PreNorm + Dense as the bf16 engine runs it (vit.py:18-22 + :39/:59): LayerNorm folded into the GEMM, its (mean, rstd)
    reduced in the epilogue from one-pass fp32 (sum, sumsq) partials of the bf16 rows.  `offset50`: rows of mean 50 and
    sigma 1 (E[x^2] - mu^2 cancels 3.4 digits); `outliers`: additionally four channels two orders of magnitude above the
    rest, as trained ViTs have.  Reference: float64 LayerNorm + matmul on the same bf16-rounded rows."""
    from vit_tensorflow_b200 import _lib
    rng = np.random.default_rng(M + K)
    x = rng.standard_normal((M, K)).astype(np.float32)
    if rows != "normal":
        x += 50.0
    if rows == "outliers":
        cols = rng.choice(K, 4, replace=False)
        x[:, cols] = (100.0 * (50.0 + rng.standard_normal((M, 4)))).astype(np.float32)
    x = bf16_round(x)
    g = rng.uniform(0.5, 1.5, K).astype(np.float32)
    b = (0.2 * rng.standard_normal(K)).astype(np.float32)
    w = (rng.standard_normal((K, N)) / np.sqrt(K)).astype(np.float32)
    bias = (0.2 * rng.standard_normal(N)).astype(np.float32)
    out, _ = _lib.op_ln_linear(x, g, b, w, bias, gelu)
    ref, y = _ln_linear_ref(x, g, b, w, bias, gelu)
    # bf16 weights (2^-9 relative each, K random terms) + bf16 output rounding; the activations enter exactly.
    # natural scale of one output: |y| . |w| summed in quadrature = sqrt(sum_k y_k^2 w_kn^2)
    scale = np.sqrt((y ** 2) @ (w.astype(np.float64) ** 2))
    err = np.abs(out - ref)
    bound = 2.0 ** -7 * np.abs(ref) + 2.0 ** -6 * scale + 1e-3
    worst = float((err / bound).max())
    print(f"\n[ln-folded linear {rows}] max err {err.max():.3e}, max |ref| {np.abs(ref).max():.3e}, worst err / bound {worst:.3f}")
    assert worst <= 1.0


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("shape", [(2, 49, 64, 5), (3, 196, 256, 8), (1, 10, 24, 3)])
def test_patch_merger_op(lib, precision, shape):
    """PatchMerger.call (vit_with_patch_merger.py:49-55) against the float64 spec."""
    from oracle import spec_numpy
    from vit_tensorflow_b200 import _lib
    B, n, D, nt = shape
    rng = np.random.default_rng(B * 1000 + n)
    x = rng.standard_normal((B, n, D)).astype(np.float32)
    w = {"patch_merger.norm.gamma": (1 + 0.2 * rng.standard_normal(D)).astype(np.float32),
         "patch_merger.norm.beta": (0.2 * rng.standard_normal(D)).astype(np.float32),
         "patch_merger.queries": rng.standard_normal((nt, D)).astype(np.float32)}
    if precision == "bf16":
        from cases import bf16_round
        x = bf16_round(x)
    got, _ = _lib.op_patch_merger(x, w["patch_merger.norm.gamma"], w["patch_merger.norm.beta"], w["patch_merger.queries"], precision=precision)
    ref = spec_numpy.patch_merger(x.astype(np.float64), {k: v.astype(np.float64) for k, v in w.items()})
    assert got.shape == (B, nt, D)
    if precision == "fp32":
        np.testing.assert_allclose(got, ref, rtol=1e-3, atol=1e-4)
    else:
        assert (np.abs(got - ref) <= 3e-2 + 3e-2 * np.abs(ref)).all()

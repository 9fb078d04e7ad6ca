"""The engine's convolution path and its pooling / gather kernels as single operators (vb_op_conv2d, vb_op_cct_pool,
vb_op_seq_pool, vb_op_pool_layernorm, vb_op_gather_grid) against float64 references written out here.

vb_op_conv2d runs vb_handle::conv, the step behind every convolution that is not depthwise: unfold_same writes the patch rows
(with the LayerNorm / GELU applied on load and VALID windows in the bf16 engine's modes), the GEMM multiplies them.  In the fp32
engine the LayerNorm is a separate launch, so the on-load arithmetic is only checked by these bf16 cases; end to end, behind a
classifier head, a wrong epsilon or a padded tap read as beta can hide inside the logits' tolerance.

TF semantics of the references: SAME gives ceil(in / s) outputs with total padding max((out - 1) s + k - in, 0), the smaller
half first; VALID gives floor((in - k) / s) + 1; the patch vector is ordered (k_row, k_col, c).  tests/test_conv_ops_reference.py
checks these references against independent statements of the same operations at every case shape below."""
import zlib

import numpy as np
import pytest
from scipy.special import erf

from cases import bf16_round

pytestmark = pytest.mark.gpu


# ------------------------------------------------------------------------------------------------ float64 references
def out_geometry(n, k, s, valid):
    """(outputs, padding before) along one side."""
    if valid:
        return (n - k) // s + 1, 0
    out = -(-n // s)
    return out, max((out - 1) * s + k - n, 0) // 2


def conv_ref(x, kernel, stride, valid=False):
    """Conv2D(k, stride, SAME | VALID) without bias, NHWC: x [B, H, W, C], kernel [k, k, C, N] -> [B, oh, ow, N], accumulated tap
    by tap; a tap outside the map reads zero."""
    x, kernel = np.asarray(x, np.float64), np.asarray(kernel, np.float64)
    B, H, W, C = x.shape
    k, N = kernel.shape[0], kernel.shape[3]
    oh, pt = out_geometry(H, k, stride, valid)
    ow, pl = out_geometry(W, k, stride, valid)
    out = np.zeros((B, oh, ow, N))
    for ky in range(k):
        ys = np.arange(oh) * stride - pt + ky
        yin = (ys >= 0) & (ys < H)
        for kx in range(k):
            xs = np.arange(ow) * stride - pl + kx
            xin = (xs >= 0) & (xs < W)
            tap = x[:, np.clip(ys, 0, H - 1)][:, :, np.clip(xs, 0, W - 1)] * (yin[:, None] & xin[None, :])[None, :, :, None]
            out += tap @ kernel[ky, kx]
    return out


def maxpool_relu_ref(x, k, stride, pos=None, rows=None, dtype=np.float32):
    """ReLU -> MaxPool2D(k, stride, SAME) (padded taps never win) -> + pos, in `dtype`: x [B, H, W, C] -> [B, rows, C]."""
    x = np.asarray(x, dtype)
    B, H, W, C = x.shape
    oh, pt = out_geometry(H, k, stride, False)
    ow, pl = out_geometry(W, k, stride, False)
    m = np.full((B, oh, ow, C), -np.inf, dtype)
    for ky in range(k):
        for kx in range(k):
            for oy in range(oh):
                y = oy * stride - pt + ky
                if not 0 <= y < H:
                    continue
                for ox in range(ow):
                    xx = ox * stride - pl + kx
                    if 0 <= xx < W:
                        m[:, oy, ox] = np.maximum(m[:, oy, ox], x[:, y, xx])
    v = np.maximum(m, dtype(0)).reshape(B, oh * ow, C)
    if pos is not None:
        v = v + np.asarray(pos, dtype).reshape(1, oh * ow, C)
    rows = oh * ow if rows is None else rows
    out = np.zeros((B, rows, C), dtype)
    out[:, :oh * ow] = v
    return out


def layer_norm(x, gamma, beta, eps):
    x = np.asarray(x, np.float64)
    mu = x.mean(-1, keepdims=True)
    var = ((x - mu) ** 2).mean(-1, keepdims=True)
    return (x - mu) / np.sqrt(var + eps) * gamma + beta


def seq_pool_ref(x, gamma, beta, pw, pb):
    """CCT's SeqPool (cct.py:291-299): y = LayerNorm(x) (eps 1e-3), w = softmax over the tokens of y . pw + pb, z = sum_t w_t y_t."""
    y = layer_norm(x, gamma, beta, 1e-3)
    s = y @ np.asarray(pw, np.float64) + pb
    w = np.exp(s - s.max(1, keepdims=True))
    w /= w.sum(1, keepdims=True)
    return (w[..., None] * y).sum(1)


def gelu(x):
    return 0.5 * x * (1 + erf(x / np.sqrt(2.0)))


ACTS = {"none": lambda v: v, "gelu": gelu, "hswish": lambda v: v * np.clip(v + 3.0, 0.0, 6.0) / 6.0, "silu": lambda v: v / (1 + np.exp(-v))}


# ------------------------------------------------------------------------------------------------ convolution cases
def _case(id, B, H, W, cin, N, k, s, valid=False, image=False, ld=None, off=0, ln=None, rows="normal", gelu_in=False, act="none",
          res=False, stats=False, bias=True):
    """ln: None or the LayerNorm's eps.  rows: the map's values ('normal', 'offset50', 'outliers', 'small' for sigma 0.01)."""
    return dict(id=id, B=B, H=H, W=W, cin=cin, N=N, k=k, s=s, valid=valid, image=image, ld=ld or cin, off=off, ln=ln, rows=rows,
                gelu_in=gelu_in, act=act, res=res, stats=stats, bias=bias)


CONV_CASES = [
    # image stems
    _case("cct_k7s2", 2, 32, 32, 3, 64, 7, 2, image=True, bias=False),              # CCT tokenizer conv
    _case("cct_k7s2_odd", 1, 31, 29, 3, 64, 7, 2, image=True, bias=False),          # CCT, odd image
    _case("levit_k3s2", 2, 30, 30, 3, 64, 3, 2, image=True),                       # LeViT stem conv 1, RegionViT 3-conv tokenizer conv 1
    _case("regionvit_k8s4", 2, 34, 30, 3, 128, 8, 4, image=True),                   # RegionViT local tokenizer
    _case("twins_kp", 2, 28, 28, 3, 64, 4, 4, image=True),                         # Twins-SVT / NesT patch embedding (k = s = p)
    _case("nest_kp_odd", 1, 21, 21, 3, 64, 7, 7, image=True),                      # NesT-like k = s = p on a 3 x 3 grid
    _case("crossformer_k32s4", 1, 40, 36, 3, 64, 32, 4, image=True),               # CrossFormer stage 1, K = 3072
    _case("pit_valid_k14s7", 2, 45, 52, 3, 64, 14, 7, valid=True, image=True),      # PiT patch embedding, (H - k) % s != 0
    # maps: both unfold paths (C < 32 per column, C >= 32 per tap) and both thread counts
    _case("map_c16_k2", 2, 9, 9, 16, 64, 2, 1),                                   # per column, 64 threads (k k C < 128)
    _case("map_c16_k3", 2, 9, 9, 16, 64, 3, 1),                                   # per column, 160 threads
    _case("map_c31_k3s2", 2, 11, 8, 31, 64, 3, 2),                                # CrossFormer-like odd widths, per column
    _case("map_c32_k3s2", 2, 11, 8, 32, 64, 3, 2),                                # per tap, 64 threads
    _case("map_c33_k3", 1, 7, 10, 33, 64, 3, 1),                                  # per tap, 64 threads, ragged channel loop
    _case("map_c127_k3s2", 2, 9, 7, 127, 128, 3, 2),                              # per tap, 64 threads
    _case("map_c128_k3", 1, 8, 8, 128, 128, 3, 1),                                # NesT Aggregate conv, per tap, 160 threads
    _case("map_c200_k3s2", 2, 7, 7, 200, 192, 3, 2),                              # LeViT / RegionViT downsample widths, 160 threads
    _case("map_rect", 1, 5, 13, 64, 64, 3, 2),                                    # rectangular
    _case("map_one_pixel", 3, 1, 1, 48, 64, 3, 2),                                # one pixel: every tap but the centre is padding
    _case("map_smaller_than_k", 2, 2, 2, 40, 64, 3, 1),                           # H = 2 < k = 3
    _case("map_k1s2", 2, 9, 6, 64, 64, 1, 2),                                     # stride larger than k
    _case("lim_ld_offset", 2, 6, 6, 64, 64, 3, 1, ld=192, off=128),               # ScalableViT LIM: v's columns of q|k|v rows
    _case("map_ld_offset_small", 1, 5, 7, 20, 64, 3, 1, ld=56, off=30),           # per-column path at a column offset
    _case("rows_past_65535", 2, 192, 192, 32, 64, 3, 1),                          # B * rows = 73,728 CTAs
    # LayerNorm on load (Twins-SVT global to_kv, ScalableViT SSA k|v and Downsample, RegionViT Downsample and 3-conv tokenizer)
    _case("ln_parts1_c40", 2, 9, 9, 40, 64, 3, 2, ln=1e-5),                       # one 64-column part, cin below it
    _case("ln_parts2_c100", 2, 8, 10, 100, 128, 3, 2, ln=1e-5, rows="offset50"),  # ScalableViT Downsample, rows of mean 50
    _case("ln_parts6_c330", 1, 6, 5, 330, 64, 3, 2, ln=1e-5, rows="outliers"),    # six parts, outlier channels
    _case("ln_eps5_small", 2, 7, 9, 64, 64, 3, 2, ln=1e-5, rows="small"),         # sigma 0.01: eps 1e-5 vs 1e-3 differ by ~3x
    _case("ln_eps3_small", 2, 7, 9, 64, 64, 3, 2, ln=1e-3, rows="small"),
    _case("ln_eps5_small_c24", 2, 7, 9, 24, 64, 3, 2, ln=1e-5, rows="small"),     # the same on the per-column path
    _case("ln_gelu_c64", 2, 9, 8, 64, 64, 3, 2, ln=1e-3, gelu_in=True),           # RegionViT 3-conv tokenizer conv 2
    _case("ln_gelu_c24", 2, 9, 8, 24, 64, 3, 1, ln=1e-3, gelu_in=True),           # RegionViT tokenizer conv 3, per column
    _case("ln_gelu_c16_small", 1, 5, 5, 16, 64, 2, 1, ln=1e-5, rows="small", gelu_in=True),   # per column, 64 threads
    _case("gelu_only_c48", 2, 7, 7, 48, 64, 3, 2, gelu_in=True),                  # GELU on load without a LayerNorm
    _case("gelu_only_c12", 2, 7, 7, 12, 64, 3, 2, gelu_in=True),
    _case("ln_valid_r1", 2, 6, 6, 64, 128, 1, 1, valid=True, ln=1e-5),            # ScalableViT SSA k|v, r = 1
    _case("ln_valid_r2", 2, 8, 6, 64, 128, 2, 2, valid=True, ln=1e-5, rows="offset50"),   # r = 2
    _case("ln_valid_r4", 2, 9, 11, 128, 128, 4, 4, valid=True, ln=1e-5),          # r = 4, Twins-SVT global to_kv (k = s)
    _case("ln_valid_r8", 1, 16, 16, 96, 128, 8, 8, valid=True, ln=1e-5, rows="small"),    # r = 8
    _case("ln_valid_r2_c20", 2, 6, 6, 20, 64, 2, 2, valid=True, ln=1e-5, rows="outliers"),  # per column
    # epilogue
    _case("act_gelu", 2, 8, 8, 64, 128, 3, 1, act="gelu"),
    _case("act_hswish", 2, 8, 8, 64, 128, 3, 2, act="hswish"),                    # LeViT
    _case("act_silu", 2, 8, 8, 32, 64, 3, 2, act="silu"),                         # MobileViT (its BatchNorm shift as the bias)
    _case("act_silu_image", 2, 16, 16, 3, 64, 3, 2, image=True, act="silu"),      # MobileViT conv1
    _case("residual", 2, 6, 6, 64, 64, 3, 1, ld=192, off=128, res=True),          # ScalableViT LIM with its residual
    _case("stats", 2, 9, 9, 64, 128, 3, 2, stats=True),                           # ScalableViT to_patches / Downsample
    _case("stats_ln_res", 2, 8, 8, 96, 128, 3, 2, ln=1e-5, res=True, stats=True, act="gelu"),
    _case("n_not_64", 2, 7, 7, 40, 96, 3, 2),                                     # N % 64 != 0 (the GEMM's other path in bf16)
]


def conv_operands(c):
    """The case's host operands: x (image [B, H, W, cin] or map [B*H*W, ld]), kernel, bias, gamma, beta, res [rows, ldr]."""
    rng = np.random.default_rng(zlib.crc32(c["id"].encode()))
    B, H, W, cin, N, k = c["B"], c["H"], c["W"], c["cin"], c["N"], c["k"]
    if c["image"]:
        x = rng.standard_normal((B, H, W, cin)).astype(np.float32)
    else:
        x = rng.standard_normal((B * H * W, c["ld"])).astype(np.float32)
        ch = slice(c["off"], c["off"] + cin)
        if c["rows"] == "small":
            x[:, ch] = 0.01 * x[:, ch] + 0.003 * rng.standard_normal((B * H * W, 1))
        elif c["rows"] in ("offset50", "outliers"):
            x[:, ch] += 50.0
        if c["rows"] == "outliers":
            cols = c["off"] + rng.choice(cin, 4, replace=False)
            x[:, cols] = 100.0 * (50.0 + rng.standard_normal((B * H * W, 4)))
        if c["ln"] is not None:
            x[:, cin:] = 0.0                                   # the engine's zero pad columns
    kernel = (rng.standard_normal((k, k, cin, N)) / np.sqrt(k * k * cin)).astype(np.float32)
    bias = (0.2 * rng.standard_normal(N)).astype(np.float32) if c["bias"] else None
    gamma = beta = None
    if c["ln"] is not None:
        gamma = rng.uniform(0.5, 1.5, cin).astype(np.float32)
        gamma[::5] *= -1.0
        beta = (1.0 + 0.3 * rng.standard_normal(cin)).astype(np.float32)   # beta well away from 0: a padded tap read as LN(0) shows
    oh, _ = out_geometry(H, k, c["s"], c["valid"])
    ow, _ = out_geometry(W, k, c["s"], c["valid"])
    res = rng.standard_normal((B * oh * ow, N + 40)).astype(np.float32) if c["res"] else None
    return x, kernel, bias, gamma, beta, res


def conv_case_ref(c, x, kernel, bias, gamma, beta, res, bf16):
    """float64 reference of the case on the operands the kernels see (bf16: the map / unfolded values, the weights and the residual
    rounded to bf16) -> (out [rows, N], scale [rows, N] = sqrt(sum over the taps of v^2 w^2))."""
    rnd = bf16_round if bf16 else (lambda a: np.asarray(a, np.float32))
    B, H, W, cin = c["B"], c["H"], c["W"], c["cin"]
    if c["image"]:
        v = np.asarray(x, np.float64)
    else:
        v = rnd(x)[:, c["off"]:c["off"] + cin].astype(np.float64)
        if c["ln"] is not None:
            v = layer_norm(v, gamma.astype(np.float64), beta.astype(np.float64), c["ln"])
        if c["gelu_in"]:
            v = gelu(v)
        v = v.reshape(B, H, W, cin)
    v = rnd(v).astype(np.float64) if bf16 else v
    w = rnd(kernel).astype(np.float64)
    pre = conv_ref(v, w, c["s"], c["valid"])
    scale = np.sqrt(conv_ref(v * v, w * w, c["s"], c["valid"]))
    N = kernel.shape[3]
    pre = pre.reshape(-1, N) + (0.0 if bias is None else bias.astype(np.float64))
    out = ACTS[c["act"]](pre)
    if res is not None:
        out = out + rnd(res)[:, :N].astype(np.float64)
    return out, scale.reshape(-1, N)


def _run_conv(c, x, kernel, bias, gamma, beta, res, precision, want_stats=False):
    from vit_tensorflow_b200 import _lib
    hw = None if c["image"] else (c["B"], c["H"], c["W"])
    return _lib.op_conv2d(x, kernel, bias, c["s"], c["valid"], c["image"], hw, c["cin"], c["off"], gamma, beta,
                          c["ln"] if c["ln"] is not None else 1e-5, c["gelu_in"], c["act"], res, want_stats, precision)


def _worst(err, bound, label):
    worst = float((err / bound).max())
    print(f"\n[{label}] max err {err.max():.3e}, worst err / bound {worst:.3f}")
    return worst


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("c", CONV_CASES, ids=[c["id"] for c in CONV_CASES])
def test_conv2d_against_float64(lib, c, precision):
    """bf16 bound (test_ln_folded_linear's shape): |err| <= 2^-7 |ref| + 2^-6 sqrt(sum v^2 w^2) + 1e-3 -- the output's bf16
    rounding, fp32 accumulation, and the on-load LayerNorm / GELU value landing one bf16 step from the float64 value's rounding.
    fp32: the same shape with 2^-16 |ref| + 2^-14 sqrt(sum v^2 w^2) + 1e-5, ~100x the fp32 accumulation error of K <= 3072 terms."""
    bf16 = precision == "bf16"
    ops = conv_operands(c)
    out, stats, _ = _run_conv(c, *ops, precision, want_stats=c["stats"] and bf16)
    ref, scale = conv_case_ref(c, *ops, bf16)
    assert out.shape == ref.shape and np.isfinite(out).all()
    err = np.abs(out - ref)
    bound = (2.0 ** -7 * np.abs(ref) + 2.0 ** -6 * scale + 1e-3) if bf16 else (2.0 ** -16 * np.abs(ref) + 2.0 ** -14 * scale + 1e-5)
    assert _worst(err, bound, f"conv {c['id']} {precision}") <= 1.0
    if stats is not None:                                  # the epilogue's (sum, sumsq) of the returned bf16 rows
        rows, N = out.shape
        ch = out.astype(np.float64).reshape(rows, N // 64, 64).transpose(1, 0, 2)
        w1 = _worst(np.abs(stats[..., 0] - ch.sum(-1)), 1e-5 * np.abs(ch).sum(-1) + 1e-30, "stats_out sum")
        w2 = _worst(np.abs(stats[..., 1] - (ch ** 2).sum(-1)), 1e-5 * (ch ** 2).sum(-1) + 1e-30, "stats_out sumsq")
        assert w1 <= 1.0 and w2 <= 1.0


PAD_SHAPES = [(7, 7, 1), (8, 6, 1), (7, 9, 2), (8, 8, 2), (1, 1, 1), (2, 3, 2)]


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("H,W,s", PAD_SHAPES)
@pytest.mark.parametrize("cin,gelu_in", [(64, False), (64, True), (20, False), (20, True)])
def test_conv2d_padded_taps_contribute_zero(lib, precision, H, W, s, cin, gelu_in):
    """A padded tap is zero after the LayerNorm / GELU on load, not LN(0) * gamma + beta = beta or GELU(beta).  Output column n
    of the kernel reads only one border of the 3 x 3 window (n % 4: top row, bottom row, left column, right column); at every
    output pixel whose window has that border in the padding the column is exactly zero (no bias; beta ~ 1).  cin 64 runs the
    per-tap path, cin 20 the per-column path."""
    c = _case("pad", 2, H, W, cin, 64, 3, s, ln=1e-5, gelu_in=gelu_in, bias=False)
    x, kernel, _, gamma, beta, _ = conv_operands(c)
    side = np.arange(64) % 4
    mask = np.zeros((3, 3, 1, 64), np.float32)
    mask[0, :, 0, side == 0] = 1.0
    mask[2, :, 0, side == 1] = 1.0
    mask[:, 0, 0, side == 2] = 1.0
    mask[:, 2, 0, side == 3] = 1.0
    kernel = kernel * mask
    out, _, _ = _run_conv(c, x, kernel, None, gamma, beta, None, precision)
    oh, pt = out_geometry(H, 3, s, False)
    ow, pl = out_geometry(W, 3, s, False)
    out = out.reshape(2, oh, ow, 64)
    oy, ox = np.arange(oh) * s - pt, np.arange(ow) * s - pl           # the window's first row / column
    padded = [(oy < 0)[:, None] & np.ones(ow, bool), (oy + 2 >= H)[:, None] & np.ones(ow, bool),
              np.ones(oh, bool)[:, None] & (ox < 0), np.ones(oh, bool)[:, None] & (ox + 2 >= W)]
    checked = 0
    for j in range(4):
        sel = out[:, padded[j]][..., side == j]
        assert (sel == 0.0).all(), f"border {j}: padded taps contribute {np.abs(sel).max():.3g}"
        checked += sel.size
    assert checked > 0
    ref, scale = conv_case_ref(c, x, kernel, None, gamma, beta, None, precision == "bf16")
    bound = 2.0 ** -7 * np.abs(ref) + 2.0 ** -6 * scale + 1e-3
    assert (np.abs(out.reshape(ref.shape) - ref) <= bound).all()


def test_conv2d_refusals(lib):
    from vit_tensorflow_b200 import _lib
    rng = np.random.default_rng(0)
    x = rng.standard_normal((2 * 4 * 4, 64)).astype(np.float32)
    kern = rng.standard_normal((3, 3, 64, 64)).astype(np.float32)
    g, b = np.ones(64, np.float32), np.zeros(64, np.float32)
    with pytest.raises(_lib.VbError, match="VALID window larger"):
        _lib.op_conv2d(x, np.zeros((5, 5, 64, 64), np.float32), valid=True, HW=(2, 4, 4))
    with pytest.raises(_lib.VbError, match="exceed ld"):
        _lib.op_conv2d(x, kern, HW=(2, 4, 4), off=8)
    with pytest.raises(_lib.VbError, match="must be zero"):
        _lib.op_conv2d(x, kern[:, :, :32], HW=(2, 4, 4), cin=32, ln_gamma=g[:32], ln_beta=b[:32])
    with pytest.raises(_lib.VbError, match="not the image"):
        _lib.op_conv2d(x.reshape(2, 4, 4, 64), kern, image=True, gelu_in=True)


# ------------------------------------------------------------------------------------------------ CCT max-pool
POOL_CASES = [(k, s, H, W, C) for k, s in [(1, 1), (2, 1), (3, 2), (5, 3), (1, 3), (2, 3), (3, 1), (5, 2)]
              for H, W, C in [(7, 9, 48), (8, 6, 130), (1, 5, 1)]]


def pool_operands(k, s, H, W, C, with_pos):
    rng = np.random.default_rng(k * 1000 + s * 100 + H * 10 + W + C)
    x = rng.standard_normal((2, H, W, C)).astype(np.float32)
    x[1, :min(H, 3), :min(W, 4)] = -np.abs(x[1, :min(H, 3), :min(W, 4)]) - 0.5   # windows that are all negative
    oh, ow = -(-H // s), -(-W // s)
    pos = rng.standard_normal((oh * ow, C)).astype(np.float32) if with_pos else None
    return x, pos, oh * ow + (0 if with_pos else 3)                  # 'none' positions: zero rows past oh * ow


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("with_pos", [False, True])
@pytest.mark.parametrize("k,s,H,W,C", POOL_CASES)
def test_cct_pool_bit_exact(lib, precision, k, s, H, W, C, with_pos):
    """The max is exact, so the result is too: fp32 equals relu(max) + pos in float32, bf16 equals bf16(float32(max) + pos)."""
    from vit_tensorflow_b200 import _lib
    x, pos, rows = pool_operands(k, s, H, W, C, with_pos)
    xin = bf16_round(x) if precision == "bf16" else x
    got, _ = _lib.op_cct_pool(x, k, s, pos, rows, precision)
    want = maxpool_relu_ref(xin, k, s, pos, rows, np.float32)
    if precision == "bf16":
        want = bf16_round(want)
    assert got.shape == want.shape
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))


# ------------------------------------------------------------------------------------------------ CCT sequence pooling
SEQ_D = [1, 33, 128, 129, 256, 257, 512, 513, 768, 1000, 1024]   # J = 4 up to 128, 8 to 256, 16 to 512, 32 to 1024
SEQ_N = [1, 3, 8, 9, 197, 1025]


def seq_operands(n, D, kind, B=3):
    """kind: 'random'; 'offset50' (rows of mean 50); 'dominant' (one middle token's score sqrt(D) |gamma pw| above the rest's
    N(0, |gamma pw|)); 'underflow' (that score 250: exp underflows to 0 for the tokens far below it); 'equal' (every score equal);
    'late' (the dominant token last: a late warp's last row raises the maximum)."""
    rng = np.random.default_rng(n * 7919 + D * 13 + len(kind))
    x = rng.standard_normal((B, n, D)).astype(np.float32)
    gamma = rng.uniform(0.5, 1.5, D).astype(np.float32)
    beta = (0.3 * rng.standard_normal(D)).astype(np.float32)
    pw = (rng.standard_normal(D) / np.sqrt(D)).astype(np.float32)
    pb = 0.1
    if kind == "offset50":
        x += 50.0
    elif kind == "equal":
        x[:] = x[:, :1]
    elif kind in ("dominant", "underflow", "late") and D > 1:
        gw = gamma * pw
        t = n - 1 if kind == "late" else n // 2
        d = (gw - gw.mean()) / np.linalg.norm(gw - gw.mean())
        x[:, t] = (d * np.sqrt(D)).astype(np.float32)             # standardised row along gamma * pw: the largest score
        if kind == "underflow":                                    # that score scaled to 250
            pw = (pw * 250.0 / (np.sqrt(D) * np.linalg.norm(gw - gw.mean()))).astype(np.float32)
    return x, gamma, beta, pw, pb


SEQ_CASES = [(n, D, "random") for n in SEQ_N for D in SEQ_D] + \
            [(n, D, kind) for kind in ("offset50", "dominant", "underflow", "equal", "late") for n, D in
             [(9, 33), (197, 256), (1025, 513), (64, 768), (3, 1024), (17, 129)]]


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("n,D,kind", SEQ_CASES)
def test_seq_pool_against_float64(lib, precision, n, D, kind):
    """The kernel computes in fp32 from the (bf16-rounded) rows: |err| <= 2e-5 * max |ref| per image, against float64 on the same
    rounded rows."""
    from vit_tensorflow_b200 import _lib
    x, gamma, beta, pw, pb = seq_operands(n, D, kind)
    if precision == "bf16":
        x = bf16_round(x)
    got, _ = _lib.op_seq_pool(x, gamma, beta, pw, pb, precision)
    ref = seq_pool_ref(x.astype(np.float64), gamma.astype(np.float64), beta.astype(np.float64), pw, pb)
    assert np.isfinite(got).all()
    scale = np.abs(ref).max(1, keepdims=True)
    assert _worst(np.abs(got - ref), 2e-5 * scale + 1e-30, f"seq_pool n={n} D={D} {kind} {precision}") <= 1.0


@pytest.mark.parametrize("n,D", [(4, 1025), (0, 64)])
def test_seq_pool_refusals(lib, n, D):
    from vit_tensorflow_b200 import _lib
    x = np.zeros((1, n, D), np.float32)
    v = np.ones(D, np.float32)
    with pytest.raises(_lib.VbError, match="seq_pool: needs 0 < dim <= 1024 and at least one token"):
        _lib.op_seq_pool(x, v, v, v, 0.0)


# ------------------------------------------------------------------------------------------------ classifier-head pooling
POOL_LN_CASES = [(1, 64, 64), (197, 768, 768), (49, 384, 448), (3136, 96, 128), (16, 2048, 2048), (5, 100, 164), (3136, 512, 512)]


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("form", ["cls_ln", "mean_ln", "mean"])
@pytest.mark.parametrize("n,D,ldx", POOL_LN_CASES)
def test_pool_layernorm_against_float64(lib, precision, form, n, D, ldx):
    """cls / mean pooling of the first D of ldx columns, with the LayerNorm (eps 1e-3) or without it (LeViT, MobileViT).  The
    kernel sums in fp32 from the (bf16-rounded) rows: |err| <= 2e-5 * max |ref| per image."""
    from vit_tensorflow_b200 import _lib
    rng = np.random.default_rng(n + D + ldx)
    B = 3
    x = (rng.standard_normal((B, n, ldx)) + rng.standard_normal(ldx)).astype(np.float32)   # per-column offsets: pooled spread O(1)
    if precision == "bf16":
        x = bf16_round(x)
    ln = form != "mean"
    gamma = rng.uniform(0.5, 1.5, D).astype(np.float32) if ln else None
    beta = (0.3 * rng.standard_normal(D)).astype(np.float32) if ln else None
    got, _ = _lib.op_pool_layernorm(x, D, gamma, beta, form != "cls_ln", precision)
    x64 = x[..., :D].astype(np.float64)
    z = x64[:, 0] if form == "cls_ln" else x64.mean(1)
    ref = layer_norm(z, gamma.astype(np.float64), beta.astype(np.float64), 1e-3) if ln else z
    scale = np.abs(ref).max(1, keepdims=True)
    assert _worst(np.abs(got - ref), 2e-5 * scale + 1e-30, f"pool_layernorm n={n} D={D} ldx={ldx} {form} {precision}") <= 1.0


# ------------------------------------------------------------------------------------------------ LeViT's strided query gather
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("C,ldi,ldo", [(128, 128, 128), (100, 100, 100), (128, 192, 136), (102, 110, 104)])
@pytest.mark.parametrize("H,W,step", [(7, 9, 2), (14, 14, 2), (1, 5, 2), (6, 5, 1)])
def test_gather_grid_bit_exact(lib, precision, C, ldi, ldo, H, W, step):
    """A copy: bit equality, on the 16-byte path (C and both pitches multiples of 16 bytes' elements: 128) and the scalar one
    (bf16 C = 100; fp32 C = 102), at odd H and W with step 2, and at step 1.  Columns past C keep the output's contents."""
    from vit_tensorflow_b200 import _lib
    rng = np.random.default_rng(C + ldi + H * W + step)
    B = 2
    x = rng.standard_normal((B * H * W, ldi)).astype(np.float32)
    oh, ow = -(-H // step), -(-W // step)
    init = rng.standard_normal((B * oh * ow, ldo)).astype(np.float32)
    if precision == "bf16":
        x, init = bf16_round(x), bf16_round(init)
    got, _ = _lib.op_gather_grid(x, B, H, W, C, step, init, precision)
    want = init.copy()
    want[:, :C] = x.reshape(B, H, W, ldi)[:, ::step, ::step, :C].reshape(-1, C)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))

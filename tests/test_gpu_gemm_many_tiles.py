"""GPU tests of the wgmma GEMM at tile counts of several waves with every epilogue mode.  The other op-level tests reach
more than one wave of 128 x BN tiles only with the plain epilogue; here every mode runs more than two waves of resident
CTAs (132 SMs on the H100, two CTAs per SM for 128-wide tiles) in a tile count that leaves a ragged last wave, K from one
k-block to more k-blocks than the ring has stages (and not a multiple of them), M % 128 in {0, 1, 127} and N in {64, 192, 256, 768, 2304, 3072}.  Values are checked
against float64 on a sample of rows with the bounds of test_gpu_ops.py, and the rows of a large-M call must equal bit for
bit the same rows computed by a small-M call: a result must not depend on which CTA or wave computed its tile.  The small
calls start on a 128-row tile boundary, so every row keeps its position within its tile: on the H100 the wgmma's fp32
result for a row can differ in the last bit when the row sits at another position of the tile (seen in a few elements
per 300 rows, where a residual then cancels most of the value)."""
import numpy as np
import pytest

from cases import bf16_round
from test_gpu_ops import BF16_ATOL, BF16_RTOL, _gelu

pytestmark = pytest.mark.gpu

SMS = 132
# (M, N, K): M % 128 in {0, 1, 127}; K = 64 (one k-block), 128 (fewer k-blocks than the 3 stages of 128-wide tiles), 320
# (5 k-blocks: not a multiple of 3), 768, 1344, 3072 (48 k-blocks, 256-wide tiles)
SHAPES = [(128 * 600, 64, 768), (128 * 280 + 1, 192, 320), (128 * 100 + 127, 768, 64), (128 * 40 + 1, 2304, 128),
          (128 * 30 + 127, 3072, 3072), (128 * 24, 3072, 768), (128 * 300 + 1, 256, 1344)]
MODES = ["plain", "bias_gelu_scale_res", "bias_scale_inplace_res_stats", "ln_fold_gelu", "ln_fold_stats", "f32_out_b_rows"]


def test_shapes_span_several_waves():
    for M, N, K in SHAPES:
        bn = 256 if N % 256 == 0 and K >= 2048 else 128        # gemm_bf16_plan's tile width
        resident = SMS * (1 if bn == 256 else 2)               # 128-wide tiles run two CTAs per SM
        tiles = -(-M // 128) * -(-N // bn)
        assert tiles > 2 * resident and tiles % resident != 0, (M, N, K, tiles)


def _case(M, N, K, mode):
    rng = np.random.default_rng(M + 7 * N + 13 * K + MODES.index(mode))
    a = bf16_round(rng.standard_normal((M, K)).astype(np.float32))
    wt = bf16_round((rng.standard_normal((N, K)) / np.sqrt(K)).astype(np.float32))
    c = dict(a=a, wt=wt, out=np.zeros((M, N), np.float32), kw={})
    bias = (0.5 * rng.standard_normal(N)).astype(np.float32)
    scale = rng.uniform(0.5, 1.5, N).astype(np.float32)
    if mode == "bias_gelu_scale_res":
        c["kw"] = dict(bias=bias, scale=scale, gelu=True, res=bf16_round(rng.standard_normal((M, N)).astype(np.float32)))
    elif mode == "bias_scale_inplace_res_stats":
        c["out"] = bf16_round(rng.standard_normal((M, N)).astype(np.float32))
        c["kw"] = dict(bias=bias, scale=scale, res="out", want_stats=True)
    elif mode.startswith("ln_fold"):
        ch = a.astype(np.float64).reshape(M, K // 64, 64).transpose(1, 0, 2)
        c["kw"] = dict(bias=bias, ln_stats=np.stack([ch.sum(-1), (ch ** 2).sum(-1)], -1).astype(np.float32),
                       ln_c1=wt.astype(np.float64).sum(1).astype(np.float32))
        if mode == "ln_fold_gelu":
            c["kw"]["gelu"] = True
        else:
            c["kw"]["want_stats"] = True
    elif mode == "f32_out_b_rows":
        c["wt"] = wt[:N - 40]                                     # rows [N - 40, N) missing: read as zero
        c["out"] = np.full((M, N), 7.0, np.float32)
        c["kw"] = dict(bias=bias, out_f32=True)
    return c


def _rows(c, lo, hi):
    """the same case restricted to rows [lo, hi)"""
    kw = dict(c["kw"])
    if isinstance(kw.get("res"), np.ndarray):
        kw["res"] = kw["res"][lo:hi]
    if "ln_stats" in kw:
        kw["ln_stats"] = np.ascontiguousarray(kw["ln_stats"][:, lo:hi])
    return dict(a=np.ascontiguousarray(c["a"][lo:hi]), wt=c["wt"], out=np.ascontiguousarray(c["out"][lo:hi]), kw=kw)


def _run(c, N, K):
    from vit_tensorflow_b200 import _lib
    return _lib.op_gemm(c["a"], c["wt"], N, K, c["out"], **c["kw"])[:2]


def _reference(c, N, K, rows, mode):
    a = c["a"][rows].astype(np.float64)
    wt = np.zeros((N, K))
    wt[:c["wt"].shape[0]] = c["wt"]
    acc = a @ wt.T
    kw = c["kw"]
    if "ln_stats" in kw:
        s = kw["ln_stats"][:, rows].astype(np.float64).sum(0)
        mu = s[:, 0] / K
        rstd = 1.0 / np.sqrt(np.maximum(s[:, 1] / K - mu * mu, 0.0) + 1e-3)
        ref = rstd[:, None] * acc - (rstd * mu)[:, None] * kw["ln_c1"].astype(np.float64) + kw["bias"]
    else:
        ref = acc + kw["bias"] if "bias" in kw else acc
    if kw.get("gelu"):
        ref = _gelu(ref)
    if "scale" in kw:
        ref = ref * kw["scale"]
    if isinstance(kw.get("res"), np.ndarray):
        ref = ref + kw["res"][rows]
    elif kw.get("res") == "out":
        ref = ref + c["out"][rows]
    if mode == "f32_out_b_rows":
        bound = K * 2.0 ** -23 * (np.abs(a) @ np.abs(wt).T) + 2.0 ** -23 * np.abs(ref) + 1e-30
    else:
        bound = BF16_ATOL + BF16_RTOL * np.abs(ref)
    return ref, bound


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("M,N,K", SHAPES)
def test_gemm_many_tiles_epilogues(lib, M, N, K, mode):
    c = _case(M, N, K, mode)
    out, stats = _run(c, N, K)
    rng = np.random.default_rng(1)
    rows = np.unique(np.concatenate([[0, 1, 63, 64, 127, 128, M // 2, M - 2, M - 1], rng.integers(0, M, 250)]))
    ref, bound = _reference(c, N, K, rows, mode)
    got = out[rows]
    assert np.isfinite(got).all()
    worst = float((np.abs(got - ref) / bound).max())
    print(f"\n[many tiles {M}x{N}x{K} {mode}] worst err / bound {worst:.3f}")
    assert worst <= 1.0
    if mode == "f32_out_b_rows":
        assert (out[:, N - 40:] == c["kw"]["bias"][N - 40:]).all()       # zero-filled weight rows: exactly the bias
    if stats is not None:
        ch = out.astype(np.float64).reshape(M, N // 64, 64).transpose(1, 0, 2)
        assert (np.abs(stats[..., 0] - ch.sum(-1)) <= 1e-5 * np.abs(ch).sum(-1) + 1e-30).all()
        assert (np.abs(stats[..., 1] - (ch ** 2).sum(-1)) <= 1e-5 * (ch ** 2).sum(-1) + 1e-30).all()
    # the same rows from small-M calls starting at the first and at a middle tile boundary: bit for bit
    for lo in (0, M // 2 // 128 * 128):
        hi = lo + 300
        o2, s2 = _run(_rows(c, lo, hi), N, K)
        np.testing.assert_array_equal(o2, out[lo:hi])
        if stats is not None:
            np.testing.assert_array_equal(s2, stats[:, lo:hi])

"""GPU tests of the wgmma GEMM's TMA epilogue: a bf16 output tile is staged in shared memory over its residual tile (which the
producer warpgroup loads by TMA ahead of the epilogue) and leaves by TMA stores, and the per-column and folded-LayerNorm
per-row operands are staged by the producer warps.  Each consumer warpgroup reuses one staging tile for all of its tiles, so
these cases run many tiles per warpgroup: the shortest main loop (K = 64, one k-block) with an in-place residual, k-block
counts around the 4-stage ring, ragged M (TMA zero-fills the last tile's residual rows and clips its store), a column-offset
output with a separate residual of another leading dimension, and the folded LayerNorm with at least 3 tiles per CTA.
Values are checked against float64 with the bounds of test_gpu_ops.py; rows of a large call must equal bit for bit the same
rows from a small call that starts on a 128-row tile boundary (see test_gpu_gemm_many_tiles.py)."""
import numpy as np
import pytest

from cases import bf16_round
from test_gpu_gemm_many_tiles import _reference, _rows, _run
from test_gpu_ops import BF16_ATOL, BF16_RTOL

pytestmark = pytest.mark.gpu

SMS = 132


def _inplace_case(M, N, K, seed):
    rng = np.random.default_rng(seed)
    a = bf16_round(rng.standard_normal((M, K)).astype(np.float32))
    wt = bf16_round((rng.standard_normal((N, K)) / np.sqrt(K)).astype(np.float32))
    out = bf16_round(rng.standard_normal((M, N)).astype(np.float32))
    kw = dict(bias=(0.5 * rng.standard_normal(N)).astype(np.float32), scale=rng.uniform(0.5, 1.5, N).astype(np.float32),
              res="out", want_stats=True)
    return dict(a=a, wt=wt, out=out, kw=kw)


def _check(c, N, K, out, stats, mode="inplace"):
    M = out.shape[0]
    rows = np.unique(np.concatenate([[0, 1, 63, 64, 127, 128, M // 2, M - 2, M - 1],
                                     np.arange(M - M % 128, M) if M % 128 else [],
                                     np.random.default_rng(1).integers(0, M, 250)]).astype(np.int64))
    ref, bound = _reference(c, N, K, rows, mode)
    got = out[rows]
    assert np.isfinite(got).all()
    worst = float((np.abs(got - ref) / bound).max())
    print(f"\n[tma epilogue {M}x{N}x{K}] worst err / bound {worst:.3f}")
    assert worst <= 1.0
    if stats is not None:
        ch = out.astype(np.float64).reshape(M, N // 64, 64).transpose(1, 0, 2)
        assert (np.abs(stats[..., 0] - ch.sum(-1)) <= 1e-5 * np.abs(ch).sum(-1) + 1e-30).all()
        assert (np.abs(stats[..., 1] - (ch ** 2).sum(-1)) <= 1e-5 * (ch ** 2).sum(-1) + 1e-30).all()


def _check_small_calls(c, N, K, out, stats):
    M = out.shape[0]
    for lo in (0, M // 2 // 128 * 128, (M - 1) // 128 * 128):
        hi = min(lo + 300, M)
        o2, s2 = _run(_rows(c, lo, hi), N, K)
        np.testing.assert_array_equal(o2, out[lo:hi])
        if stats is not None:
            np.testing.assert_array_equal(s2, stats[:, lo:hi])


def test_one_k_block_inplace_residual_many_tiles(lib):
    """K = 64: the shortest main loop, so a warpgroup's staging tile is reused as fast as it can be; ~27 tiles per CTA"""
    M, N, K = 128 * 600, 768, 64
    assert -(-M // 128) * (N // 128) >= 20 * SMS
    c = _inplace_case(M, N, K, 3)
    out, stats = _run(c, N, K)
    _check(c, N, K, out, stats)
    # the same residual as a separate array: bit for bit the in-place result
    sep = dict(c, kw=dict(c["kw"], res=c["out"].copy()), out=np.zeros_like(c["out"]))
    o_sep, s_sep = _run(sep, N, K)
    np.testing.assert_array_equal(o_sep, out)
    np.testing.assert_array_equal(s_sep, stats)
    _check_small_calls(c, N, K, out, stats)


@pytest.mark.parametrize("M,K", [(128 * 200 + 1, 256), (128 * 150 + 127, 320), (128 * 120 + 64, 448), (128 * 90 + 1, 1216)])
def test_ring_depth_and_ragged_m_inplace_residual(lib, M, K):
    """4, 5, 7 and 19 k-blocks through the 4-stage ring; M % 128 in {1, 127, 64}: the last tile's residual rows past M are
    zero-filled and its store clipped"""
    N = 768
    c = _inplace_case(M, N, K, M + K)
    out, stats = _run(c, N, K)
    _check(c, N, K, out, stats)
    _check_small_calls(c, N, K, out, stats)


def test_column_offset_output_separate_residual(lib):
    """out at column offset 64 of a sentinel-filled [M, N + 192] buffer, residual [M, N + 64]: several tiles per warpgroup;
    the columns outside [64, 64 + N) keep the sentinel, and the values equal bit for bit a contiguous call's"""
    from vit_tensorflow_b200 import _lib
    M, N, K, off = 128 * 300 + 5, 384, 192, 64
    rng = np.random.default_rng(11)
    a = bf16_round(rng.standard_normal((M, K)).astype(np.float32))
    wt = bf16_round((rng.standard_normal((N, K)) / np.sqrt(K)).astype(np.float32))
    bias = (0.5 * rng.standard_normal(N)).astype(np.float32)
    res = bf16_round(rng.standard_normal((M, N + 64)).astype(np.float32))
    wide = np.full((M, N + 192), 3.0, np.float32)
    out, stats, _ = _lib.op_gemm(a, wt, N, K, wide, bias=bias, res=res, out_off=off, want_stats=True)
    assert (out[:, :off] == 3.0).all() and (out[:, off + N:] == 3.0).all()
    flat, flat_stats, _ = _lib.op_gemm(a, wt, N, K, np.zeros((M, N), np.float32), bias=bias,
                                       res=np.ascontiguousarray(res[:, :N]), want_stats=True)
    np.testing.assert_array_equal(out[:, off:off + N], flat)
    np.testing.assert_array_equal(stats, flat_stats)
    c = dict(a=a, wt=wt, out=np.zeros((M, N), np.float32), kw=dict(bias=bias, res=np.ascontiguousarray(res[:, :N])))
    _check(c, N, K, flat, None, mode="separate")


def test_folded_layernorm_three_tiles_per_cta(lib):
    """folded LayerNorm (+ GELU): the producer warps reduce the row statistics for every tile of the CTA"""
    M, N, K = 128 * 100 + 3, 2304, 768
    assert -(-M // 128) * (N // 128) >= 3 * SMS
    rng = np.random.default_rng(5)
    a = bf16_round(rng.standard_normal((M, K)).astype(np.float32))
    wt = bf16_round((rng.standard_normal((N, K)) / np.sqrt(K)).astype(np.float32))
    ch = a.astype(np.float64).reshape(M, K // 64, 64).transpose(1, 0, 2)
    kw = dict(bias=(0.5 * rng.standard_normal(N)).astype(np.float32),
              ln_stats=np.stack([ch.sum(-1), (ch ** 2).sum(-1)], -1).astype(np.float32),
              ln_c1=wt.astype(np.float64).sum(1).astype(np.float32), gelu=True)
    c = dict(a=a, wt=wt, out=np.zeros((M, N), np.float32), kw=kw)
    out, _ = _run(c, N, K)
    _check(c, N, K, out, None, mode="ln_fold_gelu")
    _check_small_calls(c, N, K, out, None)

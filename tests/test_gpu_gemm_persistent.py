"""GPU tests of the persistent wgmma GEMM's schedule.  One CTA per SM (132 on the H100) walks the tiles b, b + 132, ... of
the flat 128 x 128 tile order, and its two consumer warpgroups take turns: warpgroup w computes the CTA's tiles i = w
(mod 2), while the producer streams the k-blocks of consecutive tiles through one 6-stage ring.  The shapes below put the
schedule's edges under test: fewer tiles than CTAs, exactly one tile per warpgroup, an odd tile count per CTA (warpgroup 0
takes one more), a ragged last round, one k-block per tile, and k-block counts that are not a multiple of the ring (so
the ring wraps inside a tile and at a tile boundary), each with the plain and the in-place residual + statistics
epilogue; then every epilogue mode at a size where every CTA runs at least 3 tiles.  Values are checked against float64
with the bounds of test_gpu_ops.py, and rows bit for bit against small-M calls that start on a 128-row tile boundary
(test_gpu_gemm_many_tiles.py explains why the start must be tile-aligned)."""
import numpy as np
import pytest

from test_gpu_gemm_many_tiles import MODES, _case, _reference, _rows, _run

pytestmark = pytest.mark.gpu

SMS = 132
STAGES = 6
SCHEDULE = [  # (M, N, K)
    (1, 64, 768), (64, 64, 768), (129, 64, 768),   # fewer tiles than CTAs
    (128 * 132, 256, 768),                          # 264 tiles: one per consumer warpgroup
    (128 * 132, 384, 768),                          # 396 tiles: 3 per CTA
    (128 * 696 + 5, 128, 768),                      # 697 tiles: 5 rounds and a ragged sixth
    (128 * 400 + 1, 128, 64),                       # one k-block per tile
    (128 * 300 + 127, 192, 200),                    # 4 k-blocks, the last one partial
    (128 * 150 + 1, 256, 840),                      # 14 k-blocks, the last one partial
]
EPILOGUE_SHAPE = (128 * 200 + 1, 256, 320)          # 402 tiles: every CTA runs 3 or 4


def _tiles_per_cta(M, N):
    tiles = -(-M // 128) * -(-N // 128)
    ctas = min(tiles, SMS)
    return tiles, ctas, tiles // ctas, tiles % ctas


def test_shapes_cover_the_schedule():
    per_cta = {_tiles_per_cta(M, N)[2:] for M, N, K in SCHEDULE}
    assert any(_tiles_per_cta(M, N)[0] < SMS for M, N, K in SCHEDULE)
    assert (2, 0) in per_cta and (3, 0) in per_cta
    assert any(q >= 3 and r != 0 for q, r in per_cta)
    kbs = {-(-K // 64) for M, N, K in SCHEDULE}
    assert 1 in kbs and any(kb % STAGES != 0 and kb > STAGES for kb in kbs) and any(K % 64 for M, N, K in SCHEDULE)
    assert _tiles_per_cta(*EPILOGUE_SHAPE[:2])[2] >= 3


def _check(M, N, K, mode):
    c = _case(M, N, K, mode)
    out, stats = _run(c, N, K)
    rng = np.random.default_rng(2)
    rows = np.unique(np.clip(np.concatenate([[0, 1, 63, 64, 127, 128, M // 2, M - 2, M - 1], rng.integers(0, M, 250)]), 0, M - 1))
    ref, bound = _reference(c, N, K, rows, mode)
    got = out[rows]
    assert np.isfinite(got).all()
    worst = float((np.abs(got - ref) / bound).max())
    print(f"\n[persistent {M}x{N}x{K} {mode}] worst err / bound {worst:.3f}")
    assert worst <= 1.0
    if mode == "f32_out_b_rows":
        assert (out[:, N - 40:] == c["kw"]["bias"][N - 40:]).all()
    if stats is not None:
        ch = out.astype(np.float64).reshape(M, N // 64, 64).transpose(1, 0, 2)
        assert (np.abs(stats[..., 0] - ch.sum(-1)) <= 1e-5 * np.abs(ch).sum(-1) + 1e-30).all()
        assert (np.abs(stats[..., 1] - (ch ** 2).sum(-1)) <= 1e-5 * (ch ** 2).sum(-1) + 1e-30).all()
    if M <= 300:
        return
    for lo in (0, M // 2 // 128 * 128, (M - 1) // 128 * 128):
        hi = min(lo + 300, M)
        o2, s2 = _run(_rows(c, lo, hi), N, K)
        np.testing.assert_array_equal(o2, out[lo:hi])
        if stats is not None:
            np.testing.assert_array_equal(s2, stats[:, lo:hi])


@pytest.mark.parametrize("mode", ["plain", "bias_scale_inplace_res_stats"])
@pytest.mark.parametrize("M,N,K", SCHEDULE)
def test_gemm_persistent_schedule(lib, M, N, K, mode):
    _check(M, N, K, mode)


@pytest.mark.parametrize("mode", MODES)
def test_gemm_persistent_epilogues(lib, mode):
    _check(*EPILOGUE_SHAPE, mode)

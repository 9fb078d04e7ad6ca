"""GPU tests of the wgmma GEMM's 128 x 192 tile, which gemm_bf16_plan picks when 192 divides N and N >= 1536 (ViT-B/16's
to_qkv at N = 2304 and fc1 at 3072).  Its ring has 3 stages of 40 KB, and each consumer warpgroup holds a whole 128 x 192
tile, so the shapes below put that schedule's edges under test: fewer tiles than CTAs, exactly one tile per warpgroup, an
odd tile count per CTA, a ragged last round, one k-block per tile, k-block counts below, at and across the 3-stage ring
(and not a multiple of it), M % 128 in {0, 1, 127} and N in {1536, 2304, 3072}; then every epilogue mode at a size where
every CTA runs at least 3 tiles, and weight rows past b_rows.  The fp32-output mode keeps the 128-wide tile by the plan's
rule, and its row is here to show that rule holds at N % 192 == 0.  (The hard-swish epilogue is not reachable through
vb_op_gemm, so its 192-wide instance is not run here.)  Values are checked against float64 with the bounds of test_gpu_ops.py, and rows
bit for bit against small-M calls that start on a 128-row tile boundary (test_gpu_gemm_many_tiles.py explains why the
start must be tile-aligned)."""
import numpy as np
import pytest

from cases import bf16_round
from test_gpu_gemm_many_tiles import MODES, _case, _reference, _rows, _run

pytestmark = pytest.mark.gpu

SMS = 132
BN = 192
STAGES = 3
SCHEDULE = [  # (M, N, K)
    (1, 1536, 768), (129, 2304, 64),                 # fewer tiles than CTAs
    (128 * 33, 1536, 192),                           # 264 tiles: one per consumer warpgroup; 3 k-blocks = the ring
    (128 * 32 + 127, 2304, 320),                     # 396 tiles: 3 per CTA; 5 k-blocks
    (128 * 40 + 1, 3072, 3072),                      # 656 tiles: 4 rounds and a ragged fifth; 48 k-blocks
    (128 * 100, 1536, 64),                           # one k-block per tile
    (128 * 60 + 1, 2304, 128),                       # 2 k-blocks: fewer than the ring
    (128 * 50 + 127, 3072, 768),                     # 12 k-blocks
]
EPILOGUE_SHAPE = (128 * 50 + 1, 1536, 320)           # 408 tiles: every CTA runs 3 or 4


def _tiles_per_cta(M, N):
    tiles = -(-M // 128) * -(-N // BN)
    ctas = min(tiles, SMS)
    return tiles, ctas, tiles // ctas, tiles % ctas


def test_shapes_cover_the_schedule():
    assert all(N % BN == 0 and N >= 8 * BN for M, N, K in SCHEDULE + [EPILOGUE_SHAPE])    # gemm_bf16_plan's rule
    assert {N for M, N, K in SCHEDULE} == {1536, 2304, 3072}
    assert {M % 128 for M, N, K in SCHEDULE} == {0, 1, 127}
    per_cta = {_tiles_per_cta(M, N)[2:] for M, N, K in SCHEDULE}
    assert any(_tiles_per_cta(M, N)[0] < SMS for M, N, K in SCHEDULE)
    assert (2, 0) in per_cta and (3, 0) in per_cta
    assert any(q >= 3 and r != 0 for q, r in per_cta)
    kbs = {-(-K // 64) for M, N, K in SCHEDULE}
    assert {1, 2, STAGES, 5, 12, 48} <= kbs
    assert _tiles_per_cta(*EPILOGUE_SHAPE[:2])[2] >= 3


def _check(M, N, K, mode):
    c = _case(M, N, K, mode)
    out, stats = _run(c, N, K)
    rng = np.random.default_rng(3)
    rows = np.unique(np.clip(np.concatenate([[0, 1, 63, 64, 127, 128, M // 2, M - 2, M - 1], rng.integers(0, M, 250)]), 0, M - 1))
    ref, bound = _reference(c, N, K, rows, mode)
    got = out[rows]
    assert np.isfinite(got).all()
    worst = float((np.abs(got - ref) / bound).max())
    print(f"\n[wide tile {M}x{N}x{K} {mode}] worst err / bound {worst:.3f}")
    assert worst <= 1.0
    if mode == "f32_out_b_rows":
        assert (out[:, N - 40:] == c["kw"]["bias"][N - 40:]).all()       # zero-filled weight rows: exactly the bias
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
def test_gemm_wide_tile_schedule(lib, M, N, K, mode):
    _check(M, N, K, mode)


@pytest.mark.parametrize("mode", MODES)
def test_gemm_wide_tile_epilogues(lib, mode):
    _check(*EPILOGUE_SHAPE, mode)


def test_gemm_wide_tile_missing_weight_rows(lib):
    """b_rows < N on the bf16 path: the B box's rows past b_rows are zero-filled, so those output columns are exactly the bias"""
    M, N, K = EPILOGUE_SHAPE
    c = _case(M, N, K, "bias_gelu_scale_res")
    c["wt"] = c["wt"][:N - 40]
    c["kw"] = dict(bias=c["kw"]["bias"])
    out, _ = _run(c, N, K)
    rows = np.arange(0, M, 7)
    ref, bound = _reference(c, N, K, rows, "b_rows")
    assert float((np.abs(out[rows] - ref) / bound).max()) <= 1.0
    assert (out[:, N - 40:] == bf16_round(c["kw"]["bias"][N - 40:])).all()

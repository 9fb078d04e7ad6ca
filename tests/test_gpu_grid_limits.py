"""GPU tests of the launches whose block count grows with the batch, past the 65 535 blocks CUDA allows in gridDim.y and
gridDim.z.  The wgmma GEMM (128-row tiles), the SIMT GEMM (64-row tiles) and the T2T V transpose (one grid slice per image)
take their tile from a flat blockIdx.x, so these sizes run:

  wgmma GEMM    M = 8 388 481 rows: 65 536 row tiles, the last holding one row
  SIMT GEMM     M = 4 194 305 rows: 65 537 row tiles of 64
  T2T           t2t_small at batch 65 664: its first soft-split layer runs GEMMs on 256 rows per image (131 328 row tiles)
                and transposes V once per image (65 664 > 65 535)
  ViT           vit_odd_dims (widths off the wgmma path) at batch 116 608: 36 rows per image, 65 592 SIMT row tiles

Every row of the GEMMs is checked.  Small-integer operands make the plain products exact in float64 and in the kernels' fp32
accumulators, so those outputs must equal the reference bit for bit.  The model cases compare a few images with the oracle,
and require the last 128 images to equal, bit for bit, the same images run as a batch of their own."""
import numpy as np
import pytest

import oracle
from cases import bf16_round, cfg_of
from test_gpu_models import BF16_ATOL as MODEL_ATOL, BF16_RTOL as MODEL_RTOL
from test_gpu_ops import BF16_ATOL, BF16_RTOL, _gelu

pytestmark = pytest.mark.gpu

WGMMA_M = 128 * 65535 + 1                                     # 8 388 481: 65 536 tiles of 128 rows, the last with one row
SIMT_M = 64 * 65536 + 1                                       # 4 194 305: 65 537 tiles of 64 rows
CHUNK = 1 << 20


def _small_ints(rng, shape, lo, hi, div=1.0):
    return (rng.integers(lo, hi + 1, shape, dtype=np.int8).astype(np.float32) / np.float32(div))


@pytest.mark.parametrize("epi", ["plain", "bias_gelu_res"])
def test_wgmma_gemm_past_65535_row_tiles(lib, epi):
    from vit_tensorflow_b200 import _lib
    M, N, K = WGMMA_M, 64, 64
    assert -(-M // 128) == 65536 and M % 128 == 1
    rng = np.random.default_rng(5)
    a = _small_ints(rng, (M, K), -4, 4)                       # exact in bf16
    wt = _small_ints(rng, (N, K), -2, 2, 4.0)                 # K-major [N, K], quarters: exact in bf16
    kw = {}
    if epi != "plain":
        kw = dict(bias=rng.standard_normal(N).astype(np.float32), gelu=True,
                  res=bf16_round(rng.standard_normal((M, N), dtype=np.float32)))
    out, _, _ = _lib.op_gemm(a, wt, N, K, np.zeros((M, N), np.float32), **kw)
    w64 = wt.T.astype(np.float64)
    worst = 0.0
    for lo in range(0, M, CHUNK):
        hi = min(M, lo + CHUNK)
        acc = a[lo:hi].astype(np.float64) @ w64                # |acc| <= 128 in quarters: exact in fp32
        if epi == "plain":
            np.testing.assert_array_equal(out[lo:hi], bf16_round(acc.astype(np.float32)), err_msg=f"rows [{lo}, {hi})")
        else:
            ref = _gelu(acc + kw["bias"]) + kw["res"][lo:hi]
            worst = max(worst, float((np.abs(out[lo:hi] - ref) / (BF16_ATOL + BF16_RTOL * np.abs(ref))).max()))
    print(f"\n[wgmma GEMM M = {M} {epi}] worst err / bound {worst:.3f}")
    assert worst <= 1.0


def test_simt_gemm_past_65535_row_tiles(lib):
    """The fp32 engine's GEMM (vb_op_linear, fp32): small integers with bias and residual, exact in fp32, every row."""
    from vit_tensorflow_b200 import _lib
    M, N, K = SIMT_M, 64, 16
    assert -(-M // 64) == 65537
    rng = np.random.default_rng(6)
    a = _small_ints(rng, (M, K), -4, 4)
    w = _small_ints(rng, (K, N), -2, 2, 4.0)
    bias = _small_ints(rng, (N,), -8, 8, 2.0)
    res = _small_ints(rng, (M, N), -8, 8)
    out, _ = _lib.op_linear(a, w, bias, None, res, False, "fp32")
    w64 = w.astype(np.float64)
    for lo in range(0, M, CHUNK):
        hi = min(M, lo + CHUNK)
        ref = a[lo:hi].astype(np.float64) @ w64 + bias + res[lo:hi]
        np.testing.assert_array_equal(out[lo:hi], ref.astype(np.float32), err_msg=f"rows [{lo}, {hi})")


@pytest.mark.parametrize("name,batch", [("t2t_small", 65664), ("vit_odd_dims", 116608)])
def test_bf16_model_batch_past_grid_limits(lib, name, batch):
    from vit_tensorflow_b200 import from_config
    assert batch % 128 == 0
    cfg = cfg_of(name)
    w = oracle.stress_weights(cfg, 11)
    img = oracle.make_image(cfg, batch, 12)
    m = from_config(cfg, precision="bf16")
    m.set_weights_dict(w)
    got = np.asarray(m(img, training=False))
    assert got.shape == (batch, cfg["num_classes"]) and np.isfinite(got).all()
    idx = np.array([0, 1, batch // 2, batch - 129, batch - 1])
    ref = oracle.forward_numpy(img[idx], w, cfg)
    err = np.abs(got[idx] - ref)
    assert (err <= MODEL_ATOL + MODEL_RTOL * np.abs(ref)).all(), f"max err {err.max():.4f}"
    # the tail starts on a 128-image boundary, so every row keeps its position within its GEMM tile in both runs
    tail = np.asarray(m(np.ascontiguousarray(img[-128:]), training=False))
    np.testing.assert_array_equal(got[-128:], tail)

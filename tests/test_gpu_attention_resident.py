"""GPU tests of the resident-head form of the flash attention (attn_flash.cu, attn_resident_kernel): plain bf16 attention with
dim_head 64 and at most 256 keys, each (image, head, query chunk of up to 256 rows) unit's Q, K and V loaded once by TMA into a
persistent CTA.  Each case is checked against the float64 reference at the bounds of test_gpu_ops.py and asserts the "flash"
path; nk = 257 takes the streaming flash kernel and must still be right.  The cases cover the key counts around the 16-key
padding and the 64-key softmax blocks, query chunks past 256 rows, separate and fused operand rows with their own pitches,
grids with fewer units than SMs and unit counts that do not divide by the grid, and the bitwise determinism of a call."""
import numpy as np
import pytest

from cases import bf16_round
from test_gpu_attention_paths import served_by  # noqa: F401 (fixture)
from test_gpu_ops import ATTN_BF16_REL, ATTN_BF16_SIGMA, _assert_close_sigma, _attention_ref

pytestmark = pytest.mark.gpu

DH = 64


def _qkv(rng, B, nq, nk, heads):
    inner = heads * DH
    q = bf16_round(rng.standard_normal((B, nq, inner), dtype=np.float32))
    k = bf16_round(rng.standard_normal((B, nk, inner), dtype=np.float32))
    v = bf16_round(rng.standard_normal((B, nk, inner), dtype=np.float32))
    return q, k, v


def _check(served_by, B, nq, nk, heads):
    from vit_tensorflow_b200 import _lib
    rng = np.random.default_rng([B, nq, nk, heads])
    q, k, v = _qkv(rng, B, nq, nk, heads)
    out, _ = served_by(lambda: _lib.op_attention(q, k, v, heads, 0, precision="bf16"), "flash")
    assert np.isfinite(out).all()
    _assert_close_sigma(out, _attention_ref(q, k, v, heads, 0, None, None, None, None), ATTN_BF16_SIGMA[0], ATTN_BF16_REL)


@pytest.mark.parametrize("n", [2, 15, 16, 17, 63, 64, 65, 191, 197, 255, 256, 257])
def test_resident_self_attention(lib, served_by, n):
    """nq = nk = n: one to four 64-key blocks, the last partial at every offset of the 16-key padding; 257 keys exceed the
    resident form and run on the streaming kernel."""
    _check(served_by, 2, n, n, 3)


@pytest.mark.parametrize("B,nq,nk,heads", [(1, 3136, 64, 1),     # Twins-SVT stage-1 global attention: 13 query chunks
                                           (2, 784, 196, 2),     # 4 chunks, the last of 16 rows
                                           (2, 257, 200, 2),     # a last chunk of a single row
                                           (3, 5, 250, 2),       # fewer queries than one 16-row slice
                                           (2, 300, 37, 3)])
def test_resident_cross_shapes(lib, served_by, B, nq, nk, heads):
    _check(served_by, B, nq, nk, heads)


@pytest.mark.parametrize("B,heads,n", [(1, 2, 197),     # two units on a grid of as many CTAs
                                       (100, 3, 197)])  # 300 units: not a multiple of the SM count
def test_resident_grid_fill(lib, served_by, B, heads, n):
    _check(served_by, B, n, n, heads)


def test_resident_separate_pitches(lib, served_by):
    """q rows of pitch inner + 24, k and v at columns 8 and inner + 16 of [k|v] rows of pitch 2 inner + 40, output rows of
    pitch inner + 8: every operand with its own pitch; the output columns outside the heads keep their contents."""
    from vit_tensorflow_b200 import _lib
    rng = np.random.default_rng(7)
    B, nq, nk, heads = 3, 150, 197, 2
    inner = heads * DH
    q = bf16_round(rng.standard_normal((B, nq, inner + 24), dtype=np.float32))
    kv = bf16_round(rng.standard_normal((B, nk, 2 * inner + 40), dtype=np.float32))
    init = bf16_round(rng.standard_normal((B, nq, inner + 8), dtype=np.float32))
    out, _ = served_by(lambda: _lib.op_attention_ex(q, heads, DH, init, kv=kv, k_off=8, v_off=inner + 16), "flash")
    assert (out[..., inner:] == init[..., inner:]).all()
    ref = _attention_ref(q[..., :inner], kv[..., 8:8 + inner], kv[..., inner + 16:2 * inner + 16], heads, 0, None, None, None, None)
    _assert_close_sigma(out[..., :inner], ref, ATTN_BF16_SIGMA[0], ATTN_BF16_REL)


def test_resident_fused_wide_rows(lib, served_by):
    """q | k | v in rows of pitch 3 inner + 64 (Twins-SVT writes its projections into wider rows in place)."""
    from vit_tensorflow_b200 import _lib
    rng = np.random.default_rng(8)
    B, n, heads = 2, 197, 3
    inner = heads * DH
    rows = bf16_round(rng.standard_normal((B, n, 3 * inner + 64), dtype=np.float32))
    out, _ = served_by(lambda: _lib.op_attention_ex(rows, heads, DH, np.zeros((B, n, inner), np.float32), k_off=inner,
                                                    v_off=2 * inner), "flash")
    ref = _attention_ref(rows[..., :inner], rows[..., inner:2 * inner], rows[..., 2 * inner:3 * inner], heads, 0, None, None, None, None)
    _assert_close_sigma(out, ref, ATTN_BF16_SIGMA[0], ATTN_BF16_REL)


def test_resident_batch_independent_and_deterministic(lib):
    """The last images of a batch give bit for bit what they give as a batch of their own (no unit reads another image's rows,
    whatever CTA runs it), and two identical calls give identical bits."""
    from vit_tensorflow_b200 import _lib
    rng = np.random.default_rng(9)
    B, n, heads = 70, 197, 4
    q, k, v = _qkv(rng, B, n, n, heads)
    whole, _ = _lib.op_attention(q, k, v, heads, 0, precision="bf16")
    again, _ = _lib.op_attention(q, k, v, heads, 0, precision="bf16")
    tail, _ = _lib.op_attention(q[-3:], k[-3:], v[-3:], heads, 0, precision="bf16")
    assert np.array_equal(whole, again)
    assert np.array_equal(whole[-3:], tail)

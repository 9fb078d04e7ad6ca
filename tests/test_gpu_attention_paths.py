"""GPU tests of every branch of the attention dispatch, each against the float64 reference, each asserting which kernels ran.

The dispatch (attention_fast in attn_flash.cu, attention_cls in attn_cls.cu, attention_generic_mma / attention_rows_path in
attn_generic_mma.cu, the SIMT kernels of attention.cu) picks a path from the precision, variant, nq, nk, heads and dim_head:

  flash      bf16, variant 0, dim_head 64, nq >= 2                   attn_flash_kernel
  cls        bf16, nq == 1, dim_head % 8 == 0, scores in shared memory attn_cls_kernel
  rows       bf16, variants 1 / 2, 8 or 16 heads, nk <= 256          scores_stripe_kernel, mid_rows_kernel<H, JS, V, WPR>, pv_rows_kernel
  mid_fused  bf16, dim_head % 16 == 0 and <= 128, heads <= 32, every head's score row in 200 KB of shared memory
                                                                      scores_mma_kernel, mid_fused_kernel, pv_mma_kernel
  simt       everything else, and every fp32 call                     attn_scores_kernel, attn_softmax_kernel, attn_pv_kernel
                                                                      (+ attn_head_mix_kernel for variants 1 and 2)

A case that silently took another branch would test another kernel, so each case asks the library which branch served its
call (vb_last_attention_path) and requires the one it names.  Bounds are those of test_gpu_ops.py.  The model
cases at the end run the dim_head > 64 and 384^2 configurations of cases.MID on the fp32 engine at the gate tolerance."""
import numpy as np
import pytest

import oracle
from cases import bf16_round, cfg_of
from test_gpu_ops import ATTN_BF16_REL, ATTN_BF16_SIGMA, _assert_close_sigma, _attention_ref

pytestmark = pytest.mark.gpu


@pytest.fixture
def served_by():
    """served_by(fn, path) -> fn()'s result, after asserting that the attention call inside fn was served by `path`'s kernels.
    The branch that launches notes itself (vb_last_attention_path, per thread, reset by reading); a call that ran no
    attention fails rather than passing vacuously."""
    from vit_tensorflow_b200 import _lib

    def run(fn, path):
        _lib.last_attention_path()                    # forget this thread's earlier calls
        result = fn()
        got = _lib.last_attention_path()
        assert got is not None, "no attention call recorded its path: the path check would pass vacuously"
        assert got == path, f"expected the {path} path, the call took the {got} path"
        return result
    return run


def _operands(rng, B, nq, nk, heads, dh, variant, precision):
    rnd = bf16_round if precision == "bf16" else (lambda t: t)
    inner = heads * dh
    q = rnd(rng.standard_normal((B, nq, inner), dtype=np.float32))
    k = rnd(rng.standard_normal((B, nk, inner), dtype=np.float32))
    v = rnd(rng.standard_normal((B, nk, inner), dtype=np.float32))
    mix_a = rng.standard_normal((heads, heads)).astype(np.float32) if variant else None
    mix_b = rng.standard_normal((heads, heads)).astype(np.float32) if variant == 2 else None
    g = rng.uniform(0.5, 1.5, heads).astype(np.float32) if variant == 1 else None
    b = rng.standard_normal(heads).astype(np.float32) if variant == 1 else None
    return q, k, v, mix_a, mix_b, g, b


def _check_case(served_by, path, precision, variant, B, nq, nk, heads, dh):
    from vit_tensorflow_b200 import _lib
    rng = np.random.default_rng([B, nq, nk, heads, dh, variant])
    q, k, v, ma, mb, g, b = _operands(rng, B, nq, nk, heads, dh, variant, precision)
    out, _ = served_by(lambda: _lib.op_attention(q, k, v, heads, variant, ma, mb, g, b, precision), path)
    ref = _attention_ref(q, k, v, heads, variant, ma, mb, g, b)
    assert np.isfinite(out).all()
    if precision == "fp32":
        np.testing.assert_allclose(out, ref, rtol=2e-4, atol=2e-4)
    else:
        _assert_close_sigma(out, ref, ATTN_BF16_SIGMA[variant], ATTN_BF16_REL)


# ------------------------------------------------------------------------------------------------------------ bf16 cases
# (path, variant, B, nq, nk, heads, dh)
MID_FUSED = (
    # dim_head 80-128 (the MAXDH = 128 fragment / accumulator arrays of scores_mma and pv_mma fully used at 128), heads 2-6
    [("mid_fused", var, 2, nq, nq, heads, dh) for var in (0, 1, 2) for dh, heads in ((80, 5), (96, 3), (112, 6), (128, 2))
     for nq in (197, 65)]
    # 8 and 16 heads past the rows path's 256 keys (DeepViT / CaiT at 384^2), and 17-32 heads
    + [("mid_fused", var, 1, nk, nk, heads, 32) for var in (1, 2) for heads in (8, 16) for nk in (257, 577)]
    + [("mid_fused", var, 1, 197, 197, heads, 16) for var in (0, 1, 2) for heads in (24, 32)]
    # 16 heads x 3168 keys + the two mix matrices fill mid_fused's 200 KB exactly; one key more falls back to the SIMT kernels
    + [(path, var, 1, 5, nk, 16, 80) for var in (0, 1, 2) for nk, path in ((3168, "mid_fused"), (3169, "simt"))]
)
# dim_head 80 / 112: the last ldmatrix.x4 of scores_stripe_kernel's B fragments reads past the head (its result unused)
ROWS = [("rows", var, 1, nk, nk, heads, dh) for var in (1, 2) for heads in (8, 16) for dh in (80, 96, 112, 128) for nk in (197, 256)]
SIMT = ([("simt", var, 2, 65, 197, 4, dh) for var in (0, 1, 2) for dh in (8, 24, 40, 72)]       # dim_head % 16 != 0
        + [("simt", var, 1, 65, 65, 2, dh) for var in (0, 1, 2) for dh in (160, 256)]        # dim_head > 128
        + [("simt", 0, 1, 65, 65, 40, 80)])                                                  # > 32 heads, no head mix
CLS = ([("cls", var, 3, 1, nk, 4, dh) for var in (0, 1, 2) for dh in (8, 24, 80, 128) for nk in (1, 2, 197, 577)]
       + [("cls", 0, 3, 1, 197, 40, 32)]
       # variant 2, 16 heads x 64: 1551 keys fit attn_cls's 200 KB of shared memory, 1552 fall back to mid_fused
       + [(path, 2, 2, 1, nk, 16, 64) for nk, path in ((1551, "cls"), (1552, "mid_fused"))])
FLASH = [("flash", 0, 2, 197, 197, 3, 64)]
BF16_CASES = FLASH + MID_FUSED + ROWS + SIMT + CLS


def _id(c):
    return f"{c[0]}-v{c[1]}-B{c[2]}-nq{c[3]}-nk{c[4]}-h{c[5]}-dh{c[6]}"


@pytest.mark.parametrize("case", BF16_CASES, ids=_id)
def test_attention_path_bf16(lib, served_by, case):
    path, variant, B, nq, nk, heads, dh = case
    _check_case(served_by, path, "bf16", variant, B, nq, nk, heads, dh)


# ------------------------------------------------------------------------------------------------------------ fp32 cases
# every dim_head and head count above once; the fp32 engine always takes the exact SIMT kernels
FP32_CASES = [
    (0, 2, 65, 65, 5, 80), (1, 2, 197, 197, 3, 96), (2, 1, 65, 65, 6, 112), (1, 1, 197, 197, 2, 128),
    (2, 1, 257, 257, 8, 32), (1, 1, 577, 577, 16, 16), (2, 1, 197, 197, 24, 16), (1, 1, 197, 197, 32, 16),
    (0, 1, 5, 3169, 16, 80), (2, 2, 65, 197, 4, 8), (1, 2, 65, 197, 4, 24), (0, 2, 65, 197, 4, 40), (2, 2, 65, 197, 4, 72),
    (1, 1, 65, 65, 2, 160), (2, 1, 65, 65, 2, 256), (0, 1, 65, 65, 40, 80),
    (2, 3, 1, 577, 4, 128), (1, 3, 1, 1, 4, 24), (0, 3, 1, 197, 40, 32), (2, 2, 1, 1551, 16, 64),
]


@pytest.mark.parametrize("case", FP32_CASES, ids=lambda c: f"v{c[0]}-B{c[1]}-nq{c[2]}-nk{c[3]}-h{c[4]}-dh{c[5]}")
def test_attention_path_fp32(lib, served_by, case):
    variant, B, nq, nk, heads, dh = case
    _check_case(served_by, "simt", "fp32", variant, B, nq, nk, heads, dh)


# ----------------------------------------------------------------------------------------------------------------- refusal
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("variant", [1, 2])
def test_head_mix_refuses_more_than_32_heads(lib, variant, precision):
    """The head mixes hold a query's 32 head values in registers: 33 heads is an error that names the limit, with no
    output, and the library stays usable."""
    from vit_tensorflow_b200 import _lib
    rng = np.random.default_rng(33 + variant)
    q, k, v, ma, mb, g, b = _operands(rng, 2, 5, 5, 33, 16, variant, precision)
    with pytest.raises(_lib.VbError, match="at most 32 heads"):
        _lib.op_attention(q, k, v, 33, variant, ma, mb, g, b, precision)
    q, k, v, ma, mb, g, b = _operands(rng, 2, 5, 5, 32, 16, variant, precision)
    out, _ = _lib.op_attention(q, k, v, 32, variant, ma, mb, g, b, precision)
    assert np.isfinite(out).all()


# ------------------------------------------------------------------------------------------------------------ model cases
FP32_MODELS = ["vit_dh80_p14", "vit_dh128", "deepvit_384_h8", "deepvit_384_h16", "cait_384_h8", "cait_384_h16", "cait_dh128"]


@pytest.mark.parametrize("name", FP32_MODELS)
def test_fp32_model_vs_oracle(lib, name):
    """The dim_head > 64 and 384^2 configurations that test_bf16_vs_oracle runs on the bf16 engine, on the fp32 engine at the
    gate tolerance."""
    from vit_tensorflow_b200 import from_config
    cfg = cfg_of(name)
    w = oracle.stress_weights(cfg, 11)
    img = oracle.make_image(cfg, 2, 12)
    m = from_config(cfg, precision="fp32")
    m.set_weights_dict(w)
    got = m(img, training=False)
    np.testing.assert_allclose(got, oracle.forward_numpy(img, w, cfg), rtol=1e-3, atol=1e-4)

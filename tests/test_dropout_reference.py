"""CPU: training-mode dropout's stream and its oracle (tests/dropout_oracle.py), and the host refusal rules.

* The mask function restated element by element from Philox4x32-10 (whose known answers tests/test_ats_vit_reference.py checks).
* LIVE (skipped where the reference checkout is absent): the unmodified reference classes over the numpy stand-in, their Dropout
  drawing from the stream, equal the numpy spec to 1e-12 in float64 at draws 0 and 1, which pins every case's site numbering to
  the reference's own call order.
* The committed fixtures equal the spec."""
import os

import numpy as np
import pytest

import dropout_oracle as o
import fake_engine
from ats_oracle import philox4x32_10

REF_DIR = os.environ.get("VB_REFERENCE_DIR", "/root/reference/vit_tensorflow")    # the reference checkout (absent on the GPU box)
live = pytest.mark.skipif(not os.path.isdir(REF_DIR), reason="reference checkout not present (GPU box): fixtures cover it")
GOLDEN = os.path.join(os.path.dirname(__file__), "golden")


@pytest.mark.parametrize("seed,draw,site", [(0, 0, 0), (o.SEED, 1, 5), (2 ** 64 - 1, 2 ** 32 - 1, 2 ** 32 - 1)])
def test_mask_is_the_stated_philox_word(seed, draw, site):
    M, N, rate = 37, 11, 0.3
    keep = o.keep_mask(seed, draw, site, M, N, rate)
    for m in range(M):
        for n in range(N):
            x = philox4x32_10(np.array([[n >> 1, ((m >> 4) << 3) | (m & 7), site, draw]], np.uint64), (seed & 0xFFFFFFFF, seed >> 32))[0]
            u = int(x[2 * ((m >> 3) & 1) + (n & 1)]) >> 8
            assert keep[m, n] == (u * 2.0 ** -24 >= np.float32(rate))


def test_one_block_covers_the_epilogue_fragment():
    """Rows m, m + 8 (m % 16 < 8) and columns n, n + 1 (n even) read the four words of one Philox block."""
    keep = o.keep_mask(o.SEED, 0, 3, 32, 8, 0.5)
    x = philox4x32_10(np.array([[1, 8 + 3, 3, 0]], np.uint64), (o.SEED & 0xFFFFFFFF, o.SEED >> 32))[0]     # m = 16 + 3, n = 2
    words = [(int(w) >> 8) * 2.0 ** -24 >= 0.5 for w in x]
    assert [keep[19, 2], keep[19, 3], keep[27, 2], keep[27, 3]] == words


@pytest.mark.parametrize("rate", [0.1, 0.5, 0.9])
def test_keep_fraction_within_5_sigma(rate):
    n = 1 << 20
    kept = o.keep_mask(o.SEED, 0, 1, 1024, 1024, rate).sum()
    p = 1.0 - rate
    assert abs(kept - n * p) <= 5.0 * np.sqrt(n * p * (1 - p))


def test_sites_are_independent_of_other_rates_and_rate_zero_is_identity():
    x = np.random.default_rng(0).standard_normal((2, 9, 64))
    a = o.apply(x, o.SEED, 0, 4, 0.3)
    np.testing.assert_array_equal(a, o.apply(x, o.SEED, 0, 4, 0.3))                       # a function of (site, draw, m, n) only
    assert not np.array_equal(a, o.apply(x, o.SEED, 0, 5, 0.3))
    assert o.apply(x, o.SEED, 0, 4, 0.0) is x
    # a case whose emb_dropout is 0: its other sites keep the masks they have when emb_dropout is set
    s0 = o._Sites(o.SEED, 0)
    s1 = o._Sites(o.SEED, 0)
    s0(x, 0.0), s1(x, 0.2)
    np.testing.assert_array_equal(s0(x, 0.1), s1(x, 0.1))


@live
@pytest.mark.parametrize("name", sorted(o.CASES))
@pytest.mark.parametrize("gen", o.WEIGHTS)
def test_live_reference_equals_the_spec(name, gen):
    for d in (0, 1):
        got, calls = o.reference(REF_DIR, name, gen, d)
        assert calls == o.site_count(name)
        np.testing.assert_allclose(got, o.spec(name, gen, d), rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("name", sorted(o.CASES))
@pytest.mark.parametrize("gen", o.WEIGHTS)
def test_fixture_equals_the_spec(name, gen):
    z = np.load(os.path.join(GOLDEN, o.fixture_name(name, gen)))
    assert int(z["seed"]) == o.SEED
    for d in (0, 1):
        spec = o.spec(name, gen, d)
        np.testing.assert_allclose(z[f"logits_d{d}_f64"], spec, rtol=1e-12, atol=1e-12)
        np.testing.assert_allclose(z[f"logits_d{d}_f32"], spec, rtol=1e-4, atol=1e-4)
    assert not np.allclose(z["logits_d0_f64"], z["logits_d1_f64"])


def _vit(**kw):
    from vit_tensorflow_b200 import ViT
    return ViT(image_size=32, patch_size=16, num_classes=4, dim=64, depth=1, heads=2, mlp_dim=64, dim_head=32, precision="fp32", **kw)


def test_host_refusals_over_the_double():
    img = np.zeros((1, 32, 32, 3), np.float32)
    with fake_engine.installed():
        from vit_tensorflow_b200 import CaiT, CrossViT, DeepViT, DistillableViT, ParallelViT, T2TViT, ViT
        m = _vit(dropout=0.1)
        with pytest.raises(NotImplementedError):
            m(img)                                             # no seed: today's refusal
        m.set_dropout_seed(1)
        m.set_dropout_seed(None)
        with pytest.raises(NotImplementedError):
            m(img)
        for bad in (1.0, 1.5, -0.1):
            b = _vit(dropout=bad)
            b.set_dropout_seed(0)
            with pytest.raises(ValueError):
                b(img)                                         # tf.nn.dropout refuses the rate at the call
            b(img, training=False)                             # Keras' Dropout never looks at it at inference
        e = _vit(emb_dropout=1.0)
        e.set_dropout_seed(0)
        with pytest.raises(ValueError):
            e(img)
        d = DistillableViT(image_size=32, patch_size=16, num_classes=4, dim=64, depth=1, heads=2, mlp_dim=64, dropout=0.1,
                           precision="fp32")
        with pytest.raises(NotImplementedError):
            d.set_dropout_seed(0)
        for cls in (ViT, DeepViT, CaiT, CrossViT):
            assert callable(getattr(cls, "set_dropout_seed"))
        for cls in (ParallelViT, T2TViT):
            assert not hasattr(cls, "set_dropout_seed")


def test_abi_declares_and_binds_the_new_entries():
    from vit_tensorflow_b200 import _lib
    header = open(os.path.join(os.path.dirname(os.path.dirname(__file__)), "include", "vitb200.h")).read()
    for fn in ("vb_set_dropout", "vb_forward_train", "vb_op_dropout_mask"):
        assert f"VB_API int {fn}(" in header and fn in _lib.SIGNATURES

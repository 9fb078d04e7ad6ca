"""GPU: DistillableT2TViT (reference distill.py:61-72) through vb_forward_distill on a T2TViT handle, against the reference's own
outputs (tests/golden/t2t_distill_*__refshim.npz, made by make_distill_golden.py) and the float64 restatement of distill_oracle.

fp32 engine: rtol 1e-3 / atol 1e-4, as every fp32 gate.  bf16 engine: the tolerances the existing tests hold the same paths to --
T2TViT's logits to test_gpu_models.py's (t2t_small) at the small sizes and to test_gpu_config_size.T2T_README_TOL for the README
model, the distillation row to test_gpu_models.test_distillable_vit_forward's.
"""
import ctypes as C
import os

import numpy as np
import pytest

import distill_oracle as do
import oracle
from test_gpu_config_size import T2T_README_TOL
from test_gpu_models import BF16_ATOL, BF16_RTOL

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")


def _kw(name):
    return {k: v for k, v in do.CASES[name].items() if k != "kind"}


def _model(name, precision, weights, cls="DistillableT2TViT", **kw):
    import vit_tensorflow_b200 as vb
    m = getattr(vb, cls)(**{**_kw(name), **kw}, precision=precision)
    m.set_weights_dict(weights)
    return m


def _within(got, ref, atol, rtol):
    err = np.abs(got - ref)
    assert np.isfinite(got).all()
    assert (err <= atol + rtol * np.abs(ref)).all(), f"max err {err.max():.4g}, worst ratio {(err / (atol + rtol * np.abs(ref))).max():.3f}"


@pytest.mark.parametrize("gen", do.WEIGHTS)
@pytest.mark.parametrize("name", list(do.CASES))
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_distillable_t2t_matches_the_reference_fixtures(lib, precision, name, gen):
    cfg, w, img, tok = do.inputs(name, gen)
    z = np.load(os.path.join(GOLDEN, do.fixture_name(name, gen)))
    m = _model(name, precision, w)
    logits, dist = m(img, distill_token=tok, training=False)
    assert logits.shape == (do.BATCH, cfg["num_classes"]) and dist.shape == (do.BATCH, cfg["dim"])
    assert logits.dtype == dist.dtype == np.float32
    ref_l, ref_d = z["logits_ref_f64"], z["distill_ref_f64"]
    if precision == "fp32":
        np.testing.assert_allclose(logits, ref_l, rtol=1e-3, atol=1e-4)
        np.testing.assert_allclose(dist, ref_d, rtol=1e-3, atol=1e-4)
    else:
        atol, rtol = T2T_README_TOL if name == "t2t_distill_readme" else (BF16_ATOL, BF16_RTOL)
        _within(logits, ref_l, atol, rtol)
        _within(dist, ref_d, BF16_ATOL, BF16_RTOL)


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_without_a_token_the_call_is_t2t_vit(lib, precision):
    """DistillMixin.call without a token is T2TViT.call: bit for bit the plain model's forward on the same weights."""
    _, w, img, _ = do.inputs("t2t_distill_4layers", "stress_weights")
    m = _model("t2t_distill_4layers", precision, w)
    plain = _model("t2t_distill_4layers", precision, w, cls="T2TViT")
    np.testing.assert_array_equal(m(img, training=False), plain(img, training=False))
    np.testing.assert_array_equal(m(img), plain(img))


@pytest.mark.parametrize("name", ["t2t_distill_cls", "t2t_distill_readme"])
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_repeated_calls_are_bit_identical(lib, precision, name):
    """At the README size the bf16 soft-split layers fork images onto side streams; the results still do not change."""
    _, w, img, tok = do.inputs(name, "stress_weights")
    m = _model(name, precision, w)
    first = m(img, distill_token=tok, training=False)
    m(img, training=False)                                        # a plain forward in between reuses the same workspace
    for _ in range(2):
        again = m(img, distill_token=tok, training=False)
        for a, b in zip(first, again):
            np.testing.assert_array_equal(a, b)


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_smaller_image_than_image_size(lib, precision):
    """pos_embedding[:, :(n + 1)] (distill.py:24): a 24 x 24 image on a 32 x 32 model."""
    cfg, w, _, tok = do.inputs("t2t_distill_4layers", "stress_weights")
    img = oracle.make_image(cfg, 3, 5, h=24, w=24)
    m = _model("t2t_distill_4layers", precision, w)
    logits, dist = m(img, distill_token=tok, training=False)
    ref_l, ref_d = do.forward_distill(img, tok, w, cfg)
    if precision == "fp32":
        np.testing.assert_allclose(logits, ref_l, rtol=1e-3, atol=1e-4)
        np.testing.assert_allclose(dist, ref_d, rtol=1e-3, atol=1e-4)
    else:
        _within(logits, ref_l, BF16_ATOL, BF16_RTOL)
        _within(dist, ref_d, BF16_ATOL, BF16_RTOL)


def test_injected_transformer_gives_the_engine_path(lib):
    """DistillableT2TViT(transformer=<another engine model's .transformer>): the call composed on the host around it gives what the
    engine's own distillation path gives, within bf16 tolerance."""
    _, w, img, tok = do.inputs("t2t_distill_cls", "stress_weights")
    m = _model("t2t_distill_cls", "bf16", w)
    ref_l, ref_d = m(img, distill_token=tok, training=False)
    inj = _model("t2t_distill_cls", "bf16", {k: v for k, v in w.items() if not k.startswith("layers.")}, transformer=m.transformer)
    logits, dist = inj(img, distill_token=tok, training=False)
    _within(logits, ref_l, BF16_ATOL, BF16_RTOL)
    _within(dist, ref_d, BF16_ATOL, BF16_RTOL)


def test_refusals(lib):
    """A depth-0 T2TViT handle (built for an injected transformer) holds no transformer and is refused with a message that says so;
    kinds without a distillation path keep their refusal."""
    from vit_tensorflow_b200 import DeepViT, T2TViT, _lib, from_config
    from cases import cfg_of
    w = do.inputs("t2t_distill_cls", "init_weights")[1]
    inj = _model("t2t_distill_cls", "fp32", {k: v for k, v in w.items() if not k.startswith("layers.")}, cls="T2TViT",
                 transformer=lambda x, training=True: x)
    deep = from_config(cfg_of("deepvit_small"), precision="fp32")
    assert isinstance(inj, T2TViT) and isinstance(deep, DeepViT)
    for m, h, msg in ((inj, 32, "built for an injected transformer (depth 0) and holds no main transformer"),
                      (deep, 64, "vb_forward_distill supports ViT and T2TViT")):
        m._finalize()
        x = np.zeros((1, h, h, 3), np.float32)
        t = np.zeros(m.dim, np.float32)
        out = np.zeros((1, max(m.num_classes, m.dim)), np.float32)
        rc = m._lib.vb_forward_distill(m._h, x.ctypes.data_as(C.c_void_p), _lib.MEM_HOST, 1, h, h, t.ctypes.data_as(C.c_void_p),
                                       out.ctypes.data_as(C.c_void_p), out.ctypes.data_as(C.c_void_p), _lib.MEM_HOST, None)
        assert rc != 0 and msg in m._lib.vb_last_error(m._h).decode()


def test_emb_dropout_with_training_is_refused(lib):
    _, w, img, tok = do.inputs("t2t_distill_cls", "init_weights")
    m = _model("t2t_distill_cls", "bf16", w, emb_dropout=0.1)
    with pytest.raises(NotImplementedError):
        m(img, distill_token=tok)
    assert m(img, distill_token=tok, training=False)[0].shape == (do.BATCH, 10)

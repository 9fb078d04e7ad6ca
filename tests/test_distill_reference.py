"""The distillation students of the reference's distill.py beyond DistillableViT: DistillableT2TViT (distill.py:61-72) and
DistillableEfficientViT (:74-85), checked against the reference's own code without a GPU.

* LIVE (skipped where the reference checkout is absent): the reference's DistillableT2TViT over the numpy stand-in for TensorFlow
  equals distill_oracle.forward_distill to 1e-12 in float64, at the configured and at a smaller image; the constructor and call
  signatures equal the reference's; DistillableEfficientViT fails as the reference does; the unmodified DistillWrapper gives the
  same loss over a drop-in DistillableT2TViT student as over the reference's.
* FIXTURES (always): tests/golden/t2t_distill_*__refshim.npz, written from the reference's class by make_distill_golden.py, equal
  the restatement; the GPU tests compare the engine with them.
* HOST LOGIC over the C-ABI double (always): marshalling of the distillation call, the host-composed call around an injected
  transformer, the training rule, the shim's exports.
"""
import inspect
import os

import numpy as np
import pytest

import distill_oracle as do
import oracle
from oracle import ref_bind, spec_numpy, tf_shim

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
REF_DIR = os.environ.get("VB_REFERENCE_DIR", "/root/reference/vit_tensorflow")    # the reference checkout (absent on the GPU box)
live = pytest.mark.skipif(not os.path.isdir(REF_DIR), reason="reference checkout not present (GPU box): fixtures cover it")

CASE = do.CASES["t2t_distill_cls"]
KW = {k: v for k, v in CASE.items() if k != "kind"}


def _ours(cls_name="DistillableT2TViT", weights=None, **kw):
    import vit_tensorflow_b200 as vb
    m = getattr(vb, cls_name)(**{**KW, **kw}, precision="fp32")
    if weights is not None:
        m.set_weights_dict(weights)
    return m


# ------------------------------------------------------------------------------------------ the restatement vs the reference
@live
@pytest.mark.parametrize("name", do.SMALL)
def test_live_reference_distillable_t2t_equals_the_restatement(name):
    cfg, w, img, tok = do.inputs(name, "stress_weights")
    logits, dist, plain = do.reference_distill(REF_DIR, name, w, img, tok)
    ref_l, ref_d = do.forward_distill(img, tok, w, cfg)
    assert logits.shape == (2, cfg["num_classes"]) and dist.shape == (2, cfg["dim"])
    np.testing.assert_allclose(logits, ref_l, rtol=0, atol=1e-12)
    np.testing.assert_allclose(dist, ref_d, rtol=0, atol=1e-12)
    np.testing.assert_allclose(plain, oracle.forward_numpy(img, w, cfg), rtol=0, atol=1e-12)   # no token: T2TViT.call


@live
@pytest.mark.parametrize("name", ["t2t_distill_cls", "t2t_distill_4layers"])
def test_live_reference_on_a_smaller_image(name):
    """pos_embedding[:, :(n + 1)] (distill.py:24) on an image smaller than image_size."""
    cfg, w, img, tok = do.inputs(name, "stress_weights")
    small = oracle.make_image(cfg, 2, 5, h=24, w=24)
    logits, dist, _ = do.reference_distill(REF_DIR, name, w, img, tok, img_call=small)
    ref_l, ref_d = do.forward_distill(small, tok, w, cfg)
    np.testing.assert_allclose(logits, ref_l, rtol=0, atol=1e-12)
    np.testing.assert_allclose(dist, ref_d, rtol=0, atol=1e-12)


def test_restatement_on_vit_equals_the_vit_distillation_spec():
    """The restatement composes spec_numpy's stages; on a ViT config it is spec_numpy.forward_distill."""
    from cases import cfg_of
    cfg = dict(cfg_of("vit_small"), pool="mean")
    w = oracle.stress_weights(cfg, 4)
    img = oracle.make_image(cfg, 2, 5)
    tok = do.make_token(cfg["dim"], 6)
    for a, b in zip(do.forward_distill(img, tok, w, cfg), spec_numpy.forward_distill(img, tok, w, cfg)):
        np.testing.assert_allclose(a, b, rtol=0, atol=1e-12)


@pytest.mark.parametrize("gen", do.WEIGHTS)
@pytest.mark.parametrize("name", list(do.CASES))
def test_reference_fixture_equals_the_restatement(name, gen):
    cfg, w, img, tok = do.inputs(name, gen)
    z = np.load(os.path.join(GOLDEN, do.fixture_name(name, gen)))
    ref_l, ref_d = do.forward_distill(img, tok, w, cfg)
    np.testing.assert_allclose(z["logits_ref_f64"], ref_l, rtol=0, atol=1e-10)
    np.testing.assert_allclose(z["distill_ref_f64"], ref_d, rtol=0, atol=1e-10)
    np.testing.assert_allclose(z["logits_ref_f32"], ref_l, rtol=0, atol=5e-5)
    np.testing.assert_allclose(z["distill_ref_f32"], ref_d, rtol=0, atol=5e-5)


# ------------------------------------------------------------------------------------------ the boundary
@live
@pytest.mark.parametrize("ours,parent", [("DistillableT2TViT", "T2TViT"), ("DistillableEfficientViT", "EfficientViT")])
def test_live_constructor_and_call_signatures_equal_the_reference(ours, parent):
    """`(*args, **kwargs)` forwarded to the parent, whose parameters and defaults are the reference's (the parent's own test checks
    those against t2t.T2TViT / efficient.ViT), and `call(img, distill_token=None, training=True)`."""
    import vit_tensorflow_b200 as vb
    with tf_shim.installed(REF_DIR):
        import distill
        ref = getattr(distill, ours)
        ref_init, ref_call = inspect.signature(ref.__init__), inspect.signature(ref.call)
        ref_parent = inspect.signature(ref.__mro__[2].__init__)                   # (DistillMixin, T2TViT / efficient.ViT)
    cls = getattr(vb, ours)
    assert issubclass(cls, getattr(vb, parent))
    sig = lambda s: [(p.name, p.kind, p.default) for p in list(s.parameters.values())[1:]]
    assert sig(inspect.signature(cls.__init__)) == sig(ref_init)
    assert sig(inspect.signature(cls.__call__)) == sig(ref_call)
    assert cls.call is cls.__call__
    pos = [(p.name, p.default) for p in list(inspect.signature(getattr(vb, parent).__init__).parameters.values())[1:]
           if p.kind is inspect.Parameter.POSITIONAL_OR_KEYWORD]
    assert pos == [(p.name, p.default) for p in list(ref_parent.parameters.values())[1:]]


@live
def test_live_distillable_efficient_vit_fails_as_the_reference_does():
    """distill.py:83: `_attend` reads `self.dropout`, which efficient.ViT never defines: every call raises AttributeError, with or
    without a token.  The class still constructs and carries what DistillWrapper's constructor reads (distill.py:91-106)."""
    import vit_tensorflow_b200 as vb
    kw = dict(image_size=32, patch_size=16, num_classes=4, dim=32)
    img = np.zeros((2, 32, 32, 3), np.float32)
    tok = np.zeros((1, 1, 32), np.float32)
    calls = (lambda m: m(img), lambda m: m(img, training=False), lambda m: m(img, distill_token=tok, training=False),
             lambda m: m.call(img, tok, False))
    got = {}
    for label in ("reference", "ours"):
        with do.fake_installed(), tf_shim.installed(REF_DIR):
            import distill
            import vit
            tr = vit.Transformer(32, 1, 2, 16, 32)
            cls = distill.DistillableEfficientViT if label == "reference" else vb.DistillableEfficientViT
            m = cls(transformer=tr, **kw)
            errs = []
            for call in calls:
                with pytest.raises(Exception) as e:
                    call(m)
                errs.append((type(e.value), str(e.value)))
            assert not hasattr(m, "dropout")
            assert (m.dim, m.num_classes, m.args, sorted(m.kwargs)) == (32, 4, (), sorted(kw) + ["transformer"])
            distill.DistillableEfficientViT = type(m)                           # INTEGRATION.md: the reference-side binding
            w = distill.DistillWrapper(teacher=lambda x, training=True: x, student=m, temperature=3, alpha=0.5)
            assert w.student is m
            with pytest.raises(KeyError) as ke:
                cls(32, 16, 4, 32, tr)                                          # positional: kwargs['dim'] (distill.py:79)
            errs.append((type(ke.value), str(ke.value)))
            got[label] = errs
    assert got["ours"] == got["reference"]
    assert got["ours"][0] == (AttributeError, "'DistillableEfficientViT' object has no attribute 'dropout'")


def test_shim_exports_the_three_students():
    import vit_tensorflow_b200 as vb
    from vit_tensorflow.distill import DistillableEfficientViT, DistillableT2TViT, DistillableViT
    assert (DistillableViT, DistillableT2TViT, DistillableEfficientViT) == (vb.DistillableViT, vb.DistillableT2TViT,
                                                                           vb.DistillableEfficientViT)
    assert {"DistillableT2TViT", "DistillableEfficientViT"} <= set(vb.__all__)


# ------------------------------------------------------------------------------------------ host logic over the double
def test_distillable_t2t_over_the_double():
    cfg, w, img, tok = do.inputs("t2t_distill_cls", "stress_weights")
    with do.fake_installed() as fake:
        m = _ours(weights=w)
        assert (m.dim, m.num_classes, m.args, m.kwargs) == (64, 10, (), {**KW, "precision": "fp32"})
        logits, dist = m(img, distill_token=tok, training=False)
        ref_l, ref_d = do.forward_distill(img, tok, w, cfg)
        np.testing.assert_allclose(logits, ref_l, atol=1e-6)
        np.testing.assert_allclose(dist, ref_d, atol=1e-6)
        assert logits.dtype == dist.dtype == np.float32 and hasattr(logits, "numpy") and hasattr(dist, "numpy")
        np.testing.assert_allclose(m(img, training=False), oracle.forward_numpy(img, w, cfg), atol=1e-6)   # no token: T2TViT
        assert [c[0] for c in fake.calls][-2:] == ["vb_forward_distill", "vb_forward"]
        with pytest.raises(ValueError, match="distill_token must hold dim = 64"):
            m(img, distill_token=np.zeros((1, 1, 32), np.float32), training=False)
        import vit_tensorflow_b200 as vb
        with pytest.raises(KeyError, match="dim"):
            vb.DistillableT2TViT(32, 10, 64, depth=1, heads=2, mlp_dim=64)      # positional: kwargs['dim'] (distill.py:66), as there


def test_training_rule_over_the_double():
    """emb_dropout > 0 with training=True cannot be reproduced (inference semantics) and raises, with or without a token."""
    cfg, w, img, tok = do.inputs("t2t_distill_cls", "init_weights")
    with do.fake_installed():
        m = _ours(weights=w, emb_dropout=0.1)
        for call in (lambda: m(img, distill_token=tok), lambda: m(img)):
            with pytest.raises(NotImplementedError):
                call()
        logits, _ = m(img, distill_token=tok, training=False)
        np.testing.assert_allclose(logits, do.forward_distill(img, tok, w, cfg)[0], atol=1e-6)


def test_injected_transformer_is_composed_on_the_host():
    """DistillableT2TViT(transformer=...): forward_embed (n + 1 rows), the token appended, the injected transformer called with
    `training=`, then forward_head on x[:, :-1] and x[:, -1] -- the engine's own distillation call refuses a depth-0 handle."""
    cfg, w, img, tok = do.inputs("t2t_distill_cls", "stress_weights")
    with do.fake_installed() as fake:
        enc = _ours(weights=w)
        seen = []

        def probe(x, training=True):
            seen.append((x.shape, training))
            return enc.transformer(x, training=training)

        inj = _ours(transformer=probe, weights={k: v for k, v in w.items() if not k.startswith("layers.")})
        fake.calls.clear()
        logits, dist = inj(img, distill_token=tok, training=False)
        ref_l, ref_d = do.forward_distill(img, tok, w, cfg)
        np.testing.assert_allclose(logits, ref_l, atol=1e-5)
        np.testing.assert_allclose(dist, ref_d, atol=1e-5)
        assert dist.shape == (2, 64) and hasattr(dist, "numpy")
        n = oracle.t2t_token_grid(cfg)[-1]
        assert seen == [((2, n[0] * n[1] + 2, 64), False)]
        assert [c[0] for c in fake.calls if c[0] != "vb_finalize"] == ["vb_forward_embed", "vb_forward_tokens", "vb_forward_head"]
        np.testing.assert_allclose(inj(img, training=False), oracle.forward_numpy(img, w, cfg), atol=1e-5)


@live
def test_live_distill_wrapper_over_a_dropin_t2t_student():
    """distill.py:87-134, unmodified, around (a) the reference's DistillableT2TViT and (b) ours with the same weights and the same
    random stream: the same soft-distillation loss.  The reference-side binding is `distill.DistillableT2TViT = <ours>`
    (INTEGRATION.md), because distill.py:91 checks isinstance against the names in its own module."""
    cfg, w, img, _ = do.inputs("t2t_distill_cls", "stress_weights")
    labels = np.eye(10, dtype=np.float32)[[1, 4]]
    out = {}
    for label in ("reference", "ours"):
        with do.fake_installed(), tf_shim.installed(REF_DIR):
            import distill
            teacher = ref_bind.build_model("t2t_vit", KW, oracle.init_weights(cfg, 9), img)
            if label == "reference":
                student = ref_bind.build_model("t2t_vit", KW, w, img, cls=distill.DistillableT2TViT)
            else:
                student = _ours(weights=w)
                distill.DistillableT2TViT = type(student)
            tf_shim.set_seed(5)
            wrapper = distill.DistillWrapper(teacher=teacher, student=student, temperature=3, alpha=0.5, hard=False)
            out[label] = np.asarray(wrapper([img, labels], training=False), dtype=np.float64)
    assert np.isfinite(out["ours"]).all() and np.abs(out["ours"] - out["reference"]).max() < 1e-5

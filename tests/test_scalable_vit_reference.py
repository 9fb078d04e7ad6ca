"""CPU tests of the ScalableViT oracle (tests/scalable_vit_oracle.py) and of the host side of ScalableViT:

1. the reference's own scalable_vit.py, run unmodified over the stand-in, equals the float64 spec (which runs the blocks in the
   order SSA, MLP, PEG, MLP, IWSA) on every small case and on 40 seeded random configs, and the PyTorch restatement equals the spec;
2. the committed fixtures tests/golden/scalable_vit_*__refshim.npz equal both restatements;
3. the image sizes the host refuses are exactly those on which the reference fails, with the same exception type;
4. the constructor / call signatures, defaults and assert messages match the reference's;
5. the vb_scalable_vit_config layout matches the header, and vb_create refuses VB_KIND_SCALABLE_VIT with a pointer to
   vb_create_scalable_vit."""
import ctypes as C
import inspect
import os
import re

import numpy as np
import pytest

import scalable_vit_oracle as so

REF_DIR = os.environ.get("VB_REFERENCE_DIR", "/root/reference/vit_tensorflow")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
live = pytest.mark.skipif(not os.path.exists(os.path.join(REF_DIR, "scalable_vit.py")),
                          reason="reference checkout not present: the fixtures cover it")
CASES = [(n, g) for n in so.SMALL for g in ("init_weights", "stress_weights")]


def _tol(ref, rel):
    return rel * max(1.0, float(np.abs(ref).max()))


# ------------------------------------------------------------------------------------------ 1. the reference's code vs the spec
@pytest.fixture(scope="module")
def ref_module():
    with so.reference_module(REF_DIR) as mod:
        yield mod


@live
@pytest.mark.parametrize("name,gen", CASES)
def test_live_reference_equals_spec(ref_module, name, gen):
    cfg = so.make_config(**so.SMALL[name])
    w, img = getattr(so, gen)(cfg, so.WEIGHT_SEED), so.make_image(cfg, so.BATCH, so.IMAGE_SEED)
    ref = so.reference_logits(ref_module, cfg, w, img)
    np.testing.assert_allclose(ref, so.forward(img, w, cfg), rtol=0, atol=_tol(ref, 1e-12))


@live
@pytest.mark.parametrize("seed", range(40))
def test_live_reference_equals_spec_on_random_configs(ref_module, seed):
    cfg = so.random_config(seed)
    w, img = so.stress_weights(cfg, seed), so.make_image(cfg, 2, seed)
    ref = so.reference_logits(ref_module, cfg, w, img)
    np.testing.assert_allclose(ref, so.forward(img, w, cfg), rtol=0, atol=_tol(ref, 1e-12))


@live
def test_spec_in_the_names_order_differs_from_the_reference(ref_module):
    """The unpacking quirk matters: running element 4 (IWSA) before element 3 (MLP), as the names ssa, ff1, peg, ff2, iwsa of a
    reader's reading would, gives other logits."""
    cfg = so.make_config(**so.SMALL["scalable_vit_1stage"])
    w, img = so.stress_weights(cfg, 3), so.make_image(cfg, 1, 3)
    ref = so.reference_logits(ref_module, cfg, w, img)

    def names_order(x, st, w, b):
        x = so.iwsa(so._ln(x, w, b + "4.norm"), w, b + "4.fn.", st) + x
        return so.mlp(so._ln(x, w, b + "3.norm"), w, b + "3.fn.") + x
    ww = {k: np.asarray(v, np.float64) for k, v in w.items()}
    st = so.stages(cfg)[0]
    x = so._conv_same(np.asarray(img, np.float64), ww, "to_patches", 4)
    for L in range(st["depth"]):
        b = so.block_prefix(0, L)
        x = so.ssa(so._ln(x, ww, b + "0.norm"), ww, b + "0.fn.", st) + x
        x = so.mlp(so._ln(x, ww, b + "1.norm"), ww, b + "1.fn.") + x
        if L == 0:
            x = so.peg(x, ww, b + "2.proj")
        x = names_order(x, st, ww, b)
    assert np.isfinite(x).all()
    z = so._ln(x, ww, "scalable_layers.0.0.norm").mean(axis=(1, 2))
    z = (z - z.mean(-1, keepdims=True)) / np.sqrt(z.var(-1, keepdims=True) + 1e-3) * ww["mlp_head.1.gamma"] + ww["mlp_head.1.beta"]
    other = z @ ww["mlp_head.2.kernel"] + ww["mlp_head.2.bias"]
    assert np.abs(other - ref).max() > 1e-3 * np.abs(ref).max()


@pytest.mark.parametrize("name,gen", CASES)
def test_torch_restatement_equals_spec(name, gen):
    cfg = so.make_config(**so.SMALL[name])
    w, img = getattr(so, gen)(cfg, so.WEIGHT_SEED), so.make_image(cfg, so.BATCH, so.IMAGE_SEED)
    want = so.forward(img, w, cfg)
    np.testing.assert_allclose(so.forward_torch(img, w, cfg), want, rtol=0, atol=_tol(want, 1e-5))


# ------------------------------------------------------------------------------------------ 2. fixtures
@pytest.mark.parametrize("name,gen", CASES)
def test_fixtures_equal_both_restatements(name, gen):
    cfg = so.make_config(**so.SMALL[name])
    w, img = getattr(so, gen)(cfg, so.WEIGHT_SEED), so.make_image(cfg, so.BATCH, so.IMAGE_SEED)
    with np.load(os.path.join(GOLDEN, f"{name}__{gen}__refshim.npz")) as z:
        ref64, ref32 = z["logits_ref_f64"], z["logits_ref_f32"]
    scale = np.abs(ref64).max()
    for got in (so.forward(img, w, cfg), so.forward_torch(img, w, cfg)):
        np.testing.assert_allclose(got, ref64, rtol=0, atol=1e-10 * scale)
        np.testing.assert_allclose(got, ref32, rtol=0, atol=1e-4 * scale)


# ------------------------------------------------------------------------------------------ 3. refused image sizes
SIZE_CFG = dict(num_classes=3, dim=8, depth=(1, 1, 1), heads=1, ssa_dim_key=4, ssa_dim_value=4, iwsa_dim_key=4, iwsa_dim_value=4,
                reduction_factor=(2, 3, 1), window_size=(2, None, 2), ff_expansion_factor=1)


@live
def test_refused_sizes_are_exactly_where_the_reference_fails(ref_module):
    from vit_tensorflow_b200.models import scalable_vit_size_error
    cfg = so.make_config(**SIZE_CFG)
    refused = 0
    for h in range(1, 41, 3):
        for wd in range(1, 41, 5):
            img = so.make_image(cfg, 1, 0, h, wd)
            err = scalable_vit_size_error(so.stages(cfg), h, wd)
            try:
                model = ref_module.ScalableViT(**so.ctor_kwargs(cfg))
                model(img, training=False)
                failed = None
            except (AssertionError, ValueError) as e:
                failed = e
            assert (err is None) == (failed is None), (h, wd, err, failed)
            if err is not None:
                refused += 1
                if err[0] is AssertionError:                    # the reference's own assert: the same type and message
                    assert isinstance(failed, AssertionError) and str(failed) in err[1], (str(failed), err[1])
    assert refused > 10


# ------------------------------------------------------------------------------------------ 4. host class surface
REF_CTOR = ("(self, num_classes, dim, depth, heads, reduction_factor, window_size=None, iwsa_dim_key=32, iwsa_dim_value=32, "
            "ssa_dim_key=32, ssa_dim_value=32, ff_expansion_factor=4, channels=3, dropout=0.0)")


def test_constructor_and_call_signatures_match_the_reference():
    from vit_tensorflow_b200 import ScalableViT
    ctor = inspect.signature(ScalableViT.__init__)
    params = [p for p in ctor.parameters.values() if p.kind is not inspect.Parameter.KEYWORD_ONLY]
    assert "(" + ", ".join(str(p) for p in params) + ")" == REF_CTOR
    assert [p.name for p in ctor.parameters.values() if p.kind is inspect.Parameter.KEYWORD_ONLY] == ["precision", "device", "seed"]
    assert str(inspect.signature(ScalableViT.call)) == "(self, img, training=True, **kwargs)"
    path = os.path.join(REF_DIR, "scalable_vit.py")
    if os.path.exists(path):
        src = re.sub(r"\s+", " ", open(path).read())
        assert ("def __init__(self, num_classes, dim, depth, heads, reduction_factor, window_size=None, iwsa_dim_key=32, "
                "iwsa_dim_value=32, ssa_dim_key=32, ssa_dim_value=32, ff_expansion_factor=4, channels=3, dropout=0.0 ):") in src
        assert "def call(self, img, training=True, **kwargs):" in src
        assert "'depth needs to be tuple if integers indicating number of transformer blocks at that stage'" in src
        assert "for ssa, ff1, peg, iwsa, ff2 in self.layers:" in src
    from vit_tensorflow.scalable_vit import ScalableViT as Shim
    assert Shim is ScalableViT


def test_constructor_asserts_match_the_reference():
    from vit_tensorflow_b200 import ScalableViT
    kw = dict(num_classes=10, dim=64, heads=(2, 4), reduction_factor=(2, 1))
    with pytest.raises(AssertionError, match="depth needs to be tuple if integers indicating number of transformer blocks at that stage"):
        ScalableViT(depth=[2, 2], **kw)
    with pytest.raises(AssertionError) as e:
        ScalableViT(depth=(2, 2, 2), **kw)
    assert str(e.value) == ""
    with pytest.raises(NotImplementedError, match="1 to 4 stages"):
        ScalableViT(num_classes=10, dim=8, depth=(1,) * 5, heads=1, reduction_factor=1)


@live
def test_reference_constructor_errors_are_the_same(ref_module):
    kw = dict(num_classes=10, dim=64, heads=(2, 4), reduction_factor=(2, 1))
    with pytest.raises(AssertionError, match="depth needs to be tuple"):
        ref_module.ScalableViT(depth=[2, 2], **kw)
    with pytest.raises(AssertionError) as e:
        ref_module.ScalableViT(depth=(2, 2, 2), **kw)
    assert str(e.value) == ""


@pytest.mark.parametrize("name", sorted(so.SMALL) + sorted(so.BENCH))
def test_size_rules_accept_every_case(name):
    from vit_tensorflow_b200.models import scalable_vit_size_error
    cfg = so.make_config(**{**so.SMALL, **so.BENCH}[name])
    assert scalable_vit_size_error(so.stages(cfg), *cfg["image_size"]) is None
    if name == "scalable_vit_readme":                           # 224^2: the 56 x 56 map is not divisible by the window of 64
        err = scalable_vit_size_error(so.stages(cfg), 224, 224)
        assert err[0] is AssertionError and "stage 1: height (56) or width (56)" in err[1] and "window size (64, 64)" in err[1]


# ------------------------------------------------------------------------------------------ 5. ABI
def test_scalable_vit_config_layout_matches_header():
    from vit_tensorflow_b200 import _lib
    src = open(os.path.join(ROOT, "include", "vitb200.h")).read()
    body = src[src.index("typedef struct vb_scalable_vit_config {"):src.index("} vb_scalable_vit_config;")]
    n = int(re.search(r"#define VB_SCALABLE_VIT_STAGES (\d+)", src).group(1))
    fields = []
    for line in body.splitlines():
        line = line.split("/*")[0].strip()
        if line.startswith("int32_t"):
            fields += [f.strip() for f in line[len("int32_t"):].rstrip(";").split(",")]
    want = []
    for f in fields:
        m = re.match(r"(\w+)(?:\[(\w+)\])?", f)
        want.append((m.group(1), 1 if m.group(2) is None else (n if m.group(2) == "VB_SCALABLE_VIT_STAGES" else int(m.group(2)))))
    got = [(name, getattr(t, "_length_", 1)) for name, t in _lib.VbScalableVitConfig._fields_]
    assert got == want and n == _lib.SCALABLE_VIT_STAGES == 4
    assert int(re.search(r"VB_KIND_SCALABLE_VIT = (\d+)", src).group(1)) == _lib.KIND["scalable_vit"] == 17


def test_vb_create_refuses_scalable_vit_and_names_vb_create_scalable_vit(lib):
    from vit_tensorflow_b200 import _lib
    cfg = _lib.VbConfig()
    cfg.struct_size = C.sizeof(_lib.VbConfig)
    cfg.kind = _lib.KIND["scalable_vit"]
    cfg.image_h = cfg.image_w = 256
    cfg.channels, cfg.num_classes = 3, 10
    h = C.c_void_p()
    assert lib.vb_create(C.byref(cfg), 0, C.byref(h)) != 0 and not h.value
    assert b"vb_create_scalable_vit" in lib.vb_last_error(None)
    sc = _lib.VbScalableVitConfig()
    sc.struct_size = C.sizeof(_lib.VbScalableVitConfig) + 4
    assert lib.vb_create_scalable_vit(C.byref(cfg), C.byref(sc), 0, C.byref(h)) != 0
    assert b"vb_scalable_vit_config.struct_size" in lib.vb_last_error(None)

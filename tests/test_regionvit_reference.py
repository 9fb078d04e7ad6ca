"""CPU tests of the RegionViT oracle (tests/regionvit_oracle.py) and of the host side of RegionViT:

1. the reference's own regionvit.py, run unmodified over the stand-in, equals the float64 spec to 1e-11 on the hand-picked cases,
   for both weight sets;
2. the image sizes the host class refuses are the ones the reference fails on (among them 168 x 168, whose stage-3 windows do
   not divide, and local_patch_size 8, whose windows leave the relative-position table), with the reference's assert messages
   for the call-time asserts;
3. the committed fixtures tests/golden/regionvit_*__refshim.npz equal the spec;
4. the constructor / call signatures, defaults and assert messages match the reference's;
5. the vb_regionvit_config layout matches the header, and vb_create refuses VB_KIND_REGIONVIT with a pointer to
   vb_create_regionvit."""
import ctypes as C
import inspect
import os
import re

import numpy as np
import pytest

import regionvit_oracle as ro

REF_DIR = os.environ.get("VB_REFERENCE_DIR", "/root/reference/vit_tensorflow")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
HAVE_REF = os.path.exists(os.path.join(REF_DIR, "regionvit.py"))
live = pytest.mark.skipif(not HAVE_REF, reason="reference checkout not present: the fixtures cover it")


def _tol(ref):
    return 1e-11 * max(1.0, float(np.abs(ref).max()))


@pytest.fixture(scope="module")
def ref_module():
    if not HAVE_REF:
        pytest.skip("reference checkout not present: the fixtures cover it")
    with ro.reference_module(REF_DIR) as mod:
        yield mod


# ------------------------------------------------------------------------------------------ 1. live reference
@live
@pytest.mark.parametrize("gen", ["init_weights", "stress_weights"])
@pytest.mark.parametrize("name", sorted(ro.SMALL))
def test_live_reference_equals_spec(ref_module, name, gen):
    cfg = ro.make_config(**ro.SMALL[name])
    w = getattr(ro, gen)(cfg, 4)
    img = ro.make_image(cfg, 2, 5)
    ref = ro.forward(img, w, cfg)
    got = ro.reference_logits(ref_module, cfg, w, img)
    assert got.shape == ref.shape and np.abs(got - ref).max() <= _tol(ref)


def test_hand_picked_cases_cover_the_ground():
    """Windows 7 x 7, 14 x 14 (197 tokens), 4 x 7 and smaller; the 3-conv tokenizer and the PEG; widths not a multiple of 64;
    int dim and depth; a rectangular image."""
    windows, conv3, peg, odd, as_int, rect = set(), False, False, False, False, False
    for kw in ro.SMALL.values():
        cfg = ro.make_config(**kw)
        from vit_tensorflow_b200.models import regionvit_maps
        for (lh, lw), (rh, rw) in regionvit_maps(cfg["image_h"], cfg["image_w"], cfg["local_patch_size"], cfg["window_size"]):
            windows.add((lh // rh, lw // rw))
        conv3 |= cfg["tokenize_local_3_conv"]
        peg |= cfg["use_peg"]
        odd |= any(d % 64 for d in ro.dims(cfg))
        as_int |= isinstance(cfg["dim"], int) and isinstance(cfg["depth"], int)
        rect |= cfg["image_h"] != cfg["image_w"]
    assert {(7, 7), (14, 14), (4, 7), (4, 4), (2, 2), (1, 2)} <= windows
    assert conv3 and peg and odd and as_int and rect


# ------------------------------------------------------------------------------------------ 2. refused sizes
@live
@pytest.mark.parametrize("lp,h,w", [(4, 224, 224), (4, 168, 168), (4, 56, 56), (4, 28, 28), (4, 28, 56), (4, 560, 560), (4, 448, 448),
                                    (4, 112, 112), (4, 30, 28), (8, 224, 224), (8, 112, 112), (2, 28, 28), (2, 14, 14)])
def test_refused_sizes_are_the_references_failures(ref_module, lp, h, w):
    """The reference enforces its shape rules by its asserts, by einops (the window split), by the concat of the regional and
    local tokens and by the Embedding lookup; the host class refuses exactly those sizes, with the asserts' messages or naming the
    stage and both maps."""
    cfg = ro.make_config(dim=8, depth=1, num_classes=3, local_patch_size=lp)
    err = ro.size_error(cfg, h, w)
    model = ref_module.RegionViT(**ro.ctor_kwargs(cfg))
    try:
        model(np.zeros((1, h, w, 3)))
        failed = False
    except Exception:                                   # AssertionError, einops.EinopsError, the stand-in's shape / index errors
        failed = True
    assert failed == (err is not None), err
    if err is not None:
        assert re.match(r"(height and width must be divisible by (region|local) patch size|RegionViT stage \d: the \d+ x \d+ local map and "
                        r"the \d+ x \d+ region map (do not make whole windows \(the local map must be the region map times the window\)|"
                        r"make \d+ x \d+ windows, larger than window_size \d+ \(the relative-position table's reach\)))$", err)


def test_the_issue_sizes_get_the_expected_verdicts():
    cfg = ro.make_config(dim=8, depth=1, num_classes=3)
    for h, w in [(224, 224), (112, 112), (56, 56), (448, 448), (28, 56), (28, 28), (560, 560)]:
        assert ro.size_error(cfg, h, w) is None, (h, w)
    assert ro.size_error(cfg, 168, 168).startswith("RegionViT stage 3: the 11 x 11 local map and the 2 x 2 region map do not make")
    assert "larger than window_size 7" in ro.size_error(ro.make_config(dim=8, depth=1, local_patch_size=8), 224, 224)


def test_oracle_embedding_refuses_indices_outside_the_table():
    with pytest.raises(IndexError):
        ro.window_bias(np.zeros((9, 4)), 2, 3, 3)       # a 3 x 3 window against the (2 * 2 - 1)^2 table of window_size 2
    with ro.installed(REF_DIR if HAVE_REF else None):
        import tensorflow.keras.layers as nn
        e = nn.Embedding(9, 4)
        e(np.array([0, 8]))
        with pytest.raises(IndexError):
            e(np.array([-1]))
        with pytest.raises(IndexError):
            e(np.array([9]))


# ------------------------------------------------------------------------------------------ 3. fixtures
@pytest.mark.parametrize("gen", ["init_weights", "stress_weights"])
@pytest.mark.parametrize("name", sorted(ro.SMALL) + sorted(ro.BENCH))
def test_fixtures_equal_spec(name, gen):
    cfg = ro.make_config(**{**ro.SMALL, **ro.BENCH}[name])
    w = getattr(ro, gen)(cfg, ro.WEIGHT_SEED)
    img = ro.make_image(cfg, ro.BATCH, ro.IMAGE_SEED)
    z = np.load(os.path.join(GOLDEN, f"{name}__{gen}__refshim.npz"))
    ref = ro.forward(img, w, cfg)
    tag = "f64" if name in ro.SMALL else "f32"
    tol = 1e-11 if tag == "f64" else 5e-4
    assert np.abs(z[f"logits_ref_{tag}"] - ref).max() <= tol * max(1.0, np.abs(ref).max())


# ------------------------------------------------------------------------------------------ 4. host class surface
CTOR = ["dim", "depth", "window_size", "num_classes", "tokenize_local_3_conv", "local_patch_size", "use_peg", "attn_dropout",
        "ff_dropout"]


def test_constructor_and_call_signatures_match_the_reference():
    from vit_tensorflow_b200 import RegionViT
    ctor = inspect.signature(RegionViT.__init__)
    params = [p for p in ctor.parameters.values() if p.kind is not inspect.Parameter.KEYWORD_ONLY]
    assert [p.name for p in params] == ["self"] + CTOR
    assert {p.name: p.default for p in params[1:]} == ro.REGIONVIT_DEFAULTS
    assert [p.name for p in ctor.parameters.values() if p.kind is inspect.Parameter.KEYWORD_ONLY] == ["precision", "device", "seed"]
    assert str(inspect.signature(RegionViT.call)) == "(self, x, training=True, **kwargs)"
    if HAVE_REF:
        with ro.reference_module(REF_DIR) as mod:
            ref = inspect.signature(mod.RegionViT.__init__)
            assert [(p.name, p.default) for p in ref.parameters.values()] == [(p.name, p.default) for p in params]
            assert str(inspect.signature(mod.RegionViT.call)) == "(self, x, training=True, **kwargs)"
    from vit_tensorflow.regionvit import RegionViT as Shim
    assert Shim is RegionViT


@pytest.mark.parametrize("kw,msg", [(dict(dim=(1, 2, 3)), "dim needs to be a single value or a tuple of length 4"),
                                    (dict(depth=(1, 2, 3, 4, 5)), "depth needs to be a single value or a tuple of length 4")])
def test_constructor_assertions_match_the_reference(kw, msg):
    from vit_tensorflow_b200 import RegionViT
    with pytest.raises(AssertionError, match=f"^{msg}$"):
        RegionViT(**kw)
    if HAVE_REF:
        with ro.reference_module(REF_DIR) as mod:
            with pytest.raises(AssertionError, match=f"^{msg}$"):
                mod.RegionViT(**kw)


def test_regionvit_config_layout_matches_header():
    from vit_tensorflow_b200 import _lib
    src = open(os.path.join(ROOT, "include", "vitb200.h")).read()
    body = src[src.index("typedef struct vb_regionvit_config {"):src.index("} vb_regionvit_config;")]
    fields = []
    for line in body.splitlines():
        line = line.split("/*")[0].strip()
        if line.startswith("int32_t"):
            fields += [f.strip() for f in line[len("int32_t"):].rstrip(";").split(",")]
    want = [(f.split("[")[0], _lib.REGIONVIT_STAGES if "[" in f else 1) for f in fields]
    got = [(n, C.sizeof(t) // 4) for n, t in _lib.VbRegionvitConfig._fields_]
    assert got == want and C.sizeof(_lib.VbRegionvitConfig) == 4 * (6 + 2 * _lib.REGIONVIT_STAGES)
    assert int(re.search(r"#define VB_REGIONVIT_STAGES (\d+)", src).group(1)) == _lib.REGIONVIT_STAGES == 4
    assert int(re.search(r"VB_KIND_REGIONVIT = (\d+)", src).group(1)) == _lib.KIND["regionvit"] == 13


def test_vb_create_refuses_regionvit_and_names_vb_create_regionvit(lib):
    from vit_tensorflow_b200 import _lib
    cfg = _lib.VbConfig()
    cfg.struct_size = C.sizeof(_lib.VbConfig)
    cfg.kind = _lib.KIND["regionvit"]
    cfg.image_h = cfg.image_w = 224
    cfg.channels, cfg.num_classes = 3, 10
    h = C.c_void_p()
    assert lib.vb_create(C.byref(cfg), 0, C.byref(h)) != 0 and not h.value
    assert b"vb_create_regionvit" in lib.vb_last_error(None)
    rc = _lib.VbRegionvitConfig()
    rc.struct_size = C.sizeof(_lib.VbRegionvitConfig) + 4
    assert lib.vb_create_regionvit(C.byref(cfg), C.byref(rc), 0, C.byref(h)) != 0
    assert b"vb_regionvit_config.struct_size" in lib.vb_last_error(None)
    rc.struct_size = C.sizeof(_lib.VbRegionvitConfig)
    rc.window_size, rc.local_patch_size, rc.mlp_mult = 7, 4, 4
    assert lib.vb_create_regionvit(C.byref(cfg), C.byref(rc), 0, C.byref(h)) != 0
    assert b"RegionViT: dims must be positive" in lib.vb_last_error(None)

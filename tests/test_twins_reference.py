"""CPU tests of the Twins-SVT oracle (tests/twins_oracle.py) and of the host side of Twins-SVT:

1. the reference's own twins_svt.py, run unmodified over the stand-in, equals the float64 spec to 1e-12 on the hand-picked cases
   and 40 seeded random configurations, and the PyTorch restatement equals the spec to 1e-5;
2. the image sizes the host class refuses are the ones the reference fails on;
3. the committed fixtures tests/golden/twins_*__refshim.npz equal the spec;
4. the constructor / call signatures and defaults match the reference's;
5. the vb_twins_svt_config layout matches the header, and vb_create refuses VB_KIND_TWINS_SVT with a pointer to
   vb_create_twins_svt."""
import ctypes as C
import inspect
import os
import re

import numpy as np
import pytest

import twins_oracle as to

REF_DIR = os.environ.get("VB_REFERENCE_DIR", "/root/reference/vit_tensorflow")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
live = pytest.mark.skipif(not os.path.exists(os.path.join(REF_DIR, "twins_svt.py")),
                          reason="reference checkout not present: the fixtures cover it")


def _tol(ref):
    return 1e-12 * max(1.0, float(np.abs(ref).max()))


@pytest.fixture(scope="module")
def ref_module():
    if not os.path.exists(os.path.join(REF_DIR, "twins_svt.py")):
        pytest.skip("reference checkout not present: the fixtures cover it")
    with to.reference_module(REF_DIR) as mod:
        yield mod


# ------------------------------------------------------------------------------------------ 1. live reference
@live
@pytest.mark.parametrize("name", sorted(to.SMALL) + sorted(to.BENCH))
def test_live_reference_equals_spec(ref_module, name):
    cfg = to.make_config(**{**to.SMALL, **to.BENCH}[name])
    w = to.stress_weights(cfg, 4)
    img = to.make_image(cfg, 2, 5)
    ref = to.forward(img, w, cfg)
    got = to.reference_logits(ref_module, cfg, w, img)
    assert got.shape == ref.shape and np.abs(got - ref).max() <= _tol(ref)
    assert np.abs(to.forward_torch(img, w, cfg) - ref).max() <= 1e-5 * max(1.0, np.abs(ref).max())


@live
def test_live_reference_equals_spec_on_random_configurations(ref_module):
    """40 seeded random configurations: windows of p^2 < 64, = 64 and > 64 tokens, global_k unlike the window with
    floor-truncated key maps, even PEG kernels, widths off 64 and non-square images."""
    windows, truncated, pegs, widths, nonsquare = set(), False, set(), set(), False
    for seed in range(40):
        cfg = to.random_config(seed)
        h, w_ = cfg["image_h"], cfg["image_w"]
        assert to.size_error(cfg, h, w_) is None, cfg
        for st in to.stages(cfg)[:3]:
            windows.add(st["local_patch_size"] ** 2)
        for st in to.stages(cfg):
            h, w_ = h // st["patch_size"], w_ // st["patch_size"]
            truncated |= (h % st["global_k"] != 0 or w_ % st["global_k"] != 0)
            widths.add(st["emb_dim"])
        pegs.add(cfg["peg_kernel_size"])
        nonsquare |= cfg["image_h"] != cfg["image_w"]
        wts = to.stress_weights(cfg, seed)
        img = to.make_image(cfg, 2, seed + 1)
        ref = to.forward(img, wts, cfg)
        got = to.reference_logits(ref_module, cfg, wts, img)
        assert got.shape == ref.shape and np.abs(got - ref).max() <= _tol(ref), (seed, cfg)
        if seed < 8:
            assert np.abs(to.forward_torch(img, wts, cfg) - ref).max() <= 1e-5 * max(1.0, np.abs(ref).max()), (seed, cfg)
    assert min(windows) < 64 and 64 in windows and max(windows) > 64
    assert truncated and {2, 4} <= pegs and {40, 72} <= widths and nonsquare


# ------------------------------------------------------------------------------------------ 2. refused sizes
@live
@pytest.mark.parametrize("h,w", [(224, 224), (224, 448), (220, 224), (224, 196), (56, 56), (112, 112), (448, 224)])
def test_refused_sizes_are_the_references_failures(ref_module, h, w):
    """The reference enforces its shape rules through einops and Keras; the host class refuses exactly those sizes, naming the
    stage (a 112 x 112 image gives a 3 x 3 stage-4 map, smaller than global_k = 7)."""
    cfg = to.make_config(image_size=h, image_w=w, num_classes=3, s1_emb_dim=8, s2_emb_dim=8, s3_emb_dim=8, s3_depth=0, s4_emb_dim=8,
                         s4_depth=0)
    err = to.size_error(cfg, h, w)
    model = ref_module.TwinsSVT(**to.ctor_kwargs(cfg))
    try:
        model(np.zeros((1, h, w, 3)))
        failed = False
    except Exception:                                   # einops.EinopsError or the stand-in's shape errors
        failed = True
    assert failed == (err is not None), err
    if err is not None:
        assert re.match(r"Twins-SVT stage [1-4]: the \d+ x \d+ map ", err)


# ------------------------------------------------------------------------------------------ 3. fixtures
@pytest.mark.parametrize("gen", ["init_weights", "stress_weights"])
@pytest.mark.parametrize("name", sorted(to.SMALL) + sorted(to.BENCH))
def test_fixtures_equal_spec(name, gen):
    cfg = to.make_config(**{**to.SMALL, **to.BENCH}[name])
    w = getattr(to, gen)(cfg, to.WEIGHT_SEED)
    img = to.make_image(cfg, to.BATCH, to.IMAGE_SEED)
    z = np.load(os.path.join(GOLDEN, f"{name}__{gen}__refshim.npz"))
    ref = to.forward(img, w, cfg)
    tag = "f64" if name in to.SMALL else "f32"
    tol = 1e-12 if tag == "f64" else 5e-4
    assert np.abs(z[f"logits_ref_{tag}"] - ref).max() <= tol * max(1.0, np.abs(ref).max())


# ------------------------------------------------------------------------------------------ 4. host class surface
def test_constructor_and_call_signatures_match_the_reference():
    from vit_tensorflow_b200 import TwinsSVT
    ctor = inspect.signature(TwinsSVT.__init__)
    params = [p for p in ctor.parameters.values() if p.kind is not inspect.Parameter.KEYWORD_ONLY]
    assert [p.name for p in params] == ["self", "num_classes"] + list(to.TWINS_DEFAULTS)
    assert {p.name: p.default for p in params[2:]} == to.TWINS_DEFAULTS
    assert str(inspect.signature(TwinsSVT.call)) == "(self, img, training=True, **kwargs)"
    if os.path.exists(os.path.join(REF_DIR, "twins_svt.py")):
        with to.reference_module(REF_DIR) as mod:
            ref = inspect.signature(mod.TwinsSVT.__init__)
            assert [(p.name, p.default) for p in ref.parameters.values()] == [(p.name, p.default) for p in params]
            assert str(inspect.signature(mod.TwinsSVT.call)) == "(self, x, training=True, **kwargs)"
    from vit_tensorflow.twins_svt import TwinsSVT as Shim
    assert Shim is TwinsSVT


def test_twins_config_layout_matches_header():
    from vit_tensorflow_b200 import _lib
    src = open(os.path.join(ROOT, "include", "vitb200.h")).read()
    body = src[src.index("typedef struct vb_twins_svt_config {"):src.index("} vb_twins_svt_config;")]
    fields = []
    for line in body.splitlines():
        line = line.split("/*")[0].strip()
        if line.startswith("int32_t"):
            fields += [f.strip() for f in line[len("int32_t"):].rstrip(";").split(",")]
    want = [(f.split("[")[0], 4 if "[" in f else 1) for f in fields]
    got = [(n, getattr(t, "_length_", 1)) for n, t in _lib.VbTwinsSvtConfig._fields_]
    assert got == want and C.sizeof(_lib.VbTwinsSvtConfig) == 4 * (1 + 5 * 4 + 1)
    assert int(re.search(r"#define VB_TWINS_STAGES (\d+)", src).group(1)) == _lib.TWINS_STAGES
    assert int(re.search(r"VB_KIND_TWINS_SVT = (\d+)", src).group(1)) == _lib.KIND["twins_svt"] == 10


def test_vb_create_refuses_twins_and_names_vb_create_twins_svt(lib):
    from vit_tensorflow_b200 import _lib
    cfg = _lib.VbConfig()
    cfg.struct_size = C.sizeof(_lib.VbConfig)
    cfg.kind = _lib.KIND["twins_svt"]
    cfg.image_h = cfg.image_w = 224
    cfg.channels, cfg.num_classes = 3, 10
    h = C.c_void_p()
    assert lib.vb_create(C.byref(cfg), 0, C.byref(h)) != 0 and not h.value
    assert b"vb_create_twins_svt" in lib.vb_last_error(None)
    tw = _lib.VbTwinsSvtConfig()
    tw.struct_size = C.sizeof(_lib.VbTwinsSvtConfig) + 4
    assert lib.vb_create_twins_svt(C.byref(cfg), C.byref(tw), 0, C.byref(h)) != 0
    assert b"vb_twins_svt_config.struct_size" in lib.vb_last_error(None)
    tw.struct_size = C.sizeof(_lib.VbTwinsSvtConfig)
    for i in range(4):
        tw.emb_dim[i] = tw.patch_size[i] = tw.local_patch_size[i] = tw.global_k[i] = 1
    tw.peg_kernel_size = 8
    assert lib.vb_create_twins_svt(C.byref(cfg), C.byref(tw), 0, C.byref(h)) != 0
    assert b"peg_kernel_size" in lib.vb_last_error(None)

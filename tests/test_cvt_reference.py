"""CPU tests of the CvT oracle (tests/cvt_oracle.py) and of the host side of CvT:

1. the stand-in's depthwise Conv2D (groups == channels, SAME, both strides) and the reference's LayerNorm against torch;
2. the reference's own cvt.py, run unmodified over the stand-in, equals the float64 spec to 1e-12 on the hand-picked cases and 40
   seeded random configurations, and the PyTorch restatement equals the spec to 1e-5;
3. the committed fixtures tests/golden/cvt_*__refshim.npz equal the spec;
4. the constructor / call signatures and defaults match the reference's;
5. the vb_cvt_config layout matches the header, and vb_create refuses VB_KIND_CVT with a pointer to vb_create_cvt."""
import ctypes as C
import inspect
import os
import re

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import cvt_oracle as co
from oracle import tf_shim

REF_DIR = os.environ.get("VB_REFERENCE_DIR", "/root/reference/vit_tensorflow")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
live = pytest.mark.skipif(not os.path.exists(os.path.join(REF_DIR, "cvt.py")), reason="reference checkout not present: the fixtures cover it")


def _tol(ref):
    return 1e-12 * max(1.0, float(np.abs(ref).max()))


# ------------------------------------------------------------------------------------------ 1. primitives vs torch
@pytest.mark.parametrize("k,s,H,W", [(3, 1, 7, 8), (3, 2, 7, 8), (5, 2, 8, 7), (7, 2, 9, 9), (1, 2, 6, 5), (7, 1, 4, 5)])
def test_shim_depthwise_conv_against_torch(k, s, H, W):
    rng = np.random.default_rng(k * 10 + s)
    x = rng.standard_normal((2, H, W, 6))
    tf_shim.set_dtype(np.float64)
    try:
        with co.installed(None):
            import tensorflow.keras.layers as nn
            conv = nn.Conv2D(filters=6, kernel_size=k, strides=s, padding='SAME', groups=6, use_bias=False)
            conv(x)
            kern = rng.standard_normal((k, k, 1, 6))
            conv.set_weights([kern])
            got = np.asarray(conv(x))
    finally:
        tf_shim.set_dtype(np.float32)
    oh, ow = -(-H // s), -(-W // s)
    ph, pw = max((oh - 1) * s + k - H, 0), max((ow - 1) * s + k - W, 0)
    xt = F.pad(torch.from_numpy(x).permute(0, 3, 1, 2), (pw // 2, pw - pw // 2, ph // 2, ph - ph // 2))
    want = F.conv2d(xt, torch.from_numpy(kern).permute(3, 2, 0, 1), stride=s, groups=6).permute(0, 2, 3, 1).numpy()
    np.testing.assert_allclose(got, want, atol=1e-12)
    np.testing.assert_allclose(co.dwconv_same(x, kern, s), want, atol=1e-12)


def test_spec_layernorm_against_torch():
    rng = np.random.default_rng(0)
    x, g, b = rng.standard_normal((2, 3, 4, 40)), rng.standard_normal((1, 1, 1, 40)), rng.standard_normal((1, 1, 1, 40))
    want = F.layer_norm(torch.from_numpy(x), (40,), torch.from_numpy(g.reshape(-1)), torch.from_numpy(b.reshape(-1)), 1e-5).numpy()
    np.testing.assert_allclose(co.layer_norm(x, g, b), want, atol=1e-12)


# ------------------------------------------------------------------------------------------ 2. live reference
@pytest.fixture(scope="module")
def ref_module():
    if not os.path.exists(os.path.join(REF_DIR, "cvt.py")):
        pytest.skip("reference checkout not present: the fixtures cover it")
    with co.reference_module(REF_DIR) as mod:
        yield mod


@live
@pytest.mark.parametrize("name", sorted(co.SMALL) + sorted(co.BENCH))
def test_live_reference_equals_spec(ref_module, name):
    cfg = co.make_config(**{**co.SMALL, **co.BENCH}[name])
    w = co.stress_weights(cfg, 4)
    img = co.make_image(cfg, 2, 5)
    ref = co.forward(img, w, cfg)
    got = co.reference_logits(ref_module, cfg, w, img)
    assert got.shape == ref.shape and np.abs(got - ref).max() <= _tol(ref)
    assert np.abs(co.forward_torch(img, w, cfg) - ref).max() <= 1e-5 * max(1.0, np.abs(ref).max())


@live
def test_live_reference_equals_spec_on_random_configurations(ref_module):
    """40 seeded random configurations: proj_kernel 1 / 3 / 5 / 7, kv strides 1 and 2, odd map sizes, widths off 64."""
    seen_k, seen_s, odd = set(), set(), False
    for seed in range(40):
        cfg = co.random_config(seed)
        for st in co.stages(cfg):
            seen_k.add(st["proj_kernel"])
            seen_s.add(st["kv_proj_stride"])
        odd |= cfg["image_h"] % 2 == 1
        w = co.stress_weights(cfg, seed)
        img = co.make_image(cfg, 2, seed + 1)
        ref = co.forward(img, w, cfg)
        got = co.reference_logits(ref_module, cfg, w, img)
        assert got.shape == ref.shape and np.abs(got - ref).max() <= _tol(ref), (seed, cfg)
        if seed < 8:
            assert np.abs(co.forward_torch(img, w, cfg) - ref).max() <= 1e-5 * max(1.0, np.abs(ref).max()), (seed, cfg)
    assert seen_k == {1, 3, 5, 7} and seen_s == {1, 2} and odd


# ------------------------------------------------------------------------------------------ 3. fixtures
@pytest.mark.parametrize("gen", ["init_weights", "stress_weights"])
@pytest.mark.parametrize("name", sorted(co.SMALL) + sorted(co.BENCH))
def test_fixtures_equal_spec(name, gen):
    cfg = co.make_config(**{**co.SMALL, **co.BENCH}[name])
    w = getattr(co, gen)(cfg, co.WEIGHT_SEED)
    img = co.make_image(cfg, co.BATCH, co.IMAGE_SEED)
    z = np.load(os.path.join(GOLDEN, f"{name}__{gen}__refshim.npz"))
    ref = co.forward(img, w, cfg)
    tag = "f64" if name in co.SMALL else "f32"
    tol = 1e-12 if tag == "f64" else 5e-4
    assert np.abs(z[f"logits_ref_{tag}"] - ref).max() <= tol * max(1.0, np.abs(ref).max())


# ------------------------------------------------------------------------------------------ 4. host class surface
def test_constructor_and_call_signatures_match_the_reference():
    from vit_tensorflow_b200 import CvT
    ctor = inspect.signature(CvT.__init__)
    params = [p for p in ctor.parameters.values() if p.kind is not inspect.Parameter.KEYWORD_ONLY]
    assert [p.name for p in params] == ["self", "num_classes"] + list(co.CVT_DEFAULTS)
    assert {p.name: p.default for p in params[2:]} == co.CVT_DEFAULTS
    assert str(inspect.signature(CvT.call)) == "(self, img, training=True, **kwargs)"
    if os.path.exists(os.path.join(REF_DIR, "cvt.py")):
        with co.reference_module(REF_DIR) as mod:
            ref = inspect.signature(mod.CvT.__init__)
            assert [(p.name, p.default) for p in ref.parameters.values()] == [(p.name, p.default) for p in params]
            assert str(inspect.signature(mod.CvT.call)) == "(self, img, training=True, **kwargs)"
    from vit_tensorflow.cvt import CvT as Shim
    assert Shim is CvT


def test_cvt_config_layout_matches_header():
    from vit_tensorflow_b200 import _lib
    src = open(os.path.join(ROOT, "include", "vitb200.h")).read()
    body = src[src.index("typedef struct vb_cvt_config {"):src.index("} vb_cvt_config;")]
    fields = []
    for line in body.splitlines():
        line = line.split("/*")[0].strip()
        if line.startswith("int32_t"):
            fields += [f.strip() for f in line[len("int32_t"):].rstrip(";").split(",")]
    want = [(f.split("[")[0], 3 if "[" in f else 1) for f in fields]
    got = [(n, getattr(t, "_length_", 1)) for n, t in _lib.VbCvtConfig._fields_]
    assert got == want and C.sizeof(_lib.VbCvtConfig) == 4 * (1 + 8 * 3)
    assert int(re.search(r"#define VB_CVT_STAGES (\d+)", src).group(1)) == _lib.CVT_STAGES
    assert int(re.search(r"VB_KIND_CVT = (\d+)", src).group(1)) == _lib.KIND["cvt"] == 9


def test_vb_create_refuses_cvt_and_names_vb_create_cvt(lib):
    from vit_tensorflow_b200 import _lib
    cfg = _lib.VbConfig()
    cfg.struct_size = C.sizeof(_lib.VbConfig)
    cfg.kind = _lib.KIND["cvt"]
    cfg.image_h = cfg.image_w = 224
    cfg.channels, cfg.num_classes = 3, 10
    h = C.c_void_p()
    assert lib.vb_create(C.byref(cfg), 0, C.byref(h)) != 0 and not h.value
    assert b"vb_create_cvt" in lib.vb_last_error(None)
    cv = _lib.VbCvtConfig()
    cv.struct_size = C.sizeof(_lib.VbCvtConfig) + 4
    assert lib.vb_create_cvt(C.byref(cfg), C.byref(cv), 0, C.byref(h)) != 0
    assert b"vb_cvt_config.struct_size" in lib.vb_last_error(None)

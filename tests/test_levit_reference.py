"""CPU tests of the LeViT oracle (tests/levit_oracle.py) and of the host side of LeViT:

1. the stand-in's BatchNormalization (both branches) and 1x1 stride-2 'valid' Conv2D against torch;
2. the reference's own levit.py, run unmodified over the stand-in (its import-time usage block included), equals the float64
   spec to 1e-12 on the hand-picked cases and 40 seeded random configurations, and the PyTorch restatement equals the spec;
3. the committed fixtures tests/golden/levit_*__refshim.npz equal the spec;
4. the constructor / call signatures and constructor errors match the reference's;
5. the vb_levit_config layout matches the header, and vb_create refuses VB_KIND_LEVIT with a pointer to vb_create_levit."""
import ctypes as C
import inspect
import os
import re

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import levit_oracle as lo
from oracle import tf_shim

REF_DIR = os.environ.get("VB_REFERENCE_DIR", "/root/reference/vit_tensorflow")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
live = pytest.mark.skipif(not os.path.exists(os.path.join(REF_DIR, "levit.py")), reason="reference checkout not present: the fixtures cover it")


def _tol(ref):
    return 1e-12 * max(1.0, float(np.abs(ref).max()))


def _pairs(a, b):
    a, b = (a if isinstance(a, tuple) else (a,)), (b if isinstance(b, tuple) else (b,))
    assert len(a) == len(b)
    return zip(a, b)


# ------------------------------------------------------------------------------------------ 1. primitives vs torch
@pytest.mark.parametrize("training", [False, True])
def test_shim_batchnorm_against_torch(training):
    rng = np.random.default_rng(3)
    x = rng.standard_normal((2, 5, 4, 6))
    tf_shim.set_dtype(np.float64)
    try:
        with lo.installed(None):
            import tensorflow.keras.layers as nn
            bn = nn.BatchNormalization(momentum=0.9, epsilon=1e-05)
            bn(x, training=False)
            g, b, mu, var = rng.standard_normal(6), rng.standard_normal(6), rng.standard_normal(6), rng.uniform(0.5, 2, 6)
            bn.set_weights([g, b, mu, var])
            got = np.asarray(bn(x, training=training))
            moved = np.asarray(bn.moving_mean)
    finally:
        tf_shim.set_dtype(np.float32)
    xt = torch.from_numpy(x).permute(0, 3, 1, 2)
    rm, rv = torch.from_numpy(mu.copy()), torch.from_numpy(var.copy())
    want = F.batch_norm(xt, rm, rv, torch.from_numpy(g), torch.from_numpy(b), training, 0.1, 1e-5).permute(0, 2, 3, 1).numpy()
    np.testing.assert_allclose(got, want, atol=1e-12)
    if training:                       # keras momentum 0.9 == torch momentum 0.1 on the mean
        np.testing.assert_allclose(moved, rm.numpy(), atol=1e-12)


@pytest.mark.parametrize("H", [7, 8, 14])
def test_shim_conv1x1_stride2_valid_against_torch(H):
    rng = np.random.default_rng(H)
    x = rng.standard_normal((2, H, H, 5))
    tf_shim.set_dtype(np.float64)
    try:
        with lo.installed(None):
            import tensorflow.keras.layers as nn
            conv = nn.Conv2D(filters=3, kernel_size=1, strides=2, use_bias=False)
            conv(x)
            kern = rng.standard_normal((1, 1, 5, 3))
            conv.set_weights([kern])
            got = np.asarray(conv(x))
    finally:
        tf_shim.set_dtype(np.float32)
    want = F.conv2d(torch.from_numpy(x).permute(0, 3, 1, 2), torch.from_numpy(kern).permute(3, 2, 0, 1), stride=2)
    np.testing.assert_allclose(got, want.permute(0, 2, 3, 1).numpy(), atol=1e-12)
    assert got.shape[1] == -(-H // 2)


# ------------------------------------------------------------------------------------------ 2. live reference
@pytest.fixture(scope="module")
def ref_module():
    if not os.path.exists(os.path.join(REF_DIR, "levit.py")):
        pytest.skip("reference checkout not present: the fixtures cover it")
    with lo.reference_module(REF_DIR) as mod:     # the import runs levit.py's 224^2 usage block with BatchNorm in training mode
        yield mod


@live
@pytest.mark.parametrize("name", sorted(lo.SMALL) + sorted(lo.BENCH))
def test_live_reference_equals_spec(ref_module, name):
    cfg = lo.make_config(**{**lo.SMALL, **lo.BENCH}[name])
    w = lo.stress_weights(cfg, 4)
    img = lo.make_image(cfg, 2, 5)
    ref = lo.forward(img, w, cfg)
    for got, r in _pairs(lo.reference_logits(ref_module, cfg, w, img), ref):
        assert np.abs(got - r).max() <= _tol(r)
    for got, r in _pairs(lo.forward_torch(img, w, cfg), ref):
        assert np.abs(got - r).max() <= _tol(r)


@live
def test_live_reference_equals_spec_on_random_configurations(ref_module):
    """40 seeded random configurations: 1-4 stages, int and short-tuple dims / depths / heads, dim_key below and above
    dim_value, odd widths, with and without a distillation head."""
    seen = set()
    for seed in range(40):
        cfg = lo.random_config(seed)
        seen.add((cfg["stages"], cfg["dim_key"] < cfg["dim_value"], cfg["num_distill_classes"] is None))
        w = lo.stress_weights(cfg, seed)
        img = lo.make_image(cfg, 2, seed + 1)
        ref = lo.forward(img, w, cfg)
        for got, r in _pairs(lo.reference_logits(ref_module, cfg, w, img), ref):
            assert got.shape == r.shape and np.abs(got - r).max() <= _tol(r), (seed, cfg)
        if seed < 8:
            for got, r in _pairs(lo.forward_torch(img, w, cfg), ref):
                assert np.abs(got - r).max() <= _tol(r), (seed, cfg)
    assert {s for s, _, _ in seen} == {1, 2, 3, 4} and {k for _, k, _ in seen} == {True, False} and {d for _, _, d in seen} == {True, False}


@live
def test_live_reference_accepts_a_non_square_image_and_fails_on_a_wrong_image_size(ref_module):
    cfg = lo.make_config(image_size=224, num_classes=3, dim=32, depth=1, heads=2, mlp_mult=2, stages=2)
    w = lo.stress_weights(cfg, 1)
    img = lo.make_image(cfg, 1, 2, 210, 216)
    got = lo.reference_logits(ref_module, cfg, w, lo.make_image(cfg, 1, 3), img_call=img)
    assert np.abs(got - lo.forward(img, w, cfg)).max() <= _tol(got)
    with pytest.raises(Exception):                                    # 200 // 16 = 12, the stem gives 13: the bias cannot broadcast
        ref_module.LeViT(image_size=200, num_classes=3, dim=32, depth=1, heads=2, mlp_mult=2)(np.zeros((1, 200, 200, 3)), training=False)


# ------------------------------------------------------------------------------------------ 3. fixtures
@pytest.mark.parametrize("gen", ["init_weights", "stress_weights"])
@pytest.mark.parametrize("name", sorted(lo.SMALL) + sorted(lo.BENCH))
def test_fixtures_equal_spec(name, gen):
    cfg = lo.make_config(**{**lo.SMALL, **lo.BENCH}[name])
    w = getattr(lo, gen)(cfg, lo.WEIGHT_SEED)
    img = lo.make_image(cfg, lo.BATCH, lo.IMAGE_SEED)
    z = np.load(os.path.join(GOLDEN, f"{name}__{gen}__refshim.npz"))
    ref = lo.forward(img, w, cfg)
    tag = "f64" if name in lo.SMALL else "f32"
    fix = (z[f"logits_ref_{tag}"],) + ((z[f"distill_ref_{tag}"],) if f"distill_ref_{tag}" in z.files else ())
    tol = 1e-12 if tag == "f64" else 5e-4
    for f, r in _pairs(fix if len(fix) > 1 else fix[0], ref):
        assert np.abs(f - r).max() <= tol * max(1.0, np.abs(r).max())


# ------------------------------------------------------------------------------------------ 4. host class surface
REF_CTOR = "(self, image_size, num_classes, dim, depth, heads, mlp_mult, stages=3, dim_key=32, dim_value=64, dropout=0.0, num_distill_classes=None)"


def test_constructor_and_call_signatures_match_the_reference():
    from vit_tensorflow_b200 import LeViT
    src = open(os.path.join(REF_DIR, "levit.py")).read() if os.path.exists(os.path.join(REF_DIR, "levit.py")) else None
    ctor = inspect.signature(LeViT.__init__)
    params = [p for p in ctor.parameters.values() if p.kind is not inspect.Parameter.KEYWORD_ONLY]
    assert "(" + ", ".join(str(p) for p in params) + ")" == REF_CTOR.replace(" = ", "=")
    call = inspect.signature(LeViT.call)
    assert str(call) == "(self, img, training=True, **kwargs)"
    if src is not None:
        assert re.sub(r"\s+", " ", "def __init__(self, image_size, num_classes, dim, depth, heads, mlp_mult, stages=3, dim_key=32, "
                      "dim_value=64, dropout=0.0, num_distill_classes=None ):") in re.sub(r"\s+", " ", src).replace(" = ", "=")
        assert "def call(self, img, training=True, **kwargs):" in src
    from vit_tensorflow.levit import LeViT as Shim
    assert Shim is LeViT


def test_constructor_errors_match_the_reference(lib):
    from vit_tensorflow_b200 import LeViT, models
    assert models.levit_cast_tuple(3, 3) == (3, 3, 3) and models.levit_cast_tuple((1, 2), 4) == (1, 2, 2, 2)
    assert models.levit_cast_tuple((1, 2, 3, 4), 2) == (1, 2, 3, 4)
    with pytest.raises(AssertionError, match="dimensions, depths, and heads must be a tuple that is less than the designated number of stages"):
        LeViT(image_size=64, num_classes=3, dim=(32, 32, 32, 32), depth=1, heads=2, mlp_mult=2)
    with pytest.raises(ValueError, match=r"image_size // 16 = 12"):
        LeViT(image_size=200, num_classes=3, dim=32, depth=1, heads=2, mlp_mult=2)


def test_levit_config_layout_matches_header():
    from vit_tensorflow_b200 import _lib
    src = open(os.path.join(ROOT, "include", "vitb200.h")).read()
    body = src[src.index("typedef struct vb_levit_config {"):src.index("} vb_levit_config;")]
    fields = []
    for line in body.splitlines():
        line = line.split("/*")[0].strip()
        if line.startswith("int32_t"):
            fields += [f.strip() for f in line[len("int32_t"):].rstrip(";").split(",")]
    want = [(f.split("[")[0], 8 if "[" in f else 1) for f in fields]
    got = [(n, getattr(t, "_length_", 1)) for n, t in _lib.VbLevitConfig._fields_]
    assert got == want and C.sizeof(_lib.VbLevitConfig) == 4 * (6 + 3 * 8)
    assert int(re.search(r"#define VB_LEVIT_MAX_STAGES (\d+)", src).group(1)) == _lib.LEVIT_MAX_STAGES
    assert int(re.search(r"VB_KIND_LEVIT = (\d+)", src).group(1)) == _lib.KIND["levit"] == 8


def test_vb_create_refuses_levit_and_names_vb_create_levit(lib):
    from vit_tensorflow_b200 import _lib
    cfg = _lib.VbConfig()
    cfg.struct_size = C.sizeof(_lib.VbConfig)
    cfg.kind = _lib.KIND["levit"]
    cfg.image_h = cfg.image_w = 224
    cfg.channels, cfg.num_classes = 3, 10
    h = C.c_void_p()
    assert lib.vb_create(C.byref(cfg), 0, C.byref(h)) != 0 and not h.value
    assert b"vb_create_levit" in lib.vb_last_error(None)
    lv = _lib.VbLevitConfig()
    lv.struct_size = C.sizeof(_lib.VbLevitConfig) + 4
    assert lib.vb_create_levit(C.byref(cfg), C.byref(lv), 0, C.byref(h)) != 0
    assert b"vb_levit_config.struct_size" in lib.vb_last_error(None)

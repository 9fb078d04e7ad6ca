"""CPU tests of the MobileViT oracle (tests/mobilevit_oracle.py) and of the host side of MobileViT:

1. the stand-in's grouped Conv2D (depthwise, stride 1 and 2, SAME) against torch;
2. the reference's own mobile_vit.py, run unmodified over the stand-in, equals the float64 spec, and the PyTorch restatement equals
   the spec, on every small case with both weight generators;
3. the committed fixtures tests/golden/mobilevit_*__refshim.npz equal both restatements, relative to each case's logit scale;
4. the constructor / call signatures, defaults and assert messages match the reference's, and the configurations the engine
   refuses (expansion 1 with channels[2] != channels[3], trunk maps not divisible by patch_size) raise ValueError naming the block
   or stage;
5. the vb_mobilevit_config layout matches the header, and vb_create refuses VB_KIND_MOBILEVIT with a pointer to vb_create_mobilevit."""
import ctypes as C
import inspect
import os
import re

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import mobilevit_oracle as mo
from oracle import tf_shim

REF_DIR = os.environ.get("VB_REFERENCE_DIR", "/root/reference/vit_tensorflow")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
live = pytest.mark.skipif(not os.path.exists(os.path.join(REF_DIR, "mobile_vit.py")),
                          reason="reference checkout not present: the fixtures cover it")
CASES = [(n, g) for n in mo.SMALL for g in ("init_weights", "stress_weights")]


def _tol(ref, rel):
    return rel * max(1.0, float(np.abs(ref).max()))


# ------------------------------------------------------------------------------------------ 1. the stand-in's grouped Conv2D
@pytest.mark.parametrize("H,W,stride", [(7, 6, 1), (7, 6, 2), (8, 5, 2)])
def test_shim_depthwise_conv_against_torch(H, W, stride):
    rng = np.random.default_rng(5)
    x = rng.standard_normal((2, H, W, 6))
    k = rng.standard_normal((3, 3, 1, 6))
    tf_shim.set_dtype(np.float64)
    try:
        with mo.installed(None):
            import tensorflow.keras.layers as nn
            conv = nn.Conv2D(filters=6, kernel_size=3, strides=stride, padding='SAME', groups=6, use_bias=False)
            conv(x)
            conv.set_weights([k])
            got = np.asarray(conv(x))
    finally:
        tf_shim.set_dtype(np.float32)
    xt = torch.from_numpy(x).permute(0, 3, 1, 2)
    oh, ow = -(-H // stride), -(-W // stride)
    ph, pw = max((oh - 1) * stride + 3 - H, 0), max((ow - 1) * stride + 3 - W, 0)
    want = F.conv2d(F.pad(xt, (pw // 2, pw - pw // 2, ph // 2, ph - ph // 2)), torch.from_numpy(k).permute(3, 2, 0, 1), stride=stride,
                    groups=6).permute(0, 2, 3, 1).numpy()
    np.testing.assert_allclose(got, want, atol=1e-12)
    np.testing.assert_allclose(mo._dwconv(x, k, stride), want, atol=1e-12)


# ------------------------------------------------------------------------------------------ 2. the reference's code vs the spec
@pytest.fixture(scope="module")
def ref_module():
    with mo.reference_module(REF_DIR) as mod:
        yield mod


@live
@pytest.mark.parametrize("name,gen", CASES)
def test_live_reference_equals_spec(ref_module, name, gen):
    cfg = mo.make_config(**mo.SMALL[name])
    w, img = getattr(mo, gen)(cfg, mo.WEIGHT_SEED), mo.make_image(cfg, mo.BATCH, mo.IMAGE_SEED)
    ref = mo.reference_logits(ref_module, cfg, w, img)
    np.testing.assert_allclose(ref, mo.forward(img, w, cfg), rtol=0, atol=_tol(ref, 1e-12))


@pytest.mark.parametrize("name,gen", CASES)
def test_torch_restatement_equals_spec(name, gen):
    cfg = mo.make_config(**mo.SMALL[name])
    w, img = getattr(mo, gen)(cfg, mo.WEIGHT_SEED), mo.make_image(cfg, mo.BATCH, mo.IMAGE_SEED)
    want = mo.forward(img, w, cfg)
    np.testing.assert_allclose(mo.forward_torch(img, w, cfg), want, rtol=0, atol=_tol(want, 1e-12))


# ------------------------------------------------------------------------------------------ 3. fixtures
@pytest.mark.parametrize("name,gen", CASES)
def test_fixtures_equal_both_restatements(name, gen):
    cfg = mo.make_config(**mo.SMALL[name])
    w, img = getattr(mo, gen)(cfg, mo.WEIGHT_SEED), mo.make_image(cfg, mo.BATCH, mo.IMAGE_SEED)
    with np.load(os.path.join(GOLDEN, f"{name}__{gen}__refshim.npz")) as z:
        ref64, ref32 = z["logits_ref_f64"], z["logits_ref_f32"]
    scale = np.abs(ref64).max()                     # relative to the case's own logits: with initial weights they are 1e-5 to 4e-2
    for got in (mo.forward(img, w, cfg), mo.forward_torch(img, w, cfg)):
        np.testing.assert_allclose(got, ref64, rtol=0, atol=1e-10 * scale)
        np.testing.assert_allclose(got, ref32, rtol=0, atol=1e-5 * scale)   # the reference run in float32: measured <= 1.5e-6


# ------------------------------------------------------------------------------------------ 4. host class surface
REF_CTOR = "(self, image_size, dims, channels, num_classes, expansion=4, kernel_size=3, patch_size=(2, 2), depths=(2, 4, 3))"


def test_constructor_and_call_signatures_match_the_reference():
    from vit_tensorflow_b200 import MobileViT
    ctor = inspect.signature(MobileViT.__init__)
    params = [p for p in ctor.parameters.values() if p.kind is not inspect.Parameter.KEYWORD_ONLY]
    assert "(" + ", ".join(str(p) for p in params) + ")" == REF_CTOR
    assert [p.name for p in ctor.parameters.values() if p.kind is inspect.Parameter.KEYWORD_ONLY] == ["precision", "device", "seed"]
    assert str(inspect.signature(MobileViT.call)) == "(self, img, training=True, **kwargs)"
    path = os.path.join(REF_DIR, "mobile_vit.py")
    if os.path.exists(path):
        src = re.sub(r"\s+", " ", open(path).read())
        assert "def __init__(self, image_size, dims, channels, num_classes, expansion=4, kernel_size=3, patch_size=(2, 2), depths=(2, 4, 3) ):" in src
        assert "def call(self, x, training=True, **kwargs):" in src
        assert "assert len(dims) == 3, 'dims must be a tuple of 3'" in src
        assert "assert len(depths) == 3, 'depths must be a tuple of 3'" in src
    from vit_tensorflow.mobile_vit import MobileViT as Shim
    assert Shim is MobileViT


XS = dict(image_size=(256, 256), num_classes=10, **mo.XS)


def test_constructor_asserts_match_the_reference():
    from vit_tensorflow_b200 import MobileViT
    with pytest.raises(AssertionError, match="dims must be a tuple of 3"):
        MobileViT(**{**XS, "dims": (96, 120)})
    with pytest.raises(AssertionError, match="depths must be a tuple of 3"):
        MobileViT(**XS, depths=(2, 4))
    with pytest.raises(AssertionError):
        MobileViT(**{**XS, "image_size": (255, 256)})


def test_expansion_one_refusal_names_the_block():
    from vit_tensorflow_b200.models import mobilevit_blocks
    ch = (16, 32, 48, 56, 64, 64, 80, 80, 96, 96, 384)
    with pytest.raises(ValueError, match=r"MobileViT stem\.3: with expansion 1 .*channels\[2\] != channels\[3\]"):
        mobilevit_blocks(ch, 1)
    blocks = mobilevit_blocks(ch, 4)                               # with an expand convolution the block runs (hidden 192, no residual)
    assert blocks[3] == ("stem.3", 56, 192, 56, 1, True, False)
    assert [b[6] for b in mobilevit_blocks(mo.XS["channels"], 4)] == [False, False, True, True, False, False, False]


@pytest.mark.parametrize("name", sorted(mo.SMALL) + sorted(mo.BENCH))
def test_host_block_widths_equal_the_oracles(name):
    """The widths, hidden widths and residual flags the host passes to the engine equal the oracle's own restatement of the wiring."""
    from vit_tensorflow_b200.models import mobilevit_blocks
    cfg = mo.make_config(**{**mo.SMALL, **mo.BENCH}[name])
    assert mobilevit_blocks(cfg["channels"], cfg["expansion"]) == mo.blocks(cfg)


@pytest.mark.parametrize("size,stage", [((96, 96), 3), ((64, 80), 2), ((40, 64), 1)])
def test_map_sizes_the_regrouping_cannot_take_are_refused(size, stage):
    from vit_tensorflow_b200 import MobileViT
    from vit_tensorflow_b200.models import mobilevit_size_error
    err = mobilevit_size_error(*size, 2, 2)
    assert err is not None and err.startswith(f"MobileViT stage {stage}: ") and "not divisible by patch_size (2, 2)" in err
    with pytest.raises(ValueError, match=f"MobileViT stage {stage}: "):
        MobileViT(**{**XS, "image_size": size})
    assert mobilevit_size_error(256, 256, 2, 2) is None and mobilevit_size_error(64, 128, 2, 4) is None


# ------------------------------------------------------------------------------------------ 5. ABI
def test_mobilevit_config_layout_matches_header():
    from vit_tensorflow_b200 import _lib
    src = open(os.path.join(ROOT, "include", "vitb200.h")).read()
    body = src[src.index("typedef struct vb_mobilevit_config {"):src.index("} vb_mobilevit_config;")]
    n = int(re.search(r"#define VB_MOBILEVIT_MV2 (\d+)", src).group(1))
    fields = []
    for line in body.splitlines():
        line = line.split("/*")[0].strip()
        if line.startswith("int32_t"):
            fields += [f.strip() for f in line[len("int32_t"):].rstrip(";").split(",")]
    want = []
    for f in fields:
        m = re.match(r"(\w+)(?:\[(\w+)\])?", f)
        want.append((m.group(1), 1 if m.group(2) is None else (n if m.group(2) == "VB_MOBILEVIT_MV2" else int(m.group(2)))))
    got = [(name, getattr(t, "_length_", 1)) for name, t in _lib.VbMobilevitConfig._fields_]
    assert got == want and n == _lib.MOBILEVIT_MV2 == 7
    assert int(re.search(r"VB_KIND_MOBILEVIT = (\d+)", src).group(1)) == _lib.KIND["mobilevit"] == 16


def test_vb_create_refuses_mobilevit_and_names_vb_create_mobilevit(lib):
    from vit_tensorflow_b200 import _lib
    cfg = _lib.VbConfig()
    cfg.struct_size = C.sizeof(_lib.VbConfig)
    cfg.kind = _lib.KIND["mobilevit"]
    cfg.image_h = cfg.image_w = 256
    cfg.channels, cfg.num_classes = 3, 10
    h = C.c_void_p()
    assert lib.vb_create(C.byref(cfg), 0, C.byref(h)) != 0 and not h.value
    assert b"vb_create_mobilevit" in lib.vb_last_error(None)
    mc = _lib.VbMobilevitConfig()
    mc.struct_size = C.sizeof(_lib.VbMobilevitConfig) + 4
    assert lib.vb_create_mobilevit(C.byref(cfg), C.byref(mc), 0, C.byref(h)) != 0
    assert b"vb_mobilevit_config.struct_size" in lib.vb_last_error(None)

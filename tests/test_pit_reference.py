"""CPU tests of the PiT oracle (tests/pit_oracle.py) and of the host side of PiT:

1. the float64 restatement equals the committed fixtures of the reference's own pit.py over the numpy stand-in
   (tests/golden/make_pit_golden.py), and a live run of the reference equals them where the checkout exists, also at call-time
   images smaller than image_size (the first n + 1 rows of pos_embedding) and rectangular ones;
2. the constructor surface: parameter list, defaults, assert messages and error types as the reference's;
3. the zip(depth, cast_tuple(heads)) truncation and the per-stage to_out rule in the weight names;
4. the vb_pit_config layout and kind number match the header, and vb_create refuses VB_KIND_PIT with a pointer to vb_create_pit."""
import ctypes as C
import inspect
import os
import re

import numpy as np
import pytest

import pit_oracle as po

REF_DIR = os.environ.get("VB_REFERENCE_DIR", "/root/reference/vit_tensorflow")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
live = pytest.mark.skipif(not os.path.exists(os.path.join(REF_DIR, "pit.py")), reason="reference checkout not present: the fixtures cover it")
CASES = [(n, g) for n in po.SMALL for g in po.WEIGHTS]


def _case(name, gen):
    cfg = po.make_config(**po.SMALL[name])
    return cfg, getattr(po, gen)(cfg, po.WEIGHT_SEED), po.make_image(cfg, po.BATCH, po.IMAGE_SEED)


# ------------------------------------------------------------------------------------------ 1. the restatement vs the reference
@pytest.mark.parametrize("name,gen", CASES)
def test_spec_matches_reference_fixture(name, gen):
    cfg, w, img = _case(name, gen)
    r = po.forward(img, w, cfg)
    with np.load(os.path.join(GOLDEN, po.fixture_name(name, gen))) as z:
        np.testing.assert_allclose(r, z["logits_ref_f64"], rtol=0, atol=1e-5)
        np.testing.assert_allclose(r, z["logits_ref_f32"], rtol=0, atol=1e-4 * max(1.0, np.abs(r).max()))


@pytest.fixture(scope="module")
def ref_module():
    with po.reference_module(REF_DIR) as mod:
        yield mod


@live
@pytest.mark.parametrize("name,gen", CASES)
def test_live_reference_matches_fixture(ref_module, name, gen):
    cfg, w, img = _case(name, gen)
    with np.load(os.path.join(GOLDEN, po.fixture_name(name, gen))) as z:
        np.testing.assert_allclose(po.reference_logits(ref_module, cfg, w, img), z["logits_ref_f64"], rtol=0, atol=1e-10)


@live
@pytest.mark.parametrize("hw", [(30, 30), (20, 32), (16, 36), (36, 16)])
def test_live_reference_at_smaller_and_rectangular_images(ref_module, hw):
    """pit_stream is built for 36^2 (289 patches): smaller and rectangular images use the first n + 1 rows of pos_embedding."""
    cfg = po.make_config(**po.SMALL["pit_stream"])
    w = po.stress_weights(cfg, 5)
    model = ref_module.PiT(**po.ctor_kwargs(cfg))
    model(po.make_image(cfg, 1), training=False)
    po.load_weights(model, {k: np.asarray(v, np.float64) for k, v in w.items()}, cfg)
    img = po.make_image(cfg, 2, 7, *hw)
    ref = np.asarray(model(img.astype(np.float64), training=False)).view(np.ndarray)
    np.testing.assert_allclose(ref, po.forward(img, w, cfg), rtol=0, atol=1e-10)


@live
def test_live_reference_fails_with_more_patches_than_the_table(ref_module):
    cfg = po.make_config(**po.SMALL["pit_p8"])
    model = ref_module.PiT(**po.ctor_kwargs(cfg))
    with pytest.raises(ValueError):                          # x += pos_embedding[:, :n + 1] cannot broadcast
        model(po.make_image(cfg, 1, 0, 40, 32), training=False)


def test_patches_known_answer():
    """Pixel (y, x) channel c holds 100 y + 10 x + c + 1: every element of a patch vector names the pixel it came from, in
    (row, column, channel) order, windows at stride p // 2 with the VALID count (odd p: the last pixels are never covered)."""
    H, W, p = 11, 8, 5
    yy, xx, cc = np.meshgrid(np.arange(H), np.arange(W), np.arange(3), indexing="ij")
    img = (100.0 * yy + 10.0 * xx + cc + 1)[None]
    got = po.patches(img, p)
    oh, ow = (H - p) // 2 + 1, (W - p) // 2 + 1
    assert got.shape == (1, oh * ow, p * p * 3) and (oh, ow) == (4, 2)
    for t in range(oh * ow):
        gy, gx = divmod(t, ow)
        for r in range(p):
            for c in range(p):
                for ch in range(3):
                    assert got[0, t, (r * p + c) * 3 + ch] == 100.0 * (2 * gy + r) + 10.0 * (2 * gx + c) + ch + 1


# ------------------------------------------------------------------------------------------ 2. constructor surface
REF_CTOR = "(self, image_size, patch_size, num_classes, dim, depth, heads, mlp_dim, dim_head=64, dropout=0.0, emb_dropout=0.0)"
ARGS = dict(image_size=32, patch_size=8, num_classes=10, dim=64, depth=(1, 1), heads=2, mlp_dim=64)
DEPTH_MSG = "depth must be a tuple of integers, specifying the number of blocks before each downsizing"
ERRORS = [(dict(image_size=30), AssertionError, "Image dimensions must be divisible by the patch size."),
          (dict(image_size=30, depth=[1]), AssertionError, "Image dimensions must be divisible by the patch size."),
          (dict(depth=[1, 1]), AssertionError, DEPTH_MSG),
          (dict(patch_size=1), ZeroDivisionError, None),
          (dict(image_size=(32, 32)), TypeError, None)]


def test_constructor_and_call_signatures_match_the_reference():
    from vit_tensorflow_b200 import PiT
    ctor = inspect.signature(PiT.__init__)
    params = [p for p in ctor.parameters.values() if p.kind is not inspect.Parameter.KEYWORD_ONLY]
    assert "(" + ", ".join(str(p) for p in params) + ")" == REF_CTOR
    assert [p.name for p in ctor.parameters.values() if p.kind is inspect.Parameter.KEYWORD_ONLY] == ["precision", "device", "seed"]
    assert str(inspect.signature(PiT.call)) == "(self, img, training=True, **kwargs)"
    from vit_tensorflow.pit import PiT as Shim
    assert Shim is PiT


@live
def test_signatures_match_live_reference(ref_module):
    from vit_tensorflow_b200 import PiT
    ref = inspect.signature(ref_module.PiT.__init__)
    assert "(" + ", ".join(str(p) for p in ref.parameters.values()) + ")" == REF_CTOR
    assert str(inspect.signature(ref_module.PiT.call)) == str(inspect.signature(PiT.call))
    src = open(os.path.join(REF_DIR, "pit.py")).read()
    assert "not_last = ind < (len(depth) < 1)" in src                      # the line that keeps Pool from ever being built


@pytest.mark.parametrize("kw,exc,msg", ERRORS)
def test_constructor_errors(kw, exc, msg):
    from vit_tensorflow_b200 import PiT
    with pytest.raises(exc) as e:
        PiT(**dict(ARGS, **kw))
    if msg is not None:
        assert str(e.value) == msg


@live
@pytest.mark.parametrize("kw,exc,msg", ERRORS)
def test_constructor_errors_match_live_reference(ref_module, kw, exc, msg):
    with pytest.raises(exc) as e:
        ref_module.PiT(**dict(ARGS, **kw))
    if msg is not None:
        assert str(e.value) == msg


@pytest.mark.parametrize("heads", [[2, 2], 2.0, (2, "4"), None, True])
def test_heads_of_another_type_refused_at_construction(heads):
    from vit_tensorflow_b200 import PiT
    with pytest.raises(TypeError, match="heads must be an int or a tuple of ints"):
        PiT(**dict(ARGS, heads=heads))


def test_engine_limits_refused_at_construction():
    """Limits the reference does not have: more than 8 stages after the zip, more than 32 heads in a stage."""
    from vit_tensorflow_b200 import PiT
    with pytest.raises(NotImplementedError, match="at most 8 stages"):
        PiT(**dict(ARGS, depth=(1,) * 9))
    with pytest.raises(NotImplementedError, match="1 to 32 heads per stage"):
        PiT(**dict(ARGS, heads=(2, 33)))


def test_mixed_folding_cases_mix_folding():
    """The bf16 engine folds a stage's LayerNorms into its GEMMs when heads * dim_head is a multiple of 64 (dim 64, mlp 64 here):
    these cases put an unfolded stage before a folded one."""
    for name, want in (("pit_unfold_fold", [False, True]), ("pit_fold_unfold_fold", [True, False, True])):
        cfg = po.make_config(**po.SMALL[name])
        assert [h * cfg["dim_head"] % 64 == 0 for _, _, h, _ in po.layer_plan(cfg)] == want


# ------------------------------------------------------------------------------------------ 3. stages and weight names
def test_zip_truncation_and_to_out_rule_in_weight_specs():
    from vit_tensorflow_b200.models import pit_stages
    assert pit_stages((1, 2, 3), (2, 4)) == ((1, 2), (2, 4))                # heads shorter: trailing stage dropped
    assert pit_stages((1, 2), (2, 4, 8)) == ((1, 2), (2, 4))                # heads longer: cut
    assert pit_stages((3, 3, 3), 16) == ((3, 16),) * 3
    assert pit_stages((), 4) == ()
    short = po.make_config(**po.SMALL["pit_heads_short"])
    names = po.weight_specs(short)
    assert [L for L, *_ in po.layer_plan(short)] == [0, 1, 2] and "layers.3.to_qkv.kernel" not in names
    assert names["layers.0.to_qkv.kernel"][0] == (48, 3 * 2 * 16) and names["layers.2.to_qkv.kernel"][0] == (48, 3 * 4 * 16)
    st = po.make_config(**po.SMALL["pit_p2_stages"])                        # stage 0: heads 1, dim_head 64 == dim
    names = po.weight_specs(st)
    assert "layers.0.to_out.kernel" not in names and "layers.0.to_out.bias" not in names
    assert names["layers.1.to_out.kernel"][0] == (128, 64) and names["layers.2.to_out.kernel"][0] == (256, 64)
    dh80 = po.weight_specs(po.make_config(**po.SMALL["pit_dh80"]))          # one head of 80 != dim 64: to_out kept
    assert dh80["layers.1.to_out.kernel"][0] == (80, 64)
    assert po.weight_specs(po.make_config(**po.SMALL["pit_p5_odd"]))["pos_embedding"][0] == (1, 13 * 13 + 1, 64)


def test_readme_geometry():
    cfg = po.make_config(**po.README)
    assert po.num_patches(cfg) == 31 * 31 == 961
    assert [L for L, *_ in po.layer_plan(cfg)] == list(range(9))


# ------------------------------------------------------------------------------------------ 4. ABI
def test_pit_config_layout_matches_header():
    from vit_tensorflow_b200 import _lib
    src = open(os.path.join(ROOT, "include", "vitb200.h")).read()
    body = src[src.index("typedef struct vb_pit_config {"):src.index("} vb_pit_config;")]
    n = int(re.search(r"#define VB_PIT_MAX_STAGES (\d+)", src).group(1))
    fields = []
    for line in body.splitlines():
        line = line.split("/*")[0].strip()
        if line.startswith("int32_t"):
            fields += [f.strip() for f in line[len("int32_t"):].rstrip(";").split(",")]
    want = []
    for f in fields:
        m = re.match(r"(\w+)(?:\[(\w+)\])?", f)
        want.append((m.group(1), 1 if m.group(2) is None else n))
    got = [(name, getattr(t, "_length_", 1)) for name, t in _lib.VbPitConfig._fields_]
    assert got == want == [("struct_size", 1), ("stages", 1), ("depth", n), ("heads", n)] and n == _lib.PIT_MAX_STAGES == 8
    assert int(re.search(r"VB_KIND_PIT = (\d+)", src).group(1)) == _lib.KIND["pit"] == 18


def test_vb_create_refuses_pit_and_names_vb_create_pit(lib):
    from vit_tensorflow_b200 import _lib
    cfg = _lib.VbConfig()
    cfg.struct_size = C.sizeof(_lib.VbConfig)
    cfg.kind = _lib.KIND["pit"]
    cfg.image_h = cfg.image_w = 224
    cfg.patch_h = cfg.patch_w = 14
    cfg.channels, cfg.num_classes, cfg.dim, cfg.dim_head, cfg.mlp_dim = 3, 10, 64, 64, 64
    h = C.c_void_p()
    assert lib.vb_create(C.byref(cfg), 0, C.byref(h)) != 0 and not h.value
    assert b"vb_create_pit" in lib.vb_last_error(None)
    pc = _lib.VbPitConfig()
    pc.struct_size = C.sizeof(_lib.VbPitConfig) + 4
    assert lib.vb_create_pit(C.byref(cfg), C.byref(pc), 0, C.byref(h)) != 0
    assert b"vb_pit_config.struct_size" in lib.vb_last_error(None)
    pc.struct_size = C.sizeof(_lib.VbPitConfig)
    pc.stages, pc.depth[0], pc.heads[0] = 1, 1, 33
    assert lib.vb_create_pit(C.byref(cfg), C.byref(pc), 0, C.byref(h)) != 0
    assert b"1 to 32 heads" in lib.vb_last_error(None)

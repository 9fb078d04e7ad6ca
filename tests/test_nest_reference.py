"""CPU tests of the NesT oracle (tests/nest_oracle.py) and of the host side of NesT:

1. the reference's own nest.py, run unmodified over the stand-in, equals the float64 spec to 1e-12 on the hand-picked cases and
   40 seeded random configurations, and the PyTorch restatement equals the spec to 1e-5;
2. block_repeats is zipped with the hierarchies as in the reference: a longer tuple is truncated, a shorter one builds fewer
   levels (and runs only on images whose blocks still fit seq_len);
3. the image sizes the host class refuses are the ones the reference fails on;
4. the committed fixtures tests/golden/nest_*__refshim.npz equal the spec;
5. the constructor / call signatures, defaults and assert message match the reference's;
6. the vb_nest_config layout matches the header, vb_create refuses VB_KIND_NEST with a pointer to vb_create_nest, and
   vb_create_nest names its level limit."""
import ctypes as C
import inspect
import os
import re

import numpy as np
import pytest

import nest_oracle as no

REF_DIR = os.environ.get("VB_REFERENCE_DIR", "/root/reference/vit_tensorflow")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
HAVE_REF = os.path.exists(os.path.join(REF_DIR, "nest.py"))
live = pytest.mark.skipif(not HAVE_REF, reason="reference checkout not present: the fixtures cover it")


def _tol(ref):
    return 1e-12 * max(1.0, float(np.abs(ref).max()))


@pytest.fixture(scope="module")
def ref_module():
    if not HAVE_REF:
        pytest.skip("reference checkout not present: the fixtures cover it")
    with no.reference_module(REF_DIR) as mod:
        yield mod


# ------------------------------------------------------------------------------------------ 1. live reference
@live
@pytest.mark.parametrize("name", sorted(no.SMALL))
def test_live_reference_equals_spec(ref_module, name):
    cfg = no.make_config(**no.SMALL[name])
    w = no.stress_weights(cfg, 4)
    img = no.make_image(cfg, 2, 5)
    ref = no.forward(img, w, cfg)
    got = no.reference_logits(ref_module, cfg, w, img)
    assert got.shape == ref.shape and np.abs(got - ref).max() <= _tol(ref)
    assert np.abs(no.forward_torch(img, w, cfg) - ref).max() <= 1e-5 * max(1.0, np.abs(ref).max())


def test_hand_picked_cases_cover_the_ground():
    """H = 1 .. 4; head widths 32, 64 and 24; a width not a multiple of 64; blocks under and over 64 tokens; block_repeats as an
    int and as a tuple; mlp_mult 2; a rectangular image."""
    hs, dhs, odd_width, small, large, as_int, as_tuple, mult2, rect = set(), set(), False, False, False, False, False, False, False
    for kw in no.SMALL.values():
        cfg = no.make_config(**kw)
        pl = no.plan(cfg)
        hs.add(cfg["num_hierarchies"])
        dhs.add(cfg["dim"] // cfg["heads"])
        odd_width |= any(lv["dim"] % 64 for lv in pl["levels"])
        h, w = cfg["image_h"] // cfg["patch_size"], cfg["image_w"] // cfg["patch_size"]
        n = len(pl["levels"])
        for i, lv in enumerate(pl["levels"]):
            bs = 2 ** (n - 1 - i)
            small |= (h // bs) * (w // bs) < 64
            large |= (h // bs) * (w // bs) > 64
            if lv["aggregate"]:
                h, w = -(-h // 2), -(-w // 2)
        as_int |= isinstance(cfg["block_repeats"], int)
        as_tuple |= isinstance(cfg["block_repeats"], tuple)
        mult2 |= cfg["mlp_mult"] == 2
        rect |= cfg["image_h"] != cfg["image_w"]
    assert {1, 2, 3, 4} <= hs and {24, 32, 64} <= dhs
    assert odd_width and small and large and as_int and as_tuple and mult2 and rect


@live
def test_live_reference_equals_spec_on_random_configurations(ref_module):
    """40 seeded random configurations: 1 to 4 hierarchies, head widths 8 to 64, block_repeats short, exact or long, and square
    or non-square images."""
    hs, lengths, nonsquare = set(), set(), False
    for seed in range(40):
        cfg = no.random_config(seed)
        hs.add(cfg["num_hierarchies"])
        br = cfg["block_repeats"]
        lengths.add(0 if isinstance(br, int) else (len(br) > cfg["num_hierarchies"]) - (len(br) < cfg["num_hierarchies"]) + 2)
        nonsquare |= cfg["image_h"] != cfg["image_w"]
        wts = no.stress_weights(cfg, seed)
        img = no.make_image(cfg, 2, seed + 1)
        ref = no.forward(img, wts, cfg)
        got = no.reference_logits(ref_module, cfg, wts, img)
        assert got.shape == ref.shape and np.abs(got - ref).max() <= _tol(ref), (seed, cfg)
        if seed < 8:
            assert np.abs(no.forward_torch(img, wts, cfg) - ref).max() <= 1e-5 * max(1.0, np.abs(ref).max()), (seed, cfg)
    assert hs == {1, 2, 3, 4} and lengths == {0, 1, 2, 3} and nonsquare


# ------------------------------------------------------------------------------------------ 2. the block_repeats zip
@live
def test_long_block_repeats_is_truncated_as_in_the_reference(ref_module):
    cfg = no.make_config(image_size=32, patch_size=4, dim=32, heads=1, num_hierarchies=2, block_repeats=(1, 2, 5), num_classes=3)
    pl = no.plan(cfg)
    assert [lv["depth"] for lv in pl["levels"]] == [1, 2]
    model = no.reference_model(ref_module, cfg, no.init_weights(cfg), no.make_image(cfg, 1))
    assert [len(tr.layers) for tr, _ in model.nest_layers] == [1, 2]
    assert set(no.weight_specs(cfg)) == set(no.weight_specs(no.make_config(**{**cfg, "block_repeats": (1, 2)})))


@live
def test_short_block_repeats_builds_fewer_levels_as_in_the_reference(ref_module):
    """A tuple one short gives num_hierarchies - 1 levels, each with an Aggregate (none is `is_last`), blocks relative to the levels
    built; it runs only on images small enough that the first level's blocks still fit seq_len.  Two short fails at the head."""
    cfg = no.make_config(**no.SMALL["nest_short"])
    pl = no.plan(cfg)
    assert len(pl["levels"]) == 2 and all(lv["aggregate"] for lv in pl["levels"])
    model = no.reference_model(ref_module, cfg, no.init_weights(cfg), no.make_image(cfg, 1))
    assert len(model.nest_layers) == 2 and all(hasattr(ag, "ag_layers") for _, ag in model.nest_layers)
    for h, w in ((64, 64), (32, 32)):
        err = no.size_error(cfg, h, w)
        try:
            ref_module.NesT(**no.ctor_kwargs(cfg))(np.zeros((1, h, w, 3)))
            failed = False
        except Exception:
            failed = True
        assert failed == (err is not None), (h, w, err)
    assert "more than seq_len" in no.size_error(cfg, 64, 64)
    two_short = no.make_config(image_size=64, patch_size=4, dim=32, heads=1, num_hierarchies=3, block_repeats=(1,), num_classes=3)
    assert "head's LayerNorm" in no.size_error(two_short, 16, 16)
    with pytest.raises(Exception):
        ref_module.NesT(**no.ctor_kwargs(two_short))(np.zeros((1, 16, 16, 3)))


# ------------------------------------------------------------------------------------------ 3. refused sizes
@live
@pytest.mark.parametrize("h,w", [(224, 224), (192, 192), (224, 112), (112, 224), (228, 224), (224, 208), (256, 256), (240, 224),
                                 (32, 32), (96, 160)])
def test_refused_sizes_are_the_references_failures(ref_module, h, w):
    """The reference enforces its shape rules through einops (the patch split, the block split, the pos_emb reshape); the host
    class refuses exactly those sizes, naming the level."""
    cfg = no.make_config(image_size=224, patch_size=4, dim=16, heads=1, num_hierarchies=3, block_repeats=1, num_classes=3)
    err = no.size_error(cfg, h, w)
    model = ref_module.NesT(**no.ctor_kwargs(cfg))
    try:
        model(np.zeros((1, h, w, 3)))
        failed = False
    except Exception:                                   # einops.EinopsError or the stand-in's shape errors
        failed = True
    assert failed == (err is not None), err
    if err is not None:
        assert re.match(r"NesT(: the \d+ x \d+ image is not divisible by patch_size \d+| level \d: the \d+ x \d+ map "
                        r"(is not divisible into \d+ x \d+ blocks|has blocks of \d+ x \d+ tokens, more than seq_len \d+ positions))$", err)


# ------------------------------------------------------------------------------------------ 4. fixtures
@pytest.mark.parametrize("gen", ["init_weights", "stress_weights"])
@pytest.mark.parametrize("name", sorted(no.SMALL) + sorted(no.BENCH))
def test_fixtures_equal_spec(name, gen):
    cfg = no.make_config(**{**no.SMALL, **no.BENCH}[name])
    w = getattr(no, gen)(cfg, no.WEIGHT_SEED)
    img = no.make_image(cfg, no.BATCH, no.IMAGE_SEED)
    z = np.load(os.path.join(GOLDEN, f"{name}__{gen}__refshim.npz"))
    ref = no.forward(img, w, cfg)
    tag = "f64" if name in no.SMALL else "f32"
    tol = 1e-12 if tag == "f64" else 5e-4
    assert np.abs(z[f"logits_ref_{tag}"] - ref).max() <= tol * max(1.0, np.abs(ref).max())


# ------------------------------------------------------------------------------------------ 5. host class surface
CTOR = ["image_size", "patch_size", "num_classes", "dim", "heads", "num_hierarchies", "block_repeats", "mlp_mult", "dropout"]


def test_constructor_and_call_signatures_match_the_reference():
    from vit_tensorflow_b200 import NesT
    ctor = inspect.signature(NesT.__init__)
    params = [p for p in ctor.parameters.values() if p.kind is not inspect.Parameter.KEYWORD_ONLY]
    assert [p.name for p in params] == ["self"] + CTOR
    assert {p.name: p.default for p in params[1:] if p.default is not inspect.Parameter.empty} == no.NEST_DEFAULTS
    assert [p.name for p in ctor.parameters.values() if p.kind is inspect.Parameter.KEYWORD_ONLY] == ["precision", "device", "seed"]
    assert str(inspect.signature(NesT.call)) == "(self, img, training=True, **kwargs)"
    if HAVE_REF:
        with no.reference_module(REF_DIR) as mod:
            ref = inspect.signature(mod.NesT.__init__)
            assert [(p.name, p.default) for p in ref.parameters.values()] == [(p.name, p.default) for p in params]
            assert str(inspect.signature(mod.NesT.call)) == "(self, img, training=True, **kwargs)"
    from vit_tensorflow.nest import NesT as Shim
    assert Shim is NesT


def test_constructor_assertion_matches_the_reference():
    from vit_tensorflow_b200 import NesT
    kw = dict(image_size=30, patch_size=4, num_classes=3, dim=32, heads=1, num_hierarchies=2, block_repeats=1)
    with pytest.raises(AssertionError, match="^Image dimensions must be divisible by the patch size.$"):
        NesT(**kw)
    if HAVE_REF:
        with no.reference_module(REF_DIR) as mod:
            with pytest.raises(AssertionError, match="^Image dimensions must be divisible by the patch size.$"):
                mod.NesT(**kw)


def test_too_many_hierarchies_are_refused_naming_the_limit():
    from vit_tensorflow_b200 import NesT, _lib
    with pytest.raises(ValueError, match=f"num_hierarchies 9 .*1 to {_lib.NEST_MAX_LEVELS}"):
        NesT(image_size=2 ** 10, patch_size=2, num_classes=3, dim=8, heads=1, num_hierarchies=9, block_repeats=0)


def test_nest_config_layout_matches_header():
    from vit_tensorflow_b200 import _lib
    src = open(os.path.join(ROOT, "include", "vitb200.h")).read()
    body = src[src.index("typedef struct vb_nest_config {"):src.index("} vb_nest_config;")]
    fields = []
    for line in body.splitlines():
        line = line.split("/*")[0].strip()
        if line.startswith("int32_t"):
            fields += [f.strip() for f in line[len("int32_t"):].rstrip(";").split(",")]
    want = [(f.split("[")[0], _lib.NEST_MAX_LEVELS if "[" in f else 1) for f in fields]
    got = [(n, C.sizeof(t) // 4) for n, t in _lib.VbNestConfig._fields_]
    assert got == want and C.sizeof(_lib.VbNestConfig) == 4 * (8 + _lib.NEST_MAX_LEVELS)
    assert int(re.search(r"#define VB_NEST_MAX_LEVELS (\d+)", src).group(1)) == _lib.NEST_MAX_LEVELS >= 5
    assert int(re.search(r"VB_KIND_NEST = (\d+)", src).group(1)) == _lib.KIND["nest"] == 12


def test_vb_create_refuses_nest_and_names_vb_create_nest(lib):
    from vit_tensorflow_b200 import _lib
    cfg = _lib.VbConfig()
    cfg.struct_size = C.sizeof(_lib.VbConfig)
    cfg.kind = _lib.KIND["nest"]
    cfg.image_h = cfg.image_w = 224
    cfg.channels, cfg.num_classes = 3, 10
    h = C.c_void_p()
    assert lib.vb_create(C.byref(cfg), 0, C.byref(h)) != 0 and not h.value
    assert b"vb_create_nest" in lib.vb_last_error(None)
    nc = _lib.VbNestConfig()
    nc.struct_size = C.sizeof(_lib.VbNestConfig) + 4
    assert lib.vb_create_nest(C.byref(cfg), C.byref(nc), 0, C.byref(h)) != 0
    assert b"vb_nest_config.struct_size" in lib.vb_last_error(None)
    nc.struct_size = C.sizeof(_lib.VbNestConfig)
    nc.patch_size, nc.dim, nc.heads, nc.num_hierarchies, nc.levels, nc.mlp_mult, nc.seq_len = 4, 96, 3, 9, 9, 4, 196
    assert lib.vb_create_nest(C.byref(cfg), C.byref(nc), 0, C.byref(h)) != 0
    assert b"VB_NEST_MAX_LEVELS = 8" in lib.vb_last_error(None)

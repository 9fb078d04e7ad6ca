"""CPU tests of the CrossFormer oracle (tests/crossformer_oracle.py) and of the host side of CrossFormer:

1. the reference's own crossformer.py, run unmodified over the stand-in, equals the float64 spec to 1e-12 on the hand-picked cases
   and 40 seeded random configurations, and the PyTorch restatement equals the spec to 1e-5;
2. the window table the engine keeps (the first (2 w - 1)^2 DynamicPositionBias outputs) is what the reference adds;
3. the image sizes the host class refuses are the ones the reference fails on;
4. the committed fixtures tests/golden/crossformer_*__refshim.npz equal the spec;
5. the constructor / call signatures, defaults and AssertionErrors match the reference's, and the kernel sets the nested
   cross-scale embedding cannot run exactly are refused;
6. the vb_crossformer_config layout matches the header, and vb_create refuses VB_KIND_CROSSFORMER with a pointer to
   vb_create_crossformer."""
import ctypes as C
import inspect
import os
import re

import numpy as np
import pytest

import crossformer_oracle as co

REF_DIR = os.environ.get("VB_REFERENCE_DIR", "/root/reference/vit_tensorflow")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
HAVE_REF = os.path.exists(os.path.join(REF_DIR, "crossformer.py"))
live = pytest.mark.skipif(not HAVE_REF, reason="reference checkout not present: the fixtures cover it")


def _tol(ref):
    return 1e-12 * max(1.0, float(np.abs(ref).max()))


@pytest.fixture(scope="module")
def ref_module():
    if not HAVE_REF:
        pytest.skip("reference checkout not present: the fixtures cover it")
    with co.reference_module(REF_DIR) as mod:
        yield mod


# ------------------------------------------------------------------------------------------ 1. live reference
@live
@pytest.mark.parametrize("name", sorted(co.SMALL))
def test_live_reference_equals_spec(ref_module, name):
    cfg = co.make_config(**co.SMALL[name])
    w = co.stress_weights(cfg, 4)
    img = co.make_image(cfg, 2, 5)
    ref = co.forward(img, w, cfg)
    got = co.reference_logits(ref_module, cfg, w, img)
    assert got.shape == ref.shape and np.abs(got - ref).max() <= _tol(ref)
    assert np.abs(co.forward_torch(img, w, cfg) - ref).max() <= 1e-5 * max(1.0, np.abs(ref).max())


@live
def test_live_reference_equals_spec_on_random_configurations(ref_module):
    """40 seeded random configurations: 1 to 4 kernel sizes of either parity, strides 1 to 4, windows of 1 to 9 tokens a side,
    dims off 64 and non-square images."""
    nkernels, parities, wsizes, nonsquare = set(), set(), set(), False
    for seed in range(40):
        cfg = co.random_config(seed)
        for st in co.stages(cfg):
            nkernels.add(len(st["kernels"]))
            parities.add(st["kernels"][0] % 2)
            wsizes |= {st["local_wsz"], st["global_wsz"]}
        nonsquare |= cfg["image_h"] != cfg["image_w"]
        wts = co.stress_weights(cfg, seed)
        img = co.make_image(cfg, 2, seed + 1)
        ref = co.forward(img, wts, cfg)
        got = co.reference_logits(ref_module, cfg, wts, img)
        assert got.shape == ref.shape and np.abs(got - ref).max() <= _tol(ref), (seed, cfg)
        if seed < 8:
            assert np.abs(co.forward_torch(img, wts, cfg) - ref).max() <= 1e-5 * max(1.0, np.abs(ref).max()), (seed, cfg)
    assert nkernels == {1, 2, 3, 4} and parities == {0, 1} and {1, 2, 3} <= wsizes and nonsquare


# ------------------------------------------------------------------------------------------ 2. the window table
@live
@pytest.mark.parametrize("wsz", [1, 2, 7, 8])
def test_window_table_is_what_the_reference_adds(ref_module, wsz):
    """The reference adds biases[rel_pos_indices] (crossformer.py:158-165); the engine keeps the first (2 wsz - 1)^2 entries and
    indexes them by the signed in-window offset."""
    cfg = co.make_config(image_size=8 * wsz, dim=(32, 32, 32, 32), depth=(1, 0, 0, 0), global_window_size=1, local_window_size=wsz,
                         cross_embed_kernel_sizes=((2,), (1,), (1,), (1,)), cross_embed_strides=(2, 1, 1, 1), num_classes=3)
    w = co.stress_weights(cfg, 7)
    img = co.make_image(cfg, 1, 8)
    model = co.reference_model(ref_module, cfg, w, img)
    attn = model.crossformer_layers[0][1].layers[0][0]
    pos = np.arange(-wsz, wsz + 1)
    rel = np.stack(np.meshgrid(pos, pos, indexing="ij")).reshape(2, -1).T.astype(np.float64)
    biases = np.asarray(attn.dpb(rel)).reshape(-1)
    want = biases[np.asarray(attn.rel_pos_indices).astype(np.int64)]
    table = co.window_table({k: np.asarray(v, np.float64) for k, v in w.items()}, "crossformer_layers.0.1.layers.0.0.dpb.dpb_layers.", wsz)
    n = wsz * wsz
    i, j = np.divmod(np.arange(n), wsz)
    idx = (i[:, None] - i[None, :] + wsz - 1) * (2 * wsz - 1) + (j[:, None] - j[None, :] + wsz - 1)
    assert table.shape == ((2 * wsz - 1) ** 2,) and np.abs(table[idx] - want).max() <= 1e-12 * max(1.0, np.abs(want).max())


# ------------------------------------------------------------------------------------------ 3. refused sizes
@live
@pytest.mark.parametrize("h,w", [(224, 224), (448, 448), (224, 448), (220, 224), (224, 200), (112, 112), (56, 224), (232, 224)])
def test_refused_sizes_are_the_references_failures(ref_module, h, w):
    """The reference enforces its shape rule through einops; the host class refuses exactly those sizes, naming the stage."""
    cfg = co.make_config(image_size=h, image_w=w, num_classes=3, dim=32, depth=(1, 1, 1, 1))
    err = co.size_error(cfg, h, w)
    model = ref_module.CrossFormer(**co.ctor_kwargs(cfg))
    try:
        model(np.zeros((1, h, w, 3)))
        failed = False
    except Exception:                                   # einops.EinopsError or the stand-in's shape errors
        failed = True
    assert failed == (err is not None), err
    if err is not None:
        assert re.match(r"CrossFormer stage [1-4]: the \d+ x \d+ map is not divisible by (local|global)_window_size \d+$", err)


# ------------------------------------------------------------------------------------------ 4. fixtures
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


# ------------------------------------------------------------------------------------------ 5. host class surface
def test_constructor_and_call_signatures_match_the_reference():
    from vit_tensorflow_b200 import CrossFormer
    ctor = inspect.signature(CrossFormer.__init__)
    params = [p for p in ctor.parameters.values() if p.kind is not inspect.Parameter.KEYWORD_ONLY]
    assert [p.name for p in params] == ["self"] + list(co.CROSSFORMER_DEFAULTS)
    assert {p.name: p.default for p in params[1:]} == co.CROSSFORMER_DEFAULTS
    assert [p.name for p in ctor.parameters.values() if p.kind is inspect.Parameter.KEYWORD_ONLY] == ["precision", "device", "seed"]
    assert str(inspect.signature(CrossFormer.call)) == "(self, img, training=True, **kwargs)"
    if HAVE_REF:
        with co.reference_module(REF_DIR) as mod:
            ref = inspect.signature(mod.CrossFormer.__init__)
            assert [(p.name, p.default) for p in ref.parameters.values()] == [(p.name, p.default) for p in params]
            assert str(inspect.signature(mod.CrossFormer.call)) == "(self, x, training=True, **kwargs)"
    from vit_tensorflow.crossformer import CrossFormer as Shim
    assert Shim is CrossFormer


BAD_TUPLES = [dict(dim=(64, 128, 256)), dict(depth=(1, 1)), dict(global_window_size=(8, 4, 2, 1, 1)), dict(local_window_size=(7,)),
              dict(cross_embed_kernel_sizes=((4, 8), (2, 4))), dict(cross_embed_strides=(4, 2, 2))]


@pytest.mark.parametrize("kw", BAD_TUPLES, ids=[next(iter(k)) for k in BAD_TUPLES])
def test_constructor_assertions_match_the_reference(kw):
    """cast_tuple keeps a tuple as it is, so a tuple of the wrong length fails `assert len(...) == 4` (crossformer.py:226-231)
    before anything is built, in both classes."""
    from vit_tensorflow_b200 import CrossFormer
    with pytest.raises(AssertionError):
        CrossFormer(**kw)
    if HAVE_REF:
        with co.reference_module(REF_DIR) as mod:
            with pytest.raises(AssertionError):
                mod.CrossFormer(**kw)


@pytest.mark.parametrize("kernels,stride,what", [(((3, 4),) + ((2, 4),) * 3, 4, "(3, 4)"),
                                                 (((4, 8, 16, 32), (1, 3), (2, 4), (2, 4)), (4, 2, 2, 2), "kernel sizes (1, 3) at stride 2"),
                                                 (((4, 8, 16, 32, 64),) + ((2, 4),) * 3, (4, 2, 2, 2), "5 cross-embedding")])
def test_unsupported_kernel_sets_are_refused(kernels, stride, what):
    """Mixed parities and kernels below the stride put the nested kernels at offsets that depend on the image size; more than four
    kernel sizes exceed the C struct.  The host class raises ValueError naming the stage before any library call."""
    from vit_tensorflow_b200 import CrossFormer
    with pytest.raises(ValueError, match=r"CrossFormer stage \d: .*" + re.escape(what)):
        CrossFormer(cross_embed_kernel_sizes=kernels, cross_embed_strides=stride)


def test_crossformer_config_layout_matches_header():
    from vit_tensorflow_b200 import _lib
    src = open(os.path.join(ROOT, "include", "vitb200.h")).read()
    body = src[src.index("typedef struct vb_crossformer_config {"):src.index("} vb_crossformer_config;")]
    fields = []
    for line in body.splitlines():
        line = line.split("/*")[0].strip()
        if line.startswith("int32_t"):
            fields += [f.strip() for f in line[len("int32_t"):].rstrip(";").split(",")]
    want = [(f.split("[")[0], 4 * (4 if f.count("[") == 2 else 1) if "[" in f else 1) for f in fields]
    got = [(n, C.sizeof(t) // 4) for n, t in _lib.VbCrossformerConfig._fields_]
    assert got == want and C.sizeof(_lib.VbCrossformerConfig) == 4 * (1 + 6 * 4 + 4 * 4)
    assert int(re.search(r"#define VB_CROSSFORMER_STAGES (\d+)", src).group(1)) == _lib.CROSSFORMER_STAGES
    assert int(re.search(r"#define VB_CROSSFORMER_MAX_KERNELS (\d+)", src).group(1)) == _lib.CROSSFORMER_MAX_KERNELS
    assert int(re.search(r"VB_KIND_CROSSFORMER = (\d+)", src).group(1)) == _lib.KIND["crossformer"] == 11


def test_vb_create_refuses_crossformer_and_names_vb_create_crossformer(lib):
    from vit_tensorflow_b200 import _lib
    cfg = _lib.VbConfig()
    cfg.struct_size = C.sizeof(_lib.VbConfig)
    cfg.kind = _lib.KIND["crossformer"]
    cfg.image_h = cfg.image_w = 224
    cfg.channels, cfg.num_classes = 3, 10
    h = C.c_void_p()
    assert lib.vb_create(C.byref(cfg), 0, C.byref(h)) != 0 and not h.value
    assert b"vb_create_crossformer" in lib.vb_last_error(None)
    cf = _lib.VbCrossformerConfig()
    cf.struct_size = C.sizeof(_lib.VbCrossformerConfig) + 4
    assert lib.vb_create_crossformer(C.byref(cfg), C.byref(cf), 0, C.byref(h)) != 0
    assert b"vb_crossformer_config.struct_size" in lib.vb_last_error(None)
    cf.struct_size = C.sizeof(_lib.VbCrossformerConfig)
    for i in range(4):
        cf.dim[i], cf.depth[i], cf.global_wsz[i], cf.local_wsz[i], cf.stride[i], cf.n_kernels[i] = 64, 1, 1, 1, 2, 2
        cf.kernels[i][0], cf.kernels[i][1] = 2, 4
    cf.kernels[1][1] = 3                                 # stage 2: (2, 3), mixed parity
    assert lib.vb_create_crossformer(C.byref(cfg), C.byref(cf), 0, C.byref(h)) != 0
    assert b"CrossFormer stage 2: kernel sizes (2, 3)" in lib.vb_last_error(None)
    cf.kernels[1][1] = 4
    cf.n_kernels[0] = 5
    assert lib.vb_create_crossformer(C.byref(cfg), C.byref(cf), 0, C.byref(h)) != 0
    assert b"CrossFormer stage 1: between 1 and 4" in lib.vb_last_error(None)

"""MAE (reference mae.py:17-92) and SimMIM (simmim.py:72-129) on the CPU.

1. LIVE (skipped where the reference checkout is absent): the float64 restatement (tests/mim_oracle.py) equals the reference's own
   classes over the numpy stand-in for TensorFlow with the same noise: loss, pred, masked patches and mask ids.
2. FIXTURES (always): every tests/golden/{mae,simmim}_*__refshim.npz exists and equals the restatement.
3. The noise, its ordering (ties included) and num_masked = int(ratio * n) in double.
4. The constructors' and calls' signatures and assert messages equal the reference's; a non-ViT encoder is refused.
5. The kind numbers and the vb_mim_config layout match the header, and vb_create refuses both kinds with a pointer to vb_create_mim."""
import ctypes as C
import inspect
import os
import re

import numpy as np
import pytest

import mim_oracle as o

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
REF_DIR = os.environ.get("VB_REFERENCE_DIR", "/root/reference/vit_tensorflow")    # the reference checkout (absent on the GPU box)
live = pytest.mark.skipif(not os.path.isdir(REF_DIR), reason="reference checkout not present (GPU box): fixtures cover it")
VARIANTS = ("init", "stress")
LIVE_CASES = ["mae_dense", "mae_identity", "mae_no_to_out", "mae_rect", "mae_small_image", "mae_ratio29", "mae_tie", "simmim_base",
              "simmim_odd", "simmim_rect", "simmim_small_image", "simmim_ratio29", "simmim_tie"]


def _spec(name, variant, **kw):
    kind, cfg = o.ALL_CASES[name]
    return o.forward(kind, o.weights(kind, cfg, variant), o.images(cfg, o.BATCH, size=o.call_size(cfg)), cfg, seed=o.case_seed(name), **kw)


def _masked_ids(name, spec):
    kind, _ = o.ALL_CASES[name]
    return spec["indices"] if kind == "mae" else spec["indices"][:, :spec["num_masked"]]


# ------------------------------------------------------------------------------------------ 1. the restatement vs the reference
@live
@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("name", LIVE_CASES)
def test_live_spec_equals_reference(name, variant):
    r = o.reference_run(REF_DIR, name, variant)
    s = _spec(name, variant)
    assert np.array_equal(r["indices"], _masked_ids(name, s))
    np.testing.assert_array_equal(r["masked_patches"], s["masked_patches"])
    np.testing.assert_allclose(r["pred"], s["pred"], rtol=0, atol=1e-11)
    assert r["loss"] == pytest.approx(s["loss"], rel=1e-12)


# ------------------------------------------------------------------------------------------ 2. the fixtures
@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("name", sorted(o.ALL_CASES))
def test_fixture_equals_spec(name, variant):
    z = np.load(os.path.join(GOLDEN, f"{name}__{variant}__refshim.npz"))
    s = _spec(name, variant)
    rows = int(z["rows"])
    assert int(z["noise_seed"]) == o.case_seed(name)
    assert np.array_equal(z["indices"], _masked_ids(name, s))
    np.testing.assert_array_equal(z["masked_patches"], s["masked_patches"][:, :rows].astype(np.float32))
    np.testing.assert_allclose(z["pred_ref"], s["pred"][:, :rows], rtol=1e-6, atol=1e-6)
    assert float(z["loss_ref_f64"]) == pytest.approx(s["loss"], rel=1e-10)
    assert float(z["loss_ref_f32"]) == pytest.approx(s["loss"], rel=1e-4)


def test_every_fixture_is_a_case():
    names = {f[:-len("__init__refshim.npz")] for f in os.listdir(GOLDEN) if re.match(r"(mae|simmim)_.*__init__refshim\.npz$", f)}
    assert names == set(o.ALL_CASES)


# ------------------------------------------------------------------------------------------ 3. noise, order, num_masked
def test_noise_is_the_ats_philox_with_the_mim_counter():
    from ats_oracle import philox4x32_10
    u = o.noise(3, 5, seed=0x1234567890ABCDEF, d=(7 << 32) | 9)
    x = philox4x32_10(np.array([[4, 2, 9, 7]], np.uint64), (0x90ABCDEF, 0x12345678))[0, 0]
    assert u[2, 4] == (int(x) >> 8) * 2.0 ** -24 and ((u >= 0) & (u < 1)).all()
    assert not np.array_equal(o.noise(3, 5, 1, 0), o.noise(3, 5, 1, 1))


def test_order_ties_go_to_the_smaller_id():
    u = np.array([[0.5, 0.25, 0.5, 0.75, 0.25]])
    assert o.permutation(u, simmim=False).tolist() == [[1, 4, 0, 2, 3]]
    assert o.permutation(u, simmim=True).tolist() == [[3, 0, 2, 1, 4]]


def test_tie_cases_hold_a_tie():
    for name, (kind, cfg) in o.TIE_CASES.items():
        H, W = cfg["image"]
        n = (H // cfg["patch"][0]) * (W // cfg["patch"][1])
        assert o.has_tie(o.noise(o.BATCH, n, o.case_seed(name), 0))


def test_num_masked_is_int_of_a_double():
    assert o.num_masked(0.29, 100) == 28 and o.num_masked(0.75, 196) == 147 and o.num_masked(0.5, 3) == 1


def test_bf16_storage_estimate_is_small_but_not_zero():
    s = _spec("mae_dense", "stress")
    b = _spec("mae_dense", "stress", bf16_storage=True)
    assert np.array_equal(s["indices"], b["indices"])
    d = np.abs(s["pred"] - b["pred"]).max()
    assert 0 < d < 0.1 * np.abs(s["pred"]).max()


# ------------------------------------------------------------------------------------------ 4. the host classes' surface
def _reference_classes():
    from oracle import tf_shim
    import importlib
    with tf_shim.installed(REF_DIR):
        import sys
        saved = sys.stdout
        try:
            sys.stdout = open(os.devnull, "w")                      # mae.py's import-time usage block prints its loss
            return importlib.import_module("mae").MAE, importlib.import_module("simmim").SimMIM
        finally:
            sys.stdout.close()
            sys.stdout = saved


@live
def test_live_signatures_equal_the_reference():
    import vit_tensorflow_b200 as vb
    ref_mae, ref_simmim = _reference_classes()
    for ref, ours in ((ref_mae, vb.MAE), (ref_simmim, vb.SimMIM)):
        pr = [(p.name, p.default) for p in inspect.signature(ref.__init__).parameters.values()]
        po = [(p.name, p.default) for p in inspect.signature(ours.__init__).parameters.values() if p.kind != p.KEYWORD_ONLY]
        assert po == pr
        cr = [(p.name, p.default, p.kind) for p in inspect.signature(ref.call).parameters.values()]
        co = [(p.name, p.default, p.kind) for p in inspect.signature(ours.__call__).parameters.values()]
        assert co == cr


@pytest.mark.parametrize("cls,args", [("MAE", dict(decoder_dim=32)), ("SimMIM", {})])
@pytest.mark.parametrize("ratio", [0.0, 1.0, -0.5, 1.5])
def test_masking_ratio_assert(cls, args, ratio):
    import vit_tensorflow_b200 as vb
    with pytest.raises(AssertionError, match="masking ratio must be kept between 0 and 1"):
        getattr(vb, cls)(image_size=32, encoder=None, masking_ratio=ratio, **args)


@pytest.mark.parametrize("cls,args", [("MAE", dict(decoder_dim=32)), ("SimMIM", {})])
def test_encoder_must_be_our_vit(cls, args):
    import vit_tensorflow_b200 as vb
    with pytest.raises(TypeError, match="the encoder must be a vit_tensorflow_b200.ViT"):
        getattr(vb, cls)(image_size=32, encoder=object(), **args)


def test_drop_in_modules():
    import vit_tensorflow
    import vit_tensorflow_b200 as vb
    from vit_tensorflow.mae import MAE
    from vit_tensorflow.simmim import SimMIM
    assert MAE is vb.MAE and SimMIM is vb.SimMIM and vit_tensorflow.MAE is vb.MAE
    assert "MAE" in vb.__all__ and "SimMIM" in vb.__all__


# ------------------------------------------------------------------------------------------ 5. the C-ABI
def test_kinds_and_config_layout_match_header():
    from vit_tensorflow_b200 import _lib
    src = open(os.path.join(ROOT, "include", "vitb200.h")).read()
    assert int(re.search(r"VB_KIND_MAE = (\d+)", src).group(1)) == _lib.KIND["mae"] == 19
    assert int(re.search(r"VB_KIND_SIMMIM = (\d+)", src).group(1)) == _lib.KIND["simmim"] == 20
    assert int(re.search(r"#define VB_MIM_MAX_PATCHES (\d+)", src).group(1)) == _lib.MIM_MAX_PATCHES >= 4096
    body = src[src.index("typedef struct vb_mim_config {"):src.index("} vb_mim_config;")]
    fields = []
    for line in body.splitlines():
        line = line.split("/*")[0].strip()
        for t in ("int32_t", "double"):
            if line.startswith(t + " "):
                fields += [(f.strip(), t) for f in line[len(t):].rstrip(";").split(",")]
    ctypes_of = {"int32_t": C.c_int32, "double": C.c_double}
    assert [(n, t) for n, t in _lib.VbMimConfig._fields_] == [(n, ctypes_of[t]) for n, t in fields]
    assert C.sizeof(_lib.VbMimConfig) == 32


@pytest.mark.parametrize("kind", ["mae", "simmim"])
def test_vb_create_refuses_the_kinds_and_names_vb_create_mim(lib, kind):
    from vit_tensorflow_b200 import _lib
    cfg = _lib.VbConfig()
    cfg.struct_size = C.sizeof(_lib.VbConfig)
    cfg.kind = _lib.KIND[kind]
    cfg.image_h = cfg.image_w = 32
    cfg.patch_h = cfg.patch_w = 8
    cfg.channels, cfg.num_classes, cfg.dim, cfg.depth, cfg.heads, cfg.dim_head, cfg.mlp_dim = 3, 10, 64, 1, 2, 32, 64
    h = C.c_void_p()
    assert lib.vb_create(C.byref(cfg), 0, C.byref(h)) != 0 and not h.value
    assert b"vb_create_mim" in lib.vb_last_error(None)
    mc = _lib.VbMimConfig()
    mc.struct_size = C.sizeof(_lib.VbMimConfig) + 8
    assert lib.vb_create_mim(C.byref(cfg), C.byref(mc), 0, C.byref(h)) != 0
    assert b"vb_mim_config.struct_size" in lib.vb_last_error(None)
    mc.struct_size = C.sizeof(_lib.VbMimConfig)
    mc.masking_ratio, mc.decoder_dim, mc.decoder_depth, mc.decoder_heads, mc.decoder_dim_head = 1.0, 32, 1, 2, 16
    assert lib.vb_create_mim(C.byref(cfg), C.byref(mc), 0, C.byref(h)) != 0
    assert b"masking ratio must be kept between 0 and 1" in lib.vb_last_error(None)
    cfg.kind = _lib.KIND["vit"]
    assert lib.vb_create_mim(C.byref(cfg), C.byref(mc), 0, C.byref(h)) != 0
    assert b"VB_KIND_MAE or VB_KIND_SIMMIM" in lib.vb_last_error(None)

"""MPP (reference mpp.py:133-218) on the CPU.

1. LIVE (skipped where the reference checkout is absent): the reference's own MPP over the numpy stand-in for TensorFlow, with
   `.numpy()` returning a copy as TF 2 does, draws exactly the restatement's mask ids, coins and random ids (tests/mpp_oracle.py);
   its logits and loss equal the restatement's with the corruption off.
2. FIXTURES (always): every tests/golden/mpp_*__refshim.npz exists and equals the restatement.
3. The draws: the mask's ceil in double, the top_k order with ties, the coins in float32.
4. The corrected cross-entropy, the constructor's and call's refusals, and the C-ABI surface (kinds, layout, vb_create)."""
import ctypes as C
import os
import re

import numpy as np
import pytest

import mpp_oracle as o

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
REF_DIR = os.environ.get("VB_REFERENCE_DIR", "/root/reference/vit_tensorflow")    # the reference checkout (absent on the GPU box)
live = pytest.mark.skipif(not os.path.isdir(REF_DIR), reason="reference checkout not present (GPU box): fixtures cover it")
VARIANTS = ("init", "stress")
# batch 1 is absent: the reference's line 197 then indexes the batch axis out of range and raises IndexError
LIVE_CASES = ["mpp_no_random", "mpp_coin_above_one", "mpp_ceil", "mpp_rect", "mpp_small_image", "mpp_bits1", "mpp_odd", "mpp_tie"]


@live
@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("name", LIVE_CASES)
def test_live_reference_draws_and_clean_forward_equal_the_restatement(name, variant):
    r = o.reference_run(REF_DIR, name, variant)
    s = o.spec(name, variant)
    assert np.array_equal(r["mask_ids"], s["mask_ids"])
    assert np.array_equal(r["replace_coin"], s["replace_coin"])
    assert np.array_equal(r["rand_coin"], s["rand_coin"])
    if o.ALL_CASES[name]["random_patch_prob"] > 0:
        assert np.array_equal(r["random_id"], s["random_id"])
    clean = o.spec(name, variant, corrupt=False)
    np.testing.assert_allclose(r["logits"], clean["logits"], rtol=0, atol=1e-12 * max(1.0, np.abs(clean["logits"]).max()))
    # mpp.py:128 casts the logits to float32 before the cross-entropy, so the reference's loss carries float32 rounding
    assert r["loss"] == pytest.approx(clean["loss"], rel=1e-6, abs=1e-6)


@live
def test_live_batch1_raises_index_error_in_the_reference():
    with pytest.raises(IndexError):
        o.reference_run(REF_DIR, "mpp_batch1", "init")


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("name", sorted(o.ALL_CASES))
def test_fixture_equals_spec(name, variant):
    z = np.load(os.path.join(GOLDEN, f"{name}__{variant}__refshim.npz"))
    s = o.spec(name, variant)
    assert int(z["noise_seed"]) == o.case_seed(name)
    assert np.array_equal(z["mask_ids"], s["mask_ids"]) and np.array_equal(z["source"], s["source"])
    np.testing.assert_array_equal(z["logits"], s["logits"].astype(np.float32))
    assert float(z["loss_f64"]) == pytest.approx(s["loss"], rel=1e-12)


def test_every_fixture_is_a_case():
    names = {f[:-len("__init__refshim.npz")] for f in os.listdir(GOLDEN) if re.match(r"mpp_.*__init__refshim\.npz$", f)}
    assert names == set(o.ALL_CASES)


def test_fixtures_cover_the_corners():
    c = o.ALL_CASES
    assert c["mpp_no_random"]["random_patch_prob"] == 0
    p = c["mpp_coin_above_one"]
    assert p["random_patch_prob"] / (1 - p["replace_prob"]) > 1
    assert o.num_masked(c["mpp_ceil"]["mask_prob"], 100) == 8
    assert {o.classes(c["mpp_bits1"]), o.classes(c["mpp_bits4"])} == {8, 4096}
    assert c["mpp_odd"]["dim"] % 64 and c["mpp_odd"]["dim_head"] != 64 and o.batch(c["mpp_batch1"]) == 1
    assert c["mpp_rect"]["image"][0] != c["mpp_rect"]["image"][1] and "call" in c["mpp_small_image"]
    s = o.spec("mpp_coin_above_one", "init")
    assert (s["source"] == -1).any() and ((s["source"] >= 0) & (s["source"] != np.arange(s["source"].shape[1]))).any()


def test_tie_case_holds_a_tie_at_the_top_k_boundary():
    cfg = o.ALL_CASES["mpp_tie"]
    n = (cfg["image"][0] // cfg["patch"]) * (cfg["image"][1] // cfg["patch"])
    k = o.num_masked(cfg["mask_prob"], n)
    u = np.sort(o.words(o.batch(cfg), n, o.case_seed("mpp_tie"))[..., 0] >> 8, -1)[:, ::-1]
    assert (u[:, k - 1] == u[:, k]).any()


def test_draws_use_words_one_to_three_and_ties_go_to_the_smaller_id():
    cfg = dict(mask_prob=0.5, replace_prob=0.5, random_patch_prob=0.25)
    d = o.draws(3, 10, cfg, seed=0x1234567890ABCDEF, d=(3 << 32) | 5)
    x = o.words(3, 10, 0x1234567890ABCDEF, (3 << 32) | 5)
    assert np.array_equal(d["random_id"], (x[..., 2].astype(np.uint64) * 10) >> 32)
    assert np.array_equal(d["replace_coin"], ((x[..., 3] >> 8).astype(np.float32) * np.float32(2 ** -24)) < np.float32(0.5))
    assert (np.diff(d["mask_ids"], axis=-1) > 0).all() and d["mask_ids"].shape == (3, 5)
    u = np.array([[0.5, 0.25, 0.5, 0.75, 0.25]])
    assert np.argsort(-u, -1, kind="stable")[:, :3].tolist() == [[3, 0, 2]]


def test_mask_count_is_ceil_of_a_double():
    assert o.num_masked(0.07, 100) == 8 and o.num_masked(0.15, 64) == 10 and o.num_masked(0.5, 4) == 2


def test_bf16_storage_estimate_is_small_but_not_zero():
    s = o.spec("mpp_bits1", "stress")
    b = o.spec("mpp_bits1", "stress", bf16_storage=True)
    d = np.abs(s["logits"] - b["logits"]).max()
    assert 0 < d < 0.1 * np.abs(s["logits"]).max()


def test_corrected_cross_entropy_equals_the_shims_on_equal_shapes():
    from oracle import tf_shim
    with tf_shim.installed() as tf:
        old = tf.nn.softmax_cross_entropy_with_logits
        rng = np.random.default_rng(3)
        a, b = rng.standard_normal((4, 6)), rng.standard_normal((4, 6))
        np.testing.assert_allclose(o._cross_entropy_broadcast(a, b), np.asarray(old(a, b)), rtol=0, atol=1e-14)
        lg = rng.standard_normal((4, 8))
        np.testing.assert_allclose(o._cross_entropy_broadcast(lg, rng.standard_normal((4, 1))), np.log(8) * lg.sum(-1), atol=1e-13)


# ------------------------------------------------------------------------------------------ the host class and the C-ABI
def test_drop_in_module():
    import vit_tensorflow_b200 as vb
    from vit_tensorflow.mpp import MPP
    assert MPP is vb.MPP and "MPP" in vb.__all__


@live
def test_live_signature_equals_the_reference():
    import inspect
    import importlib
    import sys
    import io
    from oracle import tf_shim
    import vit_tensorflow_b200 as vb
    with tf_shim.installed(REF_DIR):
        saved, sys.stdout = sys.stdout, io.StringIO()
        try:
            ref = importlib.import_module("mpp").MPP
        finally:
            sys.stdout = saved
    pr = [(p.name, p.default) for p in inspect.signature(ref.__init__).parameters.values()]
    po = [(p.name, p.default) for p in inspect.signature(vb.MPP.__init__).parameters.values() if p.kind != p.KEYWORD_ONLY]
    assert po == pr
    cr = [(p.name, p.default, p.kind) for p in inspect.signature(ref.call).parameters.values()]
    assert [(p.name, p.default, p.kind) for p in inspect.signature(vb.MPP.__call__).parameters.values()] == cr


@pytest.mark.parametrize("kw,match", [(dict(channels=1), "3 channels"), (dict(output_channel_bits=6), "2\\^18 classes")])
def test_constructor_refusals(kw, match):
    import vit_tensorflow_b200 as vb
    with pytest.raises(ValueError, match=match):
        vb.MPP(image_size=32, transformer=None, patch_size=8, **kw)


def test_kinds_and_config_layout_match_header():
    from vit_tensorflow_b200 import _lib
    src = open(os.path.join(ROOT, "include", "vitb200.h")).read()
    assert int(re.search(r"VB_KIND_MPP = (\d+)", src).group(1)) == _lib.KIND["mpp"] == 21
    body = src[src.index("typedef struct vb_mpp_config {"):src.index("} vb_mpp_config;")]
    fields = []
    for line in body.splitlines():
        line = line.split("/*")[0].strip()
        for t in ("int32_t", "double"):
            if line.startswith(t + " "):
                fields += [(f.strip(), t) for f in line[len(t):].rstrip(";").split(",")]
    assert "vb_mim_config mim;" in body
    ctypes_of = {"int32_t": C.c_int32, "double": C.c_double}
    own = _lib.VbMppConfig._fields_
    assert [(n, t) for n, t in own] == [(n, ctypes_of[t]) for n, t in fields]
    assert _lib.VbMppConfig.mask_prob.offset == C.sizeof(_lib.VbMimConfig) and C.sizeof(_lib.VbMppConfig) == 64
    assert "vb_forward_mpp" in _lib.SIGNATURES and "vb_op_mpp_draws" in _lib.SIGNATURES
    sig = re.search(r"VB_API int vb_forward_mpp\(([^;]*)\);", src).group(1)
    assert len(sig.split(",")) == len(_lib.SIGNATURES["vb_forward_mpp"][1]) == 12
    sig = re.search(r"VB_API int vb_op_mpp_draws\(([^;]*)\);", src).group(1)
    assert len(sig.split(",")) == len(_lib.SIGNATURES["vb_op_mpp_draws"][1]) == 9


def test_vb_create_refuses_mpp_and_names_vb_create_mim(lib):
    from vit_tensorflow_b200 import _lib
    cfg = _lib.VbConfig()
    cfg.struct_size = C.sizeof(_lib.VbConfig)
    cfg.kind = _lib.KIND["mpp"]
    cfg.image_h = cfg.image_w = 32
    cfg.patch_h = cfg.patch_w = 8
    cfg.channels, cfg.num_classes, cfg.dim, cfg.depth, cfg.heads, cfg.dim_head, cfg.mlp_dim = 3, 10, 64, 1, 2, 32, 64
    h = C.c_void_p()
    assert lib.vb_create(C.byref(cfg), 0, C.byref(h)) != 0 and not h.value
    assert b"vb_create_mim" in lib.vb_last_error(None)
    mc = _lib.VbMppConfig()
    mc.struct_size = C.sizeof(_lib.VbMimConfig)                     # a bare vb_mim_config is not an MPP config
    assert lib.vb_create_mim(C.byref(cfg), C.byref(mc), 0, C.byref(h)) != 0
    assert b"vb_mpp_config.struct_size" in lib.vb_last_error(None)
    mc.struct_size = C.sizeof(_lib.VbMppConfig)
    mc.mask_prob, mc.replace_prob, mc.random_patch_prob, mc.output_channel_bits = 0.15, 0.5, 0.5, 6
    assert lib.vb_create_mim(C.byref(cfg), C.byref(mc), 0, C.byref(h)) != 0
    assert b"output_channel_bits * channels" in lib.vb_last_error(None)

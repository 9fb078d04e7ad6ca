"""The small-dataset ViT on the CPU (reference vit_for_small_dataset.py):
1. the numpy SPT restatement against a known answer: the shift order, the zero edges and the (p1, p2, view, c) layout;
2. the float64 restatement against the committed fixtures of the reference's own module over the numpy shim
   (tests/golden/make_small_vit_golden.py), and one fixture against a live run where the reference checkout exists;
3. the constructor surface: parameter lists, defaults and assert messages of ViT and SPT as the reference's, a tuple patch_size
   refused at construction, SPT's missing `channels` parameter, and the kind number of the header."""
import inspect
import os
import re

import numpy as np
import pytest

import small_vit_oracle as o

REF_DIR = os.environ.get("VB_REFERENCE_DIR", "/root/reference/vit_tensorflow")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
HAVE_REF = os.path.exists(os.path.join(REF_DIR, "vit_for_small_dataset.py"))
live = pytest.mark.skipif(not HAVE_REF, reason="reference checkout not present: the fixtures cover it")


# ------------------------------------------------------------------------------------------ 1. SPT known answer
def test_spt_known_answer():
    """Pixel (y, x) channel c holds 100 y + 10 x + c, so every element names the pixel it came from."""
    H, W, p = 4, 6, 2
    yy, xx, cc = np.meshgrid(np.arange(H), np.arange(W), np.arange(3), indexing="ij")
    img = (100.0 * yy + 10.0 * xx + cc + 1)[None]                  # + 1: a real pixel is never 0
    got = o.spt_patches(img, p)
    assert got.shape == (1, (H // p) * (W // p), p * p * 15)
    for t in range(got.shape[1]):
        gy, gx = divmod(t, W // p)
        for p1 in range(p):
            for p2 in range(p):
                y, x = gy * p + p1, gx * p + p2
                # views: the image, out[:, :, w] = x[:, :, w - 1], x[:, :, w + 1], out[:, h] = x[:, h - 1], x[:, h + 1]
                for view, (sy, sx) in enumerate([(y, x), (y, x - 1), (y, x + 1), (y - 1, x), (y + 1, x)]):
                    for c in range(3):
                        want = 100.0 * sy + 10.0 * sx + c + 1 if 0 <= sy < H and 0 <= sx < W else 0.0
                        assert got[0, t, ((p1 * p + p2) * 5 + view) * 3 + c] == want, (t, p1, p2, view, c)


# ------------------------------------------------------------------------------------------ 2. the restatement vs the reference
@pytest.mark.parametrize("kind", o.WEIGHTS)
@pytest.mark.parametrize("name", sorted(o.SMALL))
def test_spec_matches_reference_fixture(name, kind):
    cfg = o.SMALL[name]
    z = np.load(os.path.join(GOLDEN, f"small_vit_{name}__{kind}__refshim.npz"))
    r = o.forward(o.weights(cfg, kind), o.images(cfg, o.BATCH), cfg)
    np.testing.assert_allclose(r, z["logits_ref_f64"], rtol=0, atol=1e-5)
    np.testing.assert_allclose(r, z["logits_ref_f32"], rtol=0, atol=1e-4 * max(1.0, np.abs(r).max()))


@live
def test_live_reference_matches_fixture():
    name = "rect_p8_dh32_mean"
    got = o.reference_run(REF_DIR, {name: o.SMALL[name]})
    for kind in o.WEIGHTS:
        z = np.load(os.path.join(GOLDEN, f"small_vit_{name}__{kind}__refshim.npz"))
        np.testing.assert_allclose(got[name, kind], z["logits_ref_f64"], rtol=0, atol=1e-10)


# ------------------------------------------------------------------------------------------ 3. constructor surface
VIT_CTOR = [("image_size", None), ("patch_size", None), ("num_classes", None), ("dim", None), ("depth", None), ("heads", None),
            ("mlp_dim", None), ("pool", "cls"), ("dim_head", 64), ("dropout", 0.0), ("emb_dropout", 0.0)]


def _params(fn):
    return [(p.name, None if p.default is inspect.Parameter.empty else p.default) for p in inspect.signature(fn).parameters.values()
            if p.kind is not inspect.Parameter.KEYWORD_ONLY and p.name != "self"]


def test_signatures():
    from vit_tensorflow_b200 import SmallDatasetViT, SPT
    assert _params(SmallDatasetViT.__init__) == VIT_CTOR
    assert _params(SPT.__init__) == [("dim", None), ("patch_size", None)]
    kw = [p.name for p in inspect.signature(SmallDatasetViT.__init__).parameters.values() if p.kind is inspect.Parameter.KEYWORD_ONLY]
    assert kw == ["precision", "device", "seed"]
    from vit_tensorflow.vit_for_small_dataset import ViT as ShimViT, SPT as ShimSPT
    assert ShimViT is SmallDatasetViT and ShimSPT is SPT


@live
def test_signatures_match_live_reference():
    from vit_tensorflow_b200 import SmallDatasetViT, SPT
    with o.installed(REF_DIR):
        import vit_for_small_dataset as ref
        assert _params(ref.ViT.__init__) == _params(SmallDatasetViT.__init__)
        assert _params(ref.SPT.__init__) == _params(SPT.__init__)


ARGS = dict(image_size=32, patch_size=8, num_classes=10, dim=64, depth=1, heads=2, mlp_dim=64)
ASSERTS = [(dict(image_size=30), "Image dimensions must be divisible by the patch size."),
           (dict(image_size=(32, 36)), "Image dimensions must be divisible by the patch size."),
           (dict(pool="max"), "pool type must be either cls (cls token) or mean (mean pooling)")]


@pytest.mark.parametrize("kw,msg", ASSERTS)
def test_constructor_asserts(kw, msg):
    from vit_tensorflow_b200 import SmallDatasetViT
    with pytest.raises(AssertionError, match=re.escape(msg)):
        SmallDatasetViT(**dict(ARGS, **kw))


@live
@pytest.mark.parametrize("kw,msg", ASSERTS)
def test_constructor_asserts_match_live_reference(kw, msg):
    with o.installed(REF_DIR):
        import vit_for_small_dataset as ref
        with pytest.raises(AssertionError, match=re.escape(msg)):
            ref.ViT(**dict(ARGS, **kw))


def test_tuple_patch_size_refused():
    from vit_tensorflow_b200 import SmallDatasetViT, SPT
    with pytest.raises(ValueError, match="one integer patch_size"):
        SmallDatasetViT(**dict(ARGS, patch_size=(8, 8)))
    with pytest.raises(ValueError, match="one integer patch_size"):
        SPT(dim=64, patch_size=(8, 8))


def test_spt_takes_no_channels():
    """The README's `SPT(dim=1024, patch_size=16, channels=3)` raises TypeError in the reference (SPT.__init__(self, dim,
    patch_size)); so it does here."""
    from vit_tensorflow_b200 import SPT
    with pytest.raises(TypeError):
        SPT(dim=1024, patch_size=16, channels=3)
    s = SPT(dim=32, patch_size=4, seed=0)
    assert {k: v.shape for k, v in s.get_weights_dict().items()} == {
        "patch_norm.gamma": (240,), "patch_norm.beta": (240,), "patch.kernel": (240, 32), "patch.bias": (32,)}


def test_header_kind():
    from vit_tensorflow_b200 import _lib
    src = open(os.path.join(ROOT, "include", "vitb200.h")).read()
    assert int(re.search(r"VB_KIND_SMALL_DATASET_VIT = (\d+)", src).group(1)) == _lib.KIND["small_dataset_vit"] == 15

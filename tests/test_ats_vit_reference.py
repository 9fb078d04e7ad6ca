"""ATS-ViT on the CPU: the float64 restatement's Philox against Random123's known-answer vectors, its sampling rules, and the
Python constructor's reference asserts (ats_vit.py:225-227, 279)."""
import os

import numpy as np
import pytest

import ats_oracle as o


def _hex(a):
    return " ".join(f"{int(v):08x}" for v in a)


@pytest.mark.parametrize("ctr,key,want", [
    ((0, 0, 0, 0), (0, 0), "6627e8d5 e169c58d bc57ac4c 9b00dbd8"),
    ((0xffffffff,) * 4, (0xffffffff, 0xffffffff), "408f276d 41c83b0e a20bc7c6 6d5451fd"),
    ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0), "d16cfe09 94fdcceb 5001e420 24126ea1"),
])
def test_philox_known_answers(ctr, key, want):
    assert _hex(o.philox4x32_10(np.array([ctr], np.uint64), key)[0]) == want


CFG = dict(image=(16, 24), patch=(4, 4), dim=32, heads=2, dim_head=16, mlp_dim=48, max_tokens_per_depth=(30, 12, 12, 5))


def test_spec_sampling_rules():
    rng = np.random.default_rng(0)
    w = o.small_weights(CFG, rng)
    img = rng.standard_normal((3, 16, 24, 3))
    r = o.forward(w, img, CFG, seed=7)
    # 24 patches <= 30: layer 0 keeps all; layer 1 samples; layer 2 only if layer 1 left more than 12; layer 3 samples
    assert r["sampled"][0] == 1 and r["sampled"][-1] == 3 and 0 not in r["sampled"]
    assert r["d"] == len(r["sampled"])
    ids = r["token_ids"]
    for row in ids:
        kept = row[row >= 0]
        assert np.all(np.diff(kept) > 0) and np.all(row[:len(row) - len(kept)] == -1)   # ascending, left-padded with -1
    assert ids.shape[1] <= 5 and np.isfinite(r["logits"]).all()
    # the same seed and counter repeat the draws; another counter draws others
    again = o.forward(w, img, CFG, seed=7)
    assert np.array_equal(again["token_ids"], ids) and np.array_equal(again["logits"], r["logits"])
    other = o.forward(w, img, CFG, seed=7, d=r["d"])
    assert not np.array_equal(other["token_ids"], ids)
    # forcing the spec's own draws changes nothing
    forced = o.forward(w, img, CFG, seed=7, forced=r["draws"])
    assert np.array_equal(forced["logits"], r["logits"])


def test_spec_no_sampling_is_vit():
    cfg = dict(CFG, max_tokens_per_depth=(100, 100, 50, 30))
    rng = np.random.default_rng(1)
    w = o.small_weights(cfg, rng)
    r = o.forward(w, rng.standard_normal((2, 16, 24, 3)), cfg)
    assert r["sampled"] == [] and r["token_ids"].shape == (2, 24)
    assert np.array_equal(r["token_ids"], np.broadcast_to(np.arange(24), (2, 24)))


@pytest.mark.parametrize("kw,msg", [
    (dict(depth=3, max_tokens_per_depth=(8, 4)), "max_tokens_per_depth must be a tuple of length that is equal to the depth of the transformer"),
    (dict(depth=2, max_tokens_per_depth=(4, 8)), "max_tokens_per_depth must be in decreasing order"),
    (dict(depth=2, max_tokens_per_depth=(4, 0)), "max_tokens_per_depth must have at least 1 token at any layer"),
    (dict(image_size=30, depth=2, max_tokens_per_depth=(4, 2)), "Image dimensions must be divisible by the patch size."),
])
def test_constructor_asserts(kw, msg):
    from vit_tensorflow_b200 import ATSViT
    args = dict(image_size=32, patch_size=8, num_classes=10, dim=64, heads=2, mlp_dim=64)
    args.update(kw)
    with pytest.raises(AssertionError, match=msg.replace(".", r"\.")):
        ATSViT(**args)


@pytest.mark.parametrize("name", sorted(o.SMALL))
def test_spec_matches_reference_fixture(name):
    """The float64 restatement against the reference's own ats_vit.py over the shim with the same noise
    (tests/golden/make_ats_golden.py): identical returned ids, logits within 1e-5 (float64 fixture) and the float32 fixture's ids."""
    cfg = o.SMALL[name]
    z = np.load(os.path.join(os.path.dirname(__file__), "golden", f"ats_{name}__refshim.npz"))
    r = o.forward(o.weights(cfg), o.images(cfg, o.BATCH), cfg, seed=o.SEED)
    assert np.array_equal(r["token_ids"], z["token_ids_f64"]) and np.array_equal(r["token_ids"], z["token_ids_f32"])
    np.testing.assert_allclose(r["logits"], z["logits_ref_f64"], rtol=0, atol=1e-5)
    np.testing.assert_allclose(r["logits"], z["logits_ref_f32"], rtol=0, atol=1e-4 * max(1.0, np.abs(r["logits"]).max()))
    assert [tuple(s) for s in z["noise_shapes"]] == [(o.BATCH, cfg["max_tokens_per_depth"][L], r["pert"][L].shape[2]) for L in r["sampled"]]
    assert float(z["margin"]) == pytest.approx(r["margin"]) and r["margin"] >= 1e-3

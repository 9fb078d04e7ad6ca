"""MPP on the H100 (mpp.py): the fp32 engine against every fixture of the float64 restatement (mask ids and source exact, logits
and loss to rtol 1e-3 / atol 1e-4), the bf16 engine within 4x the bf16-storage estimate, eager / captured / replayed calls bit for
bit, fresh draws per call that set_seed repeats, the encoder's weights (cls_token included) picked up after a change, the draw
kernels against numpy, and the refusals."""
import os

import numpy as np
import pytest

import mpp_oracle as o

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
VARIANTS = ("init", "stress")
FP32_RTOL, FP32_ATOL = 1e-3, 1e-4
BF16_FACTOR = 4.0


def build(name, precision, variant="init"):
    import vit_tensorflow_b200 as vb
    cfg = o.ALL_CASES[name]
    enc = vb.ViT(image_size=cfg["image"], patch_size=cfg["patch"], num_classes=5, dim=cfg["dim"], depth=cfg["depth"], heads=cfg["heads"],
                 mlp_dim=cfg["mlp_dim"], dim_head=cfg["dim_head"], precision=precision)
    w = o.weights(cfg, variant)
    enc.set_weights_dict({k: v for k, v in w.items() if k in enc.weight_specs()})
    m = vb.MPP(image_size=cfg["image"][0], transformer=enc, patch_size=cfg["patch"], output_channel_bits=cfg.get("bits", 3),
               mask_prob=cfg["mask_prob"], replace_prob=cfg["replace_prob"], random_patch_prob=cfg["random_patch_prob"])
    m.set_weights_dict({k: v for k, v in w.items() if k not in enc.weight_specs()})
    m.set_seed(o.case_seed(name))
    return m, enc, w


def _img(name):
    cfg = o.ALL_CASES[name]
    return o.images(cfg, o.batch(cfg), size=o.call_size(cfg))


def _loss_tol(spec, est=None):
    # the loss is ln(K) times a mean of row sums of K logits: each logit's error enters K times, scaled by ln(K)
    K = spec["logits"].shape[-1]
    if est is None:
        return FP32_RTOL * abs(spec["loss"]) + np.log(K) * K * FP32_ATOL
    return BF16_FACTOR * np.log(K) * np.abs(est["logits"] - spec["logits"]).sum(-1).mean()


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("name", sorted(o.ALL_CASES))
def test_fp32_matches_fixture_and_spec(name, variant):
    cfg = o.ALL_CASES[name]
    m, _, w = build(name, "fp32", variant)
    img = _img(name)
    z = np.load(os.path.join(GOLDEN, f"{name}__{variant}__refshim.npz"))
    spec = o.forward(w, img, cfg, seed=o.case_seed(name))
    loss, logits, ids, src = m.forward_mpp(img)
    assert np.array_equal(ids, z["mask_ids"]) and np.array_equal(src, z["source"])
    assert np.array_equal(ids, spec["mask_ids"]) and np.array_equal(src, spec["source"])
    np.testing.assert_allclose(logits, spec["logits"], rtol=FP32_RTOL, atol=FP32_ATOL)
    np.testing.assert_allclose(logits, z["logits"], rtol=FP32_RTOL, atol=FP32_ATOL)
    assert abs(float(loss) - float(z["loss_f64"])) <= _loss_tol(spec)
    nxt = o.forward(w, img, cfg, seed=o.case_seed(name), d=1)           # the call after it draws d = 1
    assert abs(float(m(img, training=False)) - nxt["loss"]) <= _loss_tol(nxt)


@pytest.mark.parametrize("name", sorted(o.ALL_CASES))
def test_bf16_within_the_bf16_storage_estimate(name):
    cfg = o.ALL_CASES[name]
    m, _, w = build(name, "bf16", "stress")
    img = _img(name)
    spec = o.forward(w, img, cfg, seed=o.case_seed(name))
    est = o.forward(w, img, cfg, seed=o.case_seed(name), bf16_storage=True)
    loss, logits, ids, src = m.forward_mpp(img)
    assert np.array_equal(ids, spec["mask_ids"]) and np.array_equal(src, spec["source"])
    tol = BF16_FACTOR * np.abs(est["logits"] - spec["logits"]).max()
    assert np.abs(logits - spec["logits"]).max() <= tol, (np.abs(logits - spec["logits"]).max(), tol)
    assert abs(float(loss) - spec["loss"]) <= _loss_tol(spec, est), (float(loss), spec["loss"])


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_eager_capture_replay_bit_identical_and_fresh_draws(precision):
    import torch
    name = "mpp_coin_above_one"
    cfg = o.ALL_CASES[name]
    m, _, w = build(name, precision)
    img = _img(name)
    stream = torch.cuda.Stream()
    outs = []
    for _ in range(3):                                                 # eager, captured, replayed
        m.set_seed(o.case_seed(name))
        outs.append(m.forward_mpp(img, stream=stream.cuda_stream))
    gs = m.graph_stats()
    assert gs["captures"] == 1 and gs["replays"] >= 1 and gs["failures"] == 0
    for o2 in outs[1:]:
        for a, b in zip(outs[0], o2):
            assert np.asarray(a).tobytes() == np.asarray(b).tobytes()
    m.set_seed(o.case_seed(name))
    n = outs[0][3].shape[1]
    seen = []
    for d in range(3):
        _, _, ids, src = m.forward_mpp(img, stream=stream.cuda_stream)
        dr = o.draws(o.batch(cfg), n, cfg, o.case_seed(name), d)
        assert np.array_equal(ids, dr["mask_ids"]) and np.array_equal(src, dr["source"])
        seen.append(src.tobytes())
    assert len(set(seen)) == 3


@pytest.mark.parametrize("n", [1, 2, 63, 64, 65, 196, 1024, 4096])
def test_draw_kernels_against_numpy(n):
    from vit_tensorflow_b200 import _lib
    for (rep, rp), (seed, counter) in zip([(0.5, 0.3), (0.8, 0.3), (0.5, 0.0)], [(0, 0), (0x0123456789ABCDEF, (5 << 32) | 3), (7, 1)]):
        cfg = dict(mask_prob=0.15, replace_prob=rep, random_patch_prob=rp)
        dr = o.draws(3, n, cfg, seed, counter)
        ids, src = _lib.op_mpp_draws(3, n, o.num_masked(0.15, n), rep, rp, seed, counter)
        assert np.array_equal(ids, dr["mask_ids"]) and np.array_equal(src, dr["source"])


def test_encoder_weight_changes_show_in_the_next_call():
    name = "mpp_rect"
    cfg = o.ALL_CASES[name]
    m, enc, w = build(name, "fp32")
    img = _img(name)
    first = float(m.forward_mpp(img)[0])
    for key, delta in (("layers.0.fc2.bias", 0.5), ("cls_token", 1.0)):
        w = dict(w)
        w[key] = w[key] + delta
        enc.set_weights_dict({key: w[key]})
        m.set_seed(o.case_seed(name))
        second = float(m.forward_mpp(img)[0])
        assert second != first
        spec = o.forward(w, img, cfg, seed=o.case_seed(name))
        assert abs(second - spec["loss"]) <= _loss_tol(spec)
        first = second


def test_call_returns_the_loss_and_refusals():
    import vit_tensorflow_b200 as vb
    from vit_tensorflow_b200 import _lib
    m, enc, w = build("mpp_bits1", "fp32")
    cfg = o.ALL_CASES["mpp_bits1"]
    img = _img("mpp_bits1")
    loss = m(img)
    assert loss.shape == () and loss.dtype == np.float32
    spec = o.forward(w, img, cfg, seed=o.case_seed("mpp_bits1"))
    assert abs(float(loss) - spec["loss"]) <= _loss_tol(spec)
    with pytest.raises(ValueError, match="divisible by the patch size"):
        m(np.zeros((1, 30, 32, 3), np.float32))
    with pytest.raises(_lib.VbError, match="pos_embedding has rows for 16"):
        m(np.zeros((1, 40, 32, 3), np.float32))
    with pytest.raises(_lib.VbError, match="vb_forward_mpp"):
        _lib.check(m._lib.vb_forward(m._h, img.ctypes.data, 0, 2, 32, 32, np.zeros(10, np.float32).ctypes.data, 0, None), m._h)
    with pytest.raises(_lib.VbError, match="vb_forward_mpp"):
        _lib.check(m._lib.vb_forward_mim(m._h, img.ctypes.data, 0, 2, 32, 32, np.zeros(1, np.float32).ctypes.data, None, None, None,
                                         0, None), m._h)
    small = vb.MPP(image_size=32, transformer=enc, patch_size=8, mask_prob=0.0)
    with pytest.raises(_lib.VbError, match="mean over no patches"):
        small(img, training=False)
    big = vb.MPP(image_size=32, transformer=enc, patch_size=8, mask_prob=1.5)
    with pytest.raises(_lib.VbError, match="more patches than the image has"):
        big(img, training=False)
    zero = vb.MPP(image_size=32, transformer=enc, patch_size=8, replace_prob=1.0, random_patch_prob=0.5)
    with pytest.raises(ZeroDivisionError):
        zero(img, training=False)
    ms = vb.MPP(image_size=32, transformer=enc, patch_size=8, mean=[0.5, 0.5, 0.5], std=[0.2, 0.2, 0.2])
    with pytest.raises(ValueError, match="broadcast"):
        ms(img, training=False)
    assert np.isfinite(float(vb.MPP(image_size=32, transformer=enc, patch_size=8, mean=[0.5], std=[0.2])(img, training=False)))
    with pytest.raises(ValueError, match="patch_size"):
        vb.MPP(image_size=32, transformer=enc, patch_size=4)


def test_training_with_encoder_dropout_is_refused():
    import vit_tensorflow_b200 as vb
    enc = vb.ViT(image_size=32, patch_size=8, num_classes=5, dim=64, depth=1, heads=2, mlp_dim=64, dim_head=32, dropout=0.1,
                 emb_dropout=0.1, precision="fp32")
    m = vb.MPP(image_size=32, transformer=enc, patch_size=8)
    img = np.zeros((1, 32, 32, 3), np.float32)
    with pytest.raises(NotImplementedError):
        m(img)
    assert np.isfinite(float(m(img, training=False)))

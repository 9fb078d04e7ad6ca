"""MAE and SimMIM on the H100 (mae.py, simmim.py): the fp32 engine against the fixtures of the reference's own classes and the
float64 restatement (same noise: identical masks), the bf16 engine within a tolerance derived from the bf16-storage restatement,
eager / captured / replayed calls bit for bit, the noise counter across calls, the mask kernel on its own, the encoder's weights
picked up after a change, and the refusals."""
import os

import numpy as np
import pytest

import mim_oracle as o

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
VARIANTS = ("init", "stress")
# fp32: the SIMT GEMMs and attention in float32 against float64 (the fp32 gates elsewhere use rtol 1e-3 / atol 1e-4)
FP32_RTOL, FP32_ATOL = 1e-3, 1e-4
# bf16: the restatement with bf16 storage rounds only what the engine stores; the engine also accumulates in another order and
# folds the LayerNorms into the GEMMs, so its error is taken to be at most this many times the restatement's own
BF16_FACTOR = 4.0


def build(name, precision, variant="init"):
    import vit_tensorflow_b200 as vb
    kind, cfg = o.ALL_CASES[name]
    enc = vb.ViT(image_size=cfg["image"], patch_size=cfg["patch"], num_classes=5, dim=cfg["dim"], depth=cfg["depth"], heads=cfg["heads"],
                 mlp_dim=cfg["mlp_dim"], dim_head=cfg["dim_head"], precision=precision)
    w = o.weights(kind, cfg, variant)
    enc.set_weights_dict(o.encoder_weights(w, cfg))
    H = cfg["image"][0]
    if kind == "mae":
        m = vb.MAE(image_size=H, encoder=enc, decoder_dim=cfg["decoder_dim"], masking_ratio=cfg["ratio"], decoder_depth=cfg["decoder_depth"],
                   decoder_heads=cfg["decoder_heads"], decoder_dim_head=cfg["decoder_dim_head"])
    else:
        m = vb.SimMIM(image_size=H, encoder=enc, masking_ratio=cfg["ratio"])
    m.set_weights_dict({k: v for k, v in w.items() if k not in enc.weight_specs()})
    m.set_seed(o.case_seed(name))
    return m, enc, w


def _img(name):
    _, cfg = o.ALL_CASES[name]
    return o.images(cfg, o.BATCH, size=o.call_size(cfg))


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("name", sorted(o.ALL_CASES))
def test_fp32_matches_fixture_and_spec(name, variant):
    kind, cfg = o.ALL_CASES[name]
    m, _, w = build(name, "fp32", variant)
    img = _img(name)
    z = np.load(os.path.join(GOLDEN, f"{name}__{variant}__refshim.npz"))
    spec = o.forward(kind, w, img, cfg, seed=o.case_seed(name))
    loss, pred, patches, idx = m.forward_mim(img)
    nm, rows = spec["num_masked"], int(z["rows"])
    assert np.array_equal(idx, spec["indices"])
    assert np.array_equal(idx if kind == "mae" else idx[:, :nm], z["indices"])
    np.testing.assert_array_equal(patches, spec["masked_patches"].astype(np.float32))
    np.testing.assert_array_equal(patches[:, :rows], z["masked_patches"])
    np.testing.assert_allclose(pred, spec["pred"], rtol=FP32_RTOL, atol=FP32_ATOL)
    np.testing.assert_allclose(pred[:, :rows], z["pred_ref"], rtol=FP32_RTOL, atol=FP32_ATOL)
    assert float(loss) == pytest.approx(spec["loss"], rel=FP32_RTOL, abs=FP32_ATOL)
    assert float(loss) == pytest.approx(float(z["loss_ref_f64"]), rel=FP32_RTOL, abs=FP32_ATOL)
    # the call after it draws the masks of d = 1
    assert float(m(img, training=False)) == pytest.approx(o.forward(kind, w, img, cfg, seed=o.case_seed(name), d=1)["loss"],
                                                          rel=FP32_RTOL, abs=FP32_ATOL)


@pytest.mark.parametrize("name", sorted(o.ALL_CASES))
def test_bf16_within_the_bf16_storage_estimate(name):
    kind, cfg = o.ALL_CASES[name]
    m, _, w = build(name, "bf16", "stress")
    img = _img(name)
    spec = o.forward(kind, w, img, cfg, seed=o.case_seed(name))
    est = o.forward(kind, w, img, cfg, seed=o.case_seed(name), bf16_storage=True)
    loss, pred, patches, idx = m.forward_mim(img)
    assert np.array_equal(idx, spec["indices"])                        # the masks do not depend on the precision
    np.testing.assert_array_equal(patches, spec["masked_patches"].astype(np.float32))
    tol = BF16_FACTOR * np.abs(est["pred"] - spec["pred"]).max()
    assert np.abs(pred - spec["pred"]).max() <= tol, (np.abs(pred - spec["pred"]).max(), tol)
    # |loss - loss64| is bounded by the mean of the per-element differences of the loss's terms
    if kind == "mae":
        ltol = BF16_FACTOR * np.mean(np.abs(est["pred"] ** 2 - spec["pred"] ** 2))
    else:
        ltol = BF16_FACTOR * np.mean(np.abs(est["pred"] - spec["pred"])) / spec["num_masked"]
    assert abs(float(loss) - spec["loss"]) <= ltol, (float(loss), spec["loss"], ltol)


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("name", ["mae_dense", "simmim_base"])
def test_eager_capture_replay_bit_identical_and_fresh_masks(name, precision):
    import torch
    kind, cfg = o.ALL_CASES[name]
    m, _, w = build(name, precision)
    img = _img(name)
    stream = torch.cuda.Stream()
    outs = []
    for _ in range(3):                                                 # eager, captured, replayed
        m.set_seed(o.case_seed(name))
        outs.append(m.forward_mim(img, stream=stream.cuda_stream))
    gs = m.graph_stats()
    assert gs["captures"] == 1 and gs["replays"] >= 1 and gs["failures"] == 0
    for o2 in outs[1:]:
        for a, b in zip(outs[0], o2):
            assert np.asarray(a).tobytes() == np.asarray(b).tobytes()
    # without a reset, consecutive calls draw the masks of d = 0, 1, 2 (eager, then the replayed graph advances d on the device)
    m.set_seed(o.case_seed(name))
    n = outs[0][3].shape[1]
    for d in range(3):
        _, _, _, idx = m.forward_mim(img, stream=stream.cuda_stream)
        assert np.array_equal(idx, o.mask_indices(kind, o.BATCH, n, o.case_seed(name), d))
    assert not np.array_equal(o.mask_indices(kind, o.BATCH, n, o.case_seed(name), 0), o.mask_indices(kind, o.BATCH, n, o.case_seed(name), 1))


@pytest.mark.parametrize("n", [1, 2, 63, 64, 65, 196, 1024, 4096])
@pytest.mark.parametrize("descending", [False, True])
def test_mask_kernel_against_numpy(n, descending):
    from vit_tensorflow_b200 import _lib
    for seed, counter in ((0, 0), (0x0123456789ABCDEF, (5 << 32) | 3)):
        got = _lib.op_mim_mask(3, n, seed, counter, descending)
        assert np.array_equal(got, o.permutation(o.noise(3, n, seed, counter), descending))


def test_mask_kernel_refuses_past_its_limit():
    from vit_tensorflow_b200 import _lib
    with pytest.raises(_lib.VbError, match="4096"):
        _lib.op_mim_mask(1, _lib.MIM_MAX_PATCHES + 1)


def test_encoder_weight_change_shows_in_the_next_call():
    m, enc, w = build("simmim_base", "fp32")
    kind, cfg = o.ALL_CASES["simmim_base"]
    img = _img("simmim_base")
    first = float(m.forward_mim(img)[0])
    w2 = dict(w)
    w2["layers.0.fc2.bias"] = w["layers.0.fc2.bias"] + 0.5
    enc.set_weights_dict({"layers.0.fc2.bias": w2["layers.0.fc2.bias"]})
    m.set_seed(o.case_seed("simmim_base"))
    second = float(m.forward_mim(img)[0])
    assert second != first
    assert second == pytest.approx(o.forward(kind, w2, img, cfg, seed=o.case_seed("simmim_base"))["loss"], rel=FP32_RTOL)


def test_call_returns_the_loss_and_refusals():
    from vit_tensorflow_b200 import _lib
    m, enc, w = build("mae_dense", "fp32")
    kind, cfg = o.ALL_CASES["mae_dense"]
    img = _img("mae_dense")
    loss = m(img)
    assert loss.shape == () and loss.dtype == np.float32 and type(loss.numpy()) is np.ndarray
    assert float(loss) == pytest.approx(o.forward(kind, w, img, cfg, seed=o.case_seed("mae_dense"))["loss"], rel=FP32_RTOL)
    with pytest.raises(ValueError, match="divisible by the patch size"):
        m(np.zeros((1, 30, 32, 3), np.float32))
    with pytest.raises(_lib.VbError, match="pos_embedding has rows for 16"):
        m(np.zeros((1, 40, 32, 3), np.float32))
    with pytest.raises(_lib.VbError, match="num_masked"):
        m(np.zeros((1, 8, 8, 3), np.float32))                       # int(0.75 * 1) == 0
    with pytest.raises(_lib.VbError, match="vb_forward_mim"):
        _lib.check(m._lib.vb_forward(m._h, img.ctypes.data, 0, 2, 32, 32, np.zeros(10, np.float32).ctypes.data, 0, None), m._h)


def test_training_with_encoder_dropout_is_refused():
    import vit_tensorflow_b200 as vb
    enc = vb.ViT(image_size=32, patch_size=8, num_classes=5, dim=64, depth=1, heads=2, mlp_dim=64, dim_head=32, dropout=0.1,
                 precision="fp32")
    m = vb.SimMIM(image_size=32, encoder=enc)
    img = np.zeros((1, 32, 32, 3), np.float32)
    with pytest.raises(NotImplementedError):
        m(img)
    assert np.isfinite(float(m(img, training=False)))

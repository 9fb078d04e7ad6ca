"""GPU: training-mode dropout (include/vitb200.h, vb_set_dropout / vb_forward_train) of ViT, DeepViT, CaiT and CrossViT against
the reference's own classes run over the numpy stand-in with the same Philox masks (tests/golden/dropout_*__refshim.npz), the stream
kernel against its numpy restatement bit for bit, and the call rules: reseeding, graph replays, the inference forward untouched."""
import os

import numpy as np
import pytest

import dropout_oracle as o

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
BF16_RTOL, BF16_ATOL = 4e-2, 6e-2          # tests/test_gpu_models.py's bf16 tolerance against the same oracle


def _model(name, precision, gen="stress", **over):
    import vit_tensorflow_b200 as vb
    kw = dict(o.CASES[name][0])
    kind = kw.pop("kind")
    kw.update(over)
    m = {"vit": vb.ViT, "deepvit": vb.DeepViT, "cait": vb.CaiT, "crossvit": vb.CrossViT}[kind](**kw, precision=precision)
    m.set_weights_dict(o.weights(name, gen))
    return m


def _close(got, ref, precision):
    if precision == "fp32":
        np.testing.assert_allclose(got, ref, rtol=1e-3, atol=1e-4)
    else:
        err = np.abs(got - ref)
        assert np.isfinite(got).all() and (err <= BF16_ATOL + BF16_RTOL * np.abs(ref)).all(), f"max err {err.max():.4f}"


@pytest.mark.parametrize("shape", [(1, 1), (7, 5), (129, 3072), (4097, 770)])
@pytest.mark.parametrize("draw", [0, 1, 2 ** 32 - 1])
def test_op_dropout_mask_matches_numpy_stream(lib, shape, draw):
    from vit_tensorflow_b200 import _lib
    M, N = shape
    for site, rate in ((0, 0.1), (37, 0.5)):
        got = _lib.op_dropout_mask(o.SEED, draw, site, M, N, rate)
        np.testing.assert_array_equal(got.astype(bool), o.keep_mask(o.SEED, draw, site, M, N, rate))


@pytest.mark.parametrize("name", sorted(o.CASES))
@pytest.mark.parametrize("gen", o.WEIGHTS)
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_family_matches_reference_fixture(lib, name, gen, precision):
    z = np.load(os.path.join(GOLDEN, o.fixture_name(name, gen)))
    m = _model(name, precision, gen)
    img = o.images(name)
    m.set_dropout_seed(int(z["seed"]))
    for d in (0, 1):
        got = np.asarray(m(img))                     # training=True, the reference's default
        _close(got, z[f"logits_d{d}_f64"], precision)


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_reseeding_repeats_the_sequence(lib, precision):
    m = _model("vit_cls", precision)
    img = o.images("vit_cls")
    m.set_dropout_seed(7)
    first = [np.asarray(m(img, training=True)) for _ in range(3)]
    assert not np.array_equal(first[0], first[1]) and not np.array_equal(first[1], first[2])
    m.set_dropout_seed(7)
    again = [np.asarray(m(img)) for _ in range(3)]
    for a, b in zip(first, again):
        np.testing.assert_array_equal(a, b)
    m.set_dropout_seed(8)
    assert not np.array_equal(np.asarray(m(img)), first[0])
    m.set_dropout_seed(None)
    with pytest.raises(NotImplementedError):
        m(img)


@pytest.mark.parametrize("name", ["vit_cls", "crossvit_proj"])
def test_graph_replays_match_eager_calls(lib, name):
    import torch
    from vit_tensorflow_b200 import _lib
    img = o.images(name)
    eager, graphed = _model(name, "bf16"), _model(name, "bf16")
    eager.set_dropout_seed(3)
    graphed.set_dropout_seed(3)
    b, h, w, _ = img.shape
    x = torch.from_numpy(np.ascontiguousarray(img)).cuda()
    out = torch.empty((b, graphed.num_classes), device="cuda")
    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    st0 = graphed.graph_stats()
    calls = 5
    for _ in range(calls):                           # eager, capture, replays
        graphed.forward_raw(x.data_ptr(), _lib.MEM_DEVICE, b, h, w, out.data_ptr(), _lib.MEM_DEVICE, s.cuda_stream, training=True)
        s.synchronize()
        np.testing.assert_array_equal(out.cpu().numpy(), np.asarray(eager(img)))
    st = graphed.graph_stats()
    assert (st["captures"] - st0["captures"], st["replays"] - st0["replays"], st["failures"] - st0["failures"]) == (1, calls - 2, 0)


@pytest.mark.parametrize("name", ["vit_cls", "cait", "crossvit_samedim"])
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_inference_forward_is_untouched(lib, name, precision):
    img = o.images(name)
    plain = np.asarray(_model(name, precision)(img, training=False))
    m = _model(name, precision)
    m.set_dropout_seed(5)
    np.asarray(m(img))                               # a training call first: the inference forward after it is unchanged
    np.testing.assert_array_equal(np.asarray(m(img, training=False)), plain)
    z = _model(name, precision, dropout=0.0, emb_dropout=0.0)
    z.set_dropout_seed(5)
    np.testing.assert_array_equal(np.asarray(z(img)), plain)     # all rates 0: the inference forward


def test_all_zero_rates_run_the_inference_forward(lib):
    """vb_forward_train with all rates 0 is vb_forward: the same launches (no counter advance) and the same logits."""
    import ctypes as C
    from vit_tensorflow_b200 import _lib
    img = o.images("vit_cls")
    m = _model("vit_cls", "fp32")
    m._finalize()
    b, h, w, _ = img.shape
    x = np.ascontiguousarray(img, np.float32)
    warm = np.empty((b, m.num_classes), np.float32)         # the first call also builds the embedding's residual operand
    _lib.check(m._lib.vb_forward(m._h, x.ctypes.data_as(C.c_void_p), _lib.MEM_HOST, b, h, w, warm.ctypes.data_as(C.c_void_p),
                                 _lib.MEM_HOST, None), m._h)
    outs = []
    for fn in (m._lib.vb_forward, m._lib.vb_forward_train):
        out = np.empty((b, m.num_classes), np.float32)
        if fn is m._lib.vb_forward_train:
            _lib.check(m._lib.vb_set_dropout(m._h, 0.0, 0.0, o.SEED), m._h)
        _lib.check(fn(m._h, x.ctypes.data_as(C.c_void_p), _lib.MEM_HOST, b, h, w, out.ctypes.data_as(C.c_void_p), _lib.MEM_HOST, None), m._h)
        outs.append((out, m.last_launch_count))
    np.testing.assert_array_equal(outs[0][0], outs[1][0])
    assert outs[0][1] == outs[1][1]
    _lib.check(m._lib.vb_set_dropout(m._h, 0.1, 0.1, o.SEED), m._h)
    out = np.empty((b, m.num_classes), np.float32)
    _lib.check(m._lib.vb_forward_train(m._h, x.ctypes.data_as(C.c_void_p), _lib.MEM_HOST, b, h, w, out.ctypes.data_as(C.c_void_p),
                                       _lib.MEM_HOST, None), m._h)
    assert m.last_launch_count == outs[0][1] + 1        # the counter's advance


def test_fp32_image_logits_do_not_depend_on_the_batch_after_it(lib):
    name = "vit_cls"
    img2 = o.images(name)
    img3 = np.concatenate([img2, img2[:1] * 0.5], axis=0)
    m = _model(name, "fp32")
    m.set_dropout_seed(11)
    a = np.asarray(m(img2))
    m.set_dropout_seed(11)
    b = np.asarray(m(img3))
    np.testing.assert_array_equal(a, b[:2])


def test_readme_usage(lib):
    import vit_tensorflow_b200 as vb
    v = vb.ViT(image_size=64, patch_size=16, num_classes=10, dim=64, depth=2, heads=4, mlp_dim=128, dropout=0.1, emb_dropout=0.1)
    img = np.random.default_rng(0).standard_normal((2, 64, 64, 3)).astype(np.float32)
    with pytest.raises(NotImplementedError):
        v(img)
    v.set_dropout_seed(0)
    preds = np.asarray(v(img))
    assert preds.shape == (2, 10) and np.isfinite(preds).all()
    c = vb.CrossViT(image_size=64, num_classes=10, sm_dim=64, lg_dim=128, sm_patch_size=8, lg_patch_size=16, depth=1,
                    sm_enc_depth=1, lg_enc_depth=1, cross_attn_depth=1, cross_attn_heads=2, cross_attn_dim_head=32)
    c.set_dropout_seed(0)
    assert np.isfinite(np.asarray(c(img))).all()

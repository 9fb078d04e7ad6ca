"""The CCT (reference cct.py) on the H100 engine: fp32 and bf16 against the float64 spec and the reference-code fixtures
(tests/golden/cct_*__refshim.npz, tests/golden/make_cct_golden.py), the two tools/cct_bench.py configurations at their own size,
the 'none' embedding on a smaller image, the training=False rule, graph replay, batch independence, and a ViT built from a
vb_config of the ABI-7 size (before the CCT fields were appended)."""
import ctypes as C
import os

import numpy as np
import pytest

import cct_oracle as co

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
FP32_RTOL, FP32_ATOL = 1e-3, 1e-4
BF16_RTOL, BF16_ATOL = 4e-2, 6e-2            # the bf16 bound of test_gpu_models.py
# config-size bound (atol, rtol), the ViT-L/16 line of test_gpu_config_size.py: bf16 operands and activations over 7 / 14 layers
BENCH_TOL = (6.0e-2, 1.5e-2)


def _model(cfg, w, precision):
    from vit_tensorflow_b200 import from_config
    m = from_config(cfg, precision=precision)
    m.set_weights_dict(w)
    return m


def _fixture(name, gen):
    return np.load(os.path.join(GOLDEN, f"{name}__{gen}__refshim.npz"))["logits_ref_f32"].astype(np.float64)


@pytest.mark.parametrize("gen", ["init_weights", "stress_weights"])
@pytest.mark.parametrize("name", sorted(co.SMALL))
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_cct_small_vs_spec_and_reference_fixture(lib, precision, name, gen):
    cfg = co.make_config(**co.SMALL[name])
    w = getattr(co, gen)(cfg, co.WEIGHT_SEED)
    img = co.make_image(cfg, co.BATCH, co.IMAGE_SEED)
    got = _model(cfg, w, precision)(img, training=False).numpy().astype(np.float64)
    ref = co.forward(img, w, cfg)
    zr = _fixture(name, gen)
    assert got.shape == ref.shape and np.isfinite(got).all()
    atol, rtol = (FP32_ATOL, FP32_RTOL) if precision == "fp32" else (BF16_ATOL, BF16_RTOL)
    for r in (ref, zr):
        assert (np.abs(got - r) <= atol + rtol * np.abs(r)).all(), f"max err {np.abs(got - r).max():.3g}"


@pytest.mark.parametrize("gen", ["stress_weights", "init_weights"])
@pytest.mark.parametrize("name", sorted(co.BENCH))
def test_cct_bf16_at_config_size(lib, name, gen):
    cfg = co.make_config(**co.BENCH[name])
    w = getattr(co, gen)(cfg, co.WEIGHT_SEED)
    img = co.make_image(cfg, co.BATCH, co.IMAGE_SEED)
    got = _model(cfg, w, "bf16")(img, training=False).numpy().astype(np.float64)
    ref = co.forward(img, w, cfg)
    zr = _fixture(name, gen)
    assert np.abs(zr - ref).max() < 5e-5
    atol, rtol = BENCH_TOL
    err = np.abs(got - ref)
    print(f"\n[cct config-size parity] {name} {gen}: max err {err.max():.4g}, worst ratio {(err / (atol + rtol * np.abs(ref))).max():.3g}, "
          f"|ref| max {np.abs(ref).max():.3g}, argmax agree {(got.argmax(-1) == ref.argmax(-1)).mean():.2f}")
    assert (err <= atol + rtol * np.abs(ref)).all(), f"max err {err.max():.4f}"
    assert (np.abs(got - zr) <= atol + rtol * np.abs(zr)).all()


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_cct_none_embedding_pads_a_smaller_image(lib, precision):
    """'none': a 14 x 14 image gives 7 x 7 = 49 tokens, zero-padded to the 100 of img_size 20 (cct.py:278-280); the padded rows
    take part in attention and pooling.  A larger image passes through with its own token count."""
    cfg = co.make_config(**co.SMALL["cct_small_none"])
    w = co.stress_weights(cfg, 3)
    m = _model(cfg, w, precision)
    atol, rtol = (FP32_ATOL, FP32_RTOL) if precision == "fp32" else (BF16_ATOL, BF16_RTOL)
    for hw in ((14, 14), (24, 20)):
        img = co.make_image(cfg, 3, 4, *hw)
        got = m(img, training=False).numpy().astype(np.float64)
        ref = co.forward(img, w, cfg)
        assert (np.abs(got - ref) <= atol + rtol * np.abs(ref)).all(), (hw, float(np.abs(got - ref).max()))


def test_cct_positional_embedding_needs_the_configured_token_count(lib):
    from vit_tensorflow_b200 import _lib
    cfg = co.make_config(**co.SMALL["cct_small_sine"])
    m = _model(cfg, co.init_weights(cfg, 1), "bf16")
    with pytest.raises(_lib.VbError, match="positional embedding has 64 rows"):
        m(co.make_image(cfg, 1, 0, 24, 24), training=False)


def test_cct_training_not_false_raises(lib):
    from vit_tensorflow_b200 import cct_2
    m = cct_2(img_size=32, kernel_size=3, n_conv_layers=1, num_classes=4)
    img = np.zeros((1, 32, 32, 3), np.float32)
    for kw in ({}, dict(training=None), dict(training=True)):
        with pytest.raises(NotImplementedError, match="training=False"):
            m(img, **kw)
    assert m(img, training=False).shape == (1, 4)


def test_cct_graph_replay_is_bit_identical_and_batch_independent(lib):
    import torch
    from vit_tensorflow_b200 import _lib
    cfg = co.make_config(**co.BENCH["cct_7_3x1"])
    m = _model(cfg, co.stress_weights(cfg, 5), "bf16")
    img = co.make_image(cfg, 16, 6)
    eager = m(img, training=False).numpy()
    x = torch.from_numpy(img).cuda()
    out = torch.empty((16, cfg["num_classes"]), device="cuda")
    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    st0 = m.graph_stats()
    outs = []
    for _ in range(4):                                       # eager, capture + launch, replay, replay
        m.forward_raw(x.data_ptr(), _lib.MEM_DEVICE, 16, 32, 32, out.data_ptr(), _lib.MEM_DEVICE, s.cuda_stream)
        s.synchronize()
        outs.append(out.cpu().numpy().copy())
    st = m.graph_stats()
    assert (st["captures"] - st0["captures"], st["replays"] - st0["replays"], st["failures"] - st0["failures"]) == (1, 2, 0), st
    for o in outs:
        np.testing.assert_array_equal(o, eager)
    for sub in (slice(0, 1), slice(3, 9)):                   # each image's logits do not depend on its batch neighbours
        np.testing.assert_array_equal(m(img[sub], training=False).numpy(), eager[sub])


def test_cct_stage_entries_are_refused(lib):
    from vit_tensorflow_b200 import _lib
    cfg = co.make_config(**co.SMALL["cct_small_sine"])
    m = _model(cfg, co.init_weights(cfg, 1), "fp32")
    img = co.make_image(cfg, 1, 0)
    for call in (lambda: m.forward_embed(img), lambda: m.forward_head(np.zeros((1, 64, 64), np.float32)),
                 lambda: m.forward_tokens(np.zeros((1, 64, 64), np.float32))):
        with pytest.raises(_lib.VbError, match="CCT|supports ViT"):
            call()


def test_abi7_sized_config_builds_the_same_vit(lib):
    """A client compiled against the ABI-7 vb_config without the CCT fields passes the shorter struct_size: vb_create reads only
    that prefix.  The same ViT built through both sizes gives bit-identical logits."""
    import oracle
    from vit_tensorflow_b200 import _lib, from_config
    cfg = oracle.make_config("vit", image_size=32, patch_size=8, num_classes=5, dim=64, depth=2, heads=2, mlp_dim=128)
    w = oracle.stress_weights(cfg, 2)
    img = oracle.make_image(cfg, 2, 3)
    m = from_config(cfg, precision="bf16")
    m.set_weights_dict(w)
    want = m(img, training=False).numpy()

    L = lib
    full = m._cfg
    raw = (C.c_char * _lib.CONFIG_SIZE_ABI7).from_buffer_copy(bytes(full)[:_lib.CONFIG_SIZE_ABI7])
    C.cast(raw, C.POINTER(C.c_int32))[0] = _lib.CONFIG_SIZE_ABI7
    h = C.c_void_p()
    _lib.check(L.vb_create(C.cast(raw, C.POINTER(_lib.VbConfig)), 0, C.byref(h)))
    try:
        for name, a in w.items():
            a = np.ascontiguousarray(a, np.float32)
            shape = (C.c_int64 * a.ndim)(*a.shape)
            _lib.check(L.vb_set_weight(h, name.encode(), a.ctypes.data_as(C.c_void_p), shape, a.ndim), h)
        _lib.check(L.vb_finalize(h), h)
        out = np.empty_like(want)
        x = np.ascontiguousarray(img)
        _lib.check(L.vb_forward(h, x.ctypes.data_as(C.c_void_p), _lib.MEM_HOST, 2, 32, 32, out.ctypes.data_as(C.c_void_p),
                                _lib.MEM_HOST, None), h)
    finally:
        L.vb_destroy(h)
    np.testing.assert_array_equal(out, want)

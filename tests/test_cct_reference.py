"""The CCT oracle (tests/cct_oracle.py) pinned on the reference's own cct.py, and the CCT host surface, without a GPU.

1. the stand-in's Conv2D / MaxPool2D 'SAME' against PyTorch with the asymmetric padding spelled out;
2. LIVE (skipped where the reference checkout is absent): cct.CCT, constructed by its own __init__ and loaded by attribute path,
   equals the float64 spec to 1e-12 on hand-picked cases and 40 seeded random configurations, and the torch restatement;
3. the committed fixtures tests/golden/cct_*__refshim.npz equal the spec;
4. the boundary: constructor / call signatures and constructor errors equal the reference's, the sine table is the
   reference's sinusoidal_embedding, and a vb_config of the ABI-7 size passes the struct-size check.
"""
import ctypes as C
import inspect
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import cct_oracle as co
from oracle import tf_shim

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
REF_DIR = os.environ.get("VB_REFERENCE_DIR", "/root/reference/vit_tensorflow")
live = pytest.mark.skipif(not os.path.exists(os.path.join(REF_DIR, "cct.py")), reason="reference checkout not present: the fixtures cover it")


@pytest.fixture
def f64():
    tf_shim.set_dtype(np.float64)
    yield
    tf_shim.set_dtype(np.float32)


def _torch_same(x, k, s, value):
    H, W = x.shape[-2:]
    oh, ow = -(-H // s), -(-W // s)
    ph, pw = max((oh - 1) * s + k - H, 0), max((ow - 1) * s + k - W, 0)
    return F.pad(x, (pw // 2, pw - pw // 2, ph // 2, ph - ph // 2), value=value)


# ------------------------------------------------------------------------------------------ 1. primitives vs torch
@pytest.mark.parametrize("H,W,k,s", [(9, 9, 3, 2), (10, 7, 7, 2), (8, 8, 2, 3), (5, 11, 5, 1), (6, 6, 1, 2), (7, 4, 3, 3)])
def test_shim_conv2d_and_maxpool2d_same_against_torch(f64, H, W, k, s):
    rng = np.random.default_rng(H * 100 + W * 10 + k + s)
    x = rng.standard_normal((2, H, W, 3))
    with co.installed(None):
        import tensorflow.keras.layers as nn
        conv = nn.Conv2D(filters=5, kernel_size=k, strides=s, padding='SAME', use_bias=False)
        conv(x)
        kern = rng.standard_normal((k, k, 3, 5))
        conv.set_weights([kern])
        got = np.asarray(conv(x))
        pool = np.asarray(nn.MaxPool2D(pool_size=k, strides=s, padding='SAME')(x))
        relu = np.asarray(nn.ReLU()(x))
    xt = torch.from_numpy(x).permute(0, 3, 1, 2)
    want = F.conv2d(_torch_same(xt, k, s, 0.0), torch.from_numpy(kern).permute(3, 2, 0, 1), stride=s).permute(0, 2, 3, 1).numpy()
    np.testing.assert_allclose(got, want, atol=1e-12)
    assert got.shape[1:3] == (-(-H // s), -(-W // s))
    pwant = F.max_pool2d(_torch_same(xt, k, s, -np.inf), k, s).permute(0, 2, 3, 1).numpy()
    np.testing.assert_array_equal(pool, pwant)
    np.testing.assert_array_equal(co.maxpool_same(x, k, s), pwant)
    np.testing.assert_array_equal(relu, np.maximum(x, 0))


def test_shim_conv2d_glorot_uses_the_receptive_field():
    with co.installed(None):
        import tensorflow.keras.layers as nn
        conv = nn.Conv2D(filters=64, kernel_size=7, strides=2, padding='SAME', use_bias=False)
        conv(np.zeros((1, 8, 8, 3), np.float32))
        lim = np.sqrt(6.0 / (49 * (3 + 64)))
        assert conv.kernel.shape == (7, 7, 3, 64) and np.abs(conv.kernel).max() <= lim and np.abs(conv.kernel).max() > 0.9 * lim


# ------------------------------------------------------------------------------------------ 2. live reference
def _random_case(rng):
    heads = int(rng.choice([1, 2, 3]))
    dim = heads * int(rng.choice([4, 8]))
    case = dict(img_size=int(rng.integers(7, 26)) if rng.random() < 0.6 else (int(rng.integers(7, 26)), int(rng.integers(7, 26))),
                embedding_dim=dim, n_conv_layers=int(rng.integers(1, 4)), kernel_size=int(rng.choice([1, 2, 3, 5, 7])),
                stride=int(rng.choice([1, 2, 3])), pooling_kernel_size=int(rng.choice([1, 2, 3])), pooling_stride=int(rng.choice([1, 2, 3])),
                num_layers=int(rng.integers(0, 3)), num_heads=heads, mlp_ratio=float(rng.choice([1, 1.5, 2])),
                num_classes=int(rng.integers(2, 6)), positional_embedding=str(rng.choice(['sine', 'learnable', 'none'])))
    return case


@live
@pytest.mark.parametrize("name", sorted(co.SMALL) + sorted(co.BENCH))
def test_live_reference_equals_spec(f64, name):
    cfg = co.make_config(**{**co.SMALL, **co.BENCH}[name])
    w = co.stress_weights(cfg, 4)
    img = co.make_image(cfg, 2, 5)
    got = co.reference_logits(cfg, w, img, reference_dir=REF_DIR)
    ref = co.forward(img, w, cfg)
    assert np.abs(got - ref).max() <= 1e-12 * max(1.0, np.abs(ref).max())
    assert np.abs(co.forward_torch(img, w, cfg) - ref).max() <= 1e-12 * max(1.0, np.abs(ref).max())


@live
def test_live_reference_equals_spec_on_random_configurations(f64):
    """40 seeded random configurations: 1-3 conv layers, kernel / stride / pooling combinations, odd and rectangular images, all
    three positional embeddings, and for 'none' also a smaller image (zero-padded tokens) -- reference == float64 spec to 1e-12."""
    for seed in range(40):
        rng = np.random.default_rng(7000 + seed)
        case = _random_case(rng)
        cfg = co.make_config(**case)
        w = co.stress_weights(cfg, seed)
        img = co.make_image(cfg, 2, seed + 1)
        got = co.reference_logits(cfg, w, img, reference_dir=REF_DIR)
        ref = co.forward(img, w, cfg)
        assert got.shape == ref.shape, (seed, case)
        assert np.abs(got - ref).max() <= 1e-12 * max(1.0, np.abs(ref).max()), (seed, case, float(np.abs(got - ref).max()))
        if seed < 8:
            assert np.abs(co.forward_torch(img, w, cfg) - ref).max() <= 1e-12 * max(1.0, np.abs(ref).max()), (seed, case)
        if cfg["positional_embedding"] == "none":
            small = co.make_image(cfg, 2, seed + 2, max(1, cfg["image_h"] - 5), max(1, cfg["image_w"] - 3))
            got = co.reference_logits(cfg, w, img, reference_dir=REF_DIR, img_call=small)
            ref = co.forward(small, w, cfg)
            assert np.abs(got - ref).max() <= 1e-12 * max(1.0, np.abs(ref).max()), (seed, case, "smaller image")


@live
def test_live_sine_table_is_the_references():
    from vit_tensorflow_b200.models import sinusoidal_embedding
    import importlib
    with co.installed(REF_DIR):
        tc = importlib.import_module("cct").TransformerClassifier
        for n, d in ((196, 384), (17, 10), (5, 7)):
            want = np.asarray(tc.sinusoidal_embedding(None, n, d))
            got = sinusoidal_embedding(n, d)
            assert got.dtype == want.dtype == np.float32 and got.shape == want.shape == (1, n, d)
            np.testing.assert_array_equal(got, want)


# ------------------------------------------------------------------------------------------ 3. fixtures
@pytest.mark.parametrize("gen", ["init_weights", "stress_weights"])
@pytest.mark.parametrize("name", sorted(co.SMALL) + sorted(co.BENCH))
def test_reference_fixture_equals_spec(name, gen):
    cfg = co.make_config(**{**co.SMALL, **co.BENCH}[name])
    w = getattr(co, gen)(cfg, co.WEIGHT_SEED)
    img = co.make_image(cfg, co.BATCH, co.IMAGE_SEED)
    z = np.load(os.path.join(GOLDEN, f"{name}__{gen}__refshim.npz"))
    ref = co.forward(img, w, cfg)
    assert np.abs(z["logits_ref_f32"] - ref).max() <= 5e-5 * max(1.0, np.abs(ref).max())
    if name in co.SMALL:
        assert np.abs(z["logits_ref_f64"] - ref).max() <= 1e-12 * max(1.0, np.abs(ref).max())


# ------------------------------------------------------------------------------------------ 4. the boundary
@live
def test_live_constructor_and_call_signatures_equal_the_reference():
    import importlib
    import vit_tensorflow_b200 as vb
    with co.installed(REF_DIR):
        m = importlib.import_module("cct")
        ref_init = list(inspect.signature(m.CCT.__init__).parameters.values())[1:]
        ref_call = list(inspect.signature(m.CCT.call).parameters.values())[1:]
        ref_factories = {n: inspect.signature(getattr(m, n)) for n in m.__all__}
        ref_inner = inspect.signature(m._cct)
    ours = [p for p in list(inspect.signature(vb.CCT.__init__).parameters.values())[1:] if p.kind is not inspect.Parameter.KEYWORD_ONLY]
    assert [(p.name, p.kind, p.default) for p in ours] == [(p.name, p.kind, p.default) for p in ref_init]
    extra = [p.name for p in inspect.signature(vb.CCT.__init__).parameters.values() if p.kind is inspect.Parameter.KEYWORD_ONLY]
    assert extra == ["precision", "device", "seed"]
    mine = list(inspect.signature(vb.CCT.__call__).parameters.values())[1:]
    assert [(p.name, p.kind, p.default) for p in mine] == [(p.name, p.kind, p.default) for p in ref_call]
    assert vb.CCT.call is vb.CCT.__call__
    from vit_tensorflow_b200 import models
    for n, sig in ref_factories.items():
        assert inspect.signature(getattr(models, n)) == sig
    assert inspect.signature(models._cct) == ref_inner
    import vit_tensorflow.cct as shim
    assert shim.CCT is vb.CCT and all(getattr(shim, n) is getattr(vb, n) for n in ref_factories)


def _strip_module(msg):
    return msg.replace("vit_tensorflow_b200.models.", "").replace("cct.", "")


@live
@pytest.mark.parametrize("args,kw", [
    ((), dict(seq_pool=False)), ((), dict(dropout_rate=0.0)), ((), dict(attention_dropout=0.0)),
    ((), dict(stochastic_depth_rate=0.0)), ((), dict(sequence_length=4)),
    ((32, 64, 3, 1, 3, 1, 3, 2, True), {}),                                  # a positional extra lands on seq_pool
])
def test_live_constructor_errors_equal_the_reference(args, kw):
    import importlib
    import vit_tensorflow_b200 as vb
    base = dict(num_layers=1, num_heads=2, embedding_dim=16) if not args else dict(num_layers=1, num_heads=2)
    if not args:
        base["img_size"] = 16
    with co.installed(REF_DIR):
        with pytest.raises(Exception) as ref_exc:
            importlib.import_module("cct").CCT(*args, **base, **kw)
    with pytest.raises(Exception) as our_exc:
        vb.CCT(*args, **base, **kw)
    assert type(our_exc.value) is type(ref_exc.value) is TypeError
    assert _strip_module(str(our_exc.value)) == _strip_module(str(ref_exc.value))


@live
def test_live_unknown_kwargs_are_swallowed_like_the_reference():
    """The README's own example passes padding / pooling_padding / mlp_radio (a typo): the reference ignores them, and so does
    the classifier configuration here (mlp_ratio stays 4.0); an unknown positional_embedding falls back to 'sine'."""
    import importlib
    from vit_tensorflow_b200.models import TransformerClassifier
    kw = dict(img_size=16, embedding_dim=16, n_conv_layers=1, kernel_size=3, stride=1, num_layers=1, num_heads=2, padding=3,
              pooling_padding=1, mlp_radio=3., positional_embedding='rotary')
    with co.installed(REF_DIR):
        ref = importlib.import_module("cct").CCT(**kw)
        ref(np.zeros((1, 16, 16, 3), np.float32), training=False)
        units = ref.classifier.blocks.layers[0].linear1.units
        has_pos = ref.classifier.positional_emb is not None
    tc = TransformerClassifier(sequence_length=64, embedding_dim=16, seq_pool=True, dropout_rate=0., attention_dropout=0.1,
                               stochastic_depth_rate=0.1, num_layers=1, num_heads=2, padding=3, pooling_padding=1, mlp_radio=3.,
                               positional_embedding='rotary')
    assert units == tc.mlp_dim == 64 and has_pos and tc.positional_embedding == 'sine'


def test_host_rejects_what_the_engine_cannot_run():
    import vit_tensorflow_b200 as vb
    with pytest.raises(ValueError, match="divisible by num_heads"):
        vb.CCT(img_size=16, embedding_dim=30, num_heads=4)
    with pytest.raises(NotImplementedError, match="3 channels"):
        vb.CCT(img_size=16, embedding_dim=32, num_heads=4, n_input_channels=1)


def test_oracle_config_of_the_bench_models():
    c14 = co.make_config(**co.BENCH["cct_14_7x2"])
    assert (c14["stride"], c14["sequence_length"], c14["dim"], c14["mlp_dim"], c14["depth"]) == (2, 196, 384, 1152, 14)
    assert co.weight_specs(c14)["tokenizer.conv.1.kernel"][0] == (7, 7, 64, 384)
    c7 = co.make_config(**co.BENCH["cct_7_3x1"])
    assert (c7["stride"], c7["sequence_length"], c7["dim"], c7["num_classes"]) == (1, 256, 256, 10)


def _has_gpu():
    try:
        return torch.cuda.is_available()
    except Exception:
        return False


@pytest.mark.skipif(_has_gpu(), reason="checks the no-GPU failure mode")
def test_abi7_sized_config_passes_the_struct_size_check(lib):
    """vb_create accepts the ABI-7 struct (without the CCT fields) and the full one: on a CPU box both get as far as the device
    check; any other struct_size is still refused before it."""
    from vit_tensorflow_b200 import _lib
    assert _lib.CONFIG_SIZE_ABI7 == 45 * 4 and C.sizeof(_lib.VbConfig) == _lib.CONFIG_SIZE_ABI7 + 6 * 4
    cfg = _lib.VbConfig(kind=0, precision=1, image_h=32, image_w=32, patch_h=16, patch_w=16, channels=3, num_classes=4, dim=64,
                        depth=1, heads=2, dim_head=32, mlp_dim=64)
    for size, msg in ((_lib.CONFIG_SIZE_ABI7, b"no CUDA device"), (C.sizeof(_lib.VbConfig), b"no CUDA device"),
                      (_lib.CONFIG_SIZE_ABI7 + 4, b"struct_size mismatch"), (C.sizeof(_lib.VbConfig) + 4, b"struct_size mismatch")):
        cfg.struct_size = size
        h = C.c_void_p()
        assert lib.vb_create(C.byref(cfg), 0, C.byref(h)) != 0
        assert msg in lib.vb_last_error(None), (size, lib.vb_last_error(None))

"""CrossFormer (reference crossformer.py) on the H100 engine: fp32 and bf16 against the float64 spec and the reference-code fixtures
(tests/golden/crossformer_*__refshim.npz, tests/golden/make_crossformer_golden.py), the two tools/crossformer_bench.py
configurations at their own size, vb_op_window_bias_attention against numpy, the kernel classes of a profiled forward, one
handle over several image sizes and the refused ones, the training / dropout rule, graph replay and batch independence."""
import os

import numpy as np
import pytest

import crossformer_oracle as co

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
FP32_RTOL, FP32_ATOL = 1e-3, 1e-4
BF16_RTOL, BF16_ATOL = 4e-2, 6e-2            # the bf16 bound of test_gpu_models.py


def _model(cfg, w, precision, **kw):
    from vit_tensorflow_b200 import CrossFormer
    m = CrossFormer(**{**co.ctor_kwargs(cfg), **kw}, precision=precision)
    m.set_weights_dict(w)
    return m


def _within(got, want, atol, rtol):
    err = np.abs(got - want)
    assert np.isfinite(got).all() and (err <= atol + rtol * np.abs(want)).all(), f"max err {err.max():.3g}"


@pytest.mark.parametrize("gen", ["init_weights", "stress_weights"])
@pytest.mark.parametrize("name", sorted(co.SMALL))
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_crossformer_small_vs_spec_and_reference_fixture(lib, precision, name, gen):
    cfg = co.make_config(**co.SMALL[name])
    w = getattr(co, gen)(cfg, co.WEIGHT_SEED)
    img = co.make_image(cfg, co.BATCH, co.IMAGE_SEED)
    got = np.asarray(_model(cfg, w, precision)(img), np.float64)
    ref = co.forward(img, w, cfg)
    fix = np.load(os.path.join(GOLDEN, f"{name}__{gen}__refshim.npz"))["logits_ref_f64"]
    atol, rtol = (FP32_ATOL, FP32_RTOL) if precision == "fp32" else (BF16_ATOL, BF16_RTOL)
    assert got.shape == ref.shape
    for want in (ref, fix):
        _within(got, want, atol, rtol)


@pytest.mark.parametrize("name", sorted(co.BENCH))
def test_crossformer_bf16_at_config_size(lib, name):
    """The two tools/crossformer_bench.py models at full size (224^2) with stress weights, against the spec and the fixture: the
    engine's error is held to twice what bf16 storage alone costs (forward_bf16_storage: the convolutions' operands and results and
    the stream after every sub-block rounded to bf16, all arithmetic in float64), as for Twins-SVT and LeViT."""
    cfg = co.make_config(**co.BENCH[name])
    img = co.make_image(cfg, co.BATCH, co.IMAGE_SEED)
    w = co.stress_weights(cfg, co.WEIGHT_SEED)
    got = _model(cfg, w, "bf16")(img).numpy().astype(np.float64)
    ref = co.forward(img, w, cfg)
    fix = np.load(os.path.join(GOLDEN, f"{name}__stress_weights__refshim.npz"))["logits_ref_f32"]
    storage = np.abs(co.forward_bf16_storage(img, w, cfg) - ref)
    err = np.abs(got - ref).max()
    print(f"{name}: bf16 max err {err:.4f}, bf16 storage alone {storage.max():.4f} (|ref| max {np.abs(ref).max():.3f})")
    assert np.isfinite(got).all() and err <= 2.0 * storage.max()
    assert np.abs(got - fix).max() <= 2.0 * storage.max() + np.abs(fix - ref).max()


def _window_bias_ref(qkv, B, H, W, wsz, long, heads, dh, table):
    inner = heads * dh
    x = co.windows(qkv[:, :3 * inner].astype(np.float64).reshape(B, H, W, 3 * inner), wsz, long)
    q, k, v = (x[..., i * inner:(i + 1) * inner].reshape(x.shape[0], -1, heads, dh).transpose(0, 2, 1, 3) for i in range(3))
    i, j = np.divmod(np.arange(wsz * wsz), wsz)
    bias = table[(i[:, None] - i[None, :] + wsz - 1) * (2 * wsz - 1) + (j[:, None] - j[None, :] + wsz - 1)]
    s = q @ np.swapaxes(k, -1, -2) * dh ** -0.5 + bias
    a = np.exp(s - s.max(-1, keepdims=True))
    o = (a / a.sum(-1, keepdims=True)) @ v
    return co.unwindows(o.transpose(0, 2, 1, 3).reshape(x.shape[0], -1, inner), B, H, W, wsz, long).reshape(B * H * W, inner)


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("dh", [32, 64])
@pytest.mark.parametrize("long", [False, True], ids=["short", "long"])
@pytest.mark.parametrize("wsz,gy,gx", [(2, 3, 5), (3, 2, 7), (4, 5, 2), (7, 2, 3), (8, 1, 2), (9, 2, 1)])
def test_op_window_bias_attention_against_numpy(lib, precision, dh, long, wsz, gy, gx):
    """Windows of 4, 9 and 16 tokens (packed 16, 7 and 4 to a query tile, a partial last tile among them), 49 and 64 (one per tile)
    and 81 (two query tiles and key blocks), contiguous and dilated, on non-square window grids; the q|k|v rows are read in place
    (pitch wider than q|k|v), the output rows written pixel-major.  bf16 runs the windowed-bias flash kernel, fp32 the permuted
    materialised-scores path with the table added."""
    from vit_tensorflow_b200 import _lib
    B, heads = 3, 3
    H, W = gy * wsz, gx * wsz
    rng = np.random.default_rng(wsz * 1000 + gy * 100 + gx * 10 + dh + long)
    qkv = rng.standard_normal((B * H * W, 3 * heads * dh + 64)).astype(np.float32)
    table = (2.0 * rng.standard_normal((2 * wsz - 1) ** 2)).astype(np.float32)
    _lib.last_attention_path()
    got, _ = _lib.op_window_bias_attention(qkv, H, W, wsz, long, heads, dh, table, precision=precision)
    assert _lib.last_attention_path() == ("flash" if precision == "bf16" else "simt")
    ref = _window_bias_ref(qkv, B, H, W, wsz, long, heads, dh, table.astype(np.float64))
    atol, rtol = (1e-4, 1e-4) if precision == "fp32" else (2e-2, 2e-2)
    _within(got.astype(np.float64), ref, atol, rtol)


@pytest.mark.parametrize("name", ["crossformer_small", "crossformer_odd"])
def test_crossformer_bf16_profile_flash_and_no_fallbacks(lib, name):
    """One profiled bf16 forward: one flash launch per attention sub-block whose windows hold more than one token and none for
    one-token windows (there the output is v itself), no launch of the "other" class (a GEMM on the SIMT fallback or a window
    permutation would be counted there, for width 96 as well), and one LayerNorm-folded GELU fc1 per MLP."""
    from vit_tensorflow_b200 import _lib
    cfg = co.make_config(**co.SMALL[name])
    w = co.stress_weights(cfg, co.WEIGHT_SEED)
    img = co.make_image(cfg, co.BATCH, co.IMAGE_SEED)
    m = _model(cfg, w, "bf16")
    m(img)
    m.profile(True)
    m.profile_read(reset=True)
    _lib.last_attention_path()
    got = m(img).numpy().astype(np.float64)
    prof = m.profile_read(reset=True)
    m.profile(False)
    st = co.stages(cfg)
    n_attn = sum(s["depth"] * ((s["local_wsz"] > 1) + (s["global_wsz"] > 1)) for s in st)
    n_one = sum(s["depth"] * ((s["local_wsz"] == 1) + (s["global_wsz"] == 1)) for s in st)
    assert n_attn > 0 and n_one > 0
    assert _lib.last_attention_path() == "flash"
    assert prof["attention"]["launches"] == n_attn, prof
    assert prof["other"]["launches"] == 0, prof
    assert prof["gemm_wgmma_gelu"]["launches"] == 2 * sum(s["depth"] for s in st), prof
    _within(got, co.forward(img, w, cfg), BF16_ATOL, BF16_RTOL)


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_crossformer_image_sizes_and_refusals(lib, precision):
    """One handle serves 224^2, 448^2 and 224 x 448 images (its arena grows; nothing depends on the image size but the maps).
    Sizes that break the shape rule raise ValueError naming the stage, the map and the window size."""
    cfg = co.make_config(image_size=224, num_classes=7, dim=(32, 64, 64, 96), depth=(1, 1, 1, 1))
    w = co.stress_weights(cfg, 3)
    m = _model(cfg, w, precision)
    atol, rtol = (FP32_ATOL, FP32_RTOL) if precision == "fp32" else (BF16_ATOL, BF16_RTOL)
    for h, wd, batch in ((224, 224, 2), (448, 448, 1), (224, 448, 2), (224, 224, 1)):
        img = co.make_image(cfg, batch, h + wd, h, wd)
        got = m(img)
        assert got.shape == (batch, 7)
        _within(np.asarray(got, np.float64), co.forward(img, w, cfg), atol, rtol)
    for h, wd, msg in ((220, 224, "stage 1: the 55 x 56 map is not divisible by local_window_size 7"),
                       (224, 200, "stage 1: the 56 x 50 map is not divisible by local_window_size 7"),
                       (112, 112, "stage 1: the 28 x 28 map is not divisible by global_window_size 8"),
                       (232, 224, "stage 1: the 58 x 56 map is not divisible by local_window_size 7")):
        with pytest.raises(ValueError, match=msg):
            m(co.make_image(cfg, 1, 0, h, wd))


def test_crossformer_training_and_dropout_rule(lib):
    """No BatchNorm: with ff_dropout = 0 training=True computes what training=False does; with ff_dropout > 0 only training=True
    is refused, as for ViT; attn_dropout is accepted at any value (the reference never applies it)."""
    from vit_tensorflow_b200 import _lib
    cfg = co.make_config(**co.SMALL["crossformer_small"])
    w = co.stress_weights(cfg, 2)
    img = co.make_image(cfg, 2, 3)
    m = _model(cfg, w, "bf16")
    assert np.array_equal(m(img), m(img, training=False)) and np.array_equal(m(img, training=True, mask=None), m(img))
    ma = _model(cfg, w, "bf16", attn_dropout=0.3)
    assert np.array_equal(ma(img), m(img))
    md = _model(cfg, w, "bf16", ff_dropout=0.1)
    with pytest.raises(NotImplementedError):
        md(img)
    assert np.array_equal(md(img, training=False), m(img))
    with pytest.raises(_lib.VbError, match="whole forward only"):
        m.forward_head(np.zeros((1, 4, 64), np.float32))
    with pytest.raises(_lib.VbError):
        m.forward_embed(img)


def test_crossformer_graph_replay_and_batch_independence(lib):
    import torch
    cfg = co.make_config(**co.BENCH["crossformer_readme"])
    w = co.stress_weights(cfg, 7)
    m = _model(cfg, w, "bf16")
    B = 8
    img = torch.from_numpy(co.make_image(cfg, B, 8)).cuda()
    out = torch.empty((B, cfg["num_classes"]), dtype=torch.float32, device="cuda")
    s = torch.cuda.Stream()
    outs = []
    with torch.cuda.stream(s):
        for _ in range(4):                                              # eager, capture, replay, replay
            m.forward_raw(img.data_ptr(), 1, B, 224, 224, out.data_ptr(), 1, s.cuda_stream)
            s.synchronize()
            outs.append(out.clone())
    st = m.graph_stats()
    assert st["captures"] == 1 and st["replays"] == 2 and st["failures"] == 0, st
    for o in outs[1:]:
        assert torch.equal(o, outs[0])
    single = m(img[:1].cpu().numpy())
    assert np.array_equal(single, outs[0][:1].cpu().numpy())
    half = m(img[3:7].cpu().numpy())
    assert np.array_equal(half, outs[0][3:7].cpu().numpy())

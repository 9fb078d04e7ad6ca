"""Twins-SVT (reference twins_svt.py) on the H100 engine: fp32 and bf16 against the float64 spec and the reference-code fixtures
(tests/golden/twins_*__refshim.npz, tests/golden/make_twins_golden.py), the two tools/twins_bench.py configurations at their own
size, vb_op_window_attention against numpy, the kernel classes of a profiled forward, one handle over several image sizes and
the refused ones, the training / dropout rule, graph replay and batch independence."""
import os

import numpy as np
import pytest

import twins_oracle as to

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
FP32_RTOL, FP32_ATOL = 1e-3, 1e-4
BF16_RTOL, BF16_ATOL = 4e-2, 6e-2            # the bf16 bound of test_gpu_models.py
BENCH_TOL = (6.0e-2, 1.5e-2)                 # (atol, rtol): the config-size bound of test_gpu_cct.py


def _model(cfg, w, precision, **kw):
    from vit_tensorflow_b200 import TwinsSVT
    m = TwinsSVT(**{**to.ctor_kwargs(cfg), **kw}, precision=precision)
    m.set_weights_dict(w)
    return m


def _within(got, want, atol, rtol):
    err = np.abs(got - want)
    assert np.isfinite(got).all() and (err <= atol + rtol * np.abs(want)).all(), f"max err {err.max():.3g}"


@pytest.mark.parametrize("gen", ["init_weights", "stress_weights"])
@pytest.mark.parametrize("name", sorted(to.SMALL))
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_twins_small_vs_spec_and_reference_fixture(lib, precision, name, gen):
    cfg = to.make_config(**to.SMALL[name])
    w = getattr(to, gen)(cfg, to.WEIGHT_SEED)
    img = to.make_image(cfg, to.BATCH, to.IMAGE_SEED)
    got = np.asarray(_model(cfg, w, precision)(img), np.float64)
    ref = to.forward(img, w, cfg)
    fix = np.load(os.path.join(GOLDEN, f"{name}__{gen}__refshim.npz"))["logits_ref_f64"]
    atol, rtol = (FP32_ATOL, FP32_RTOL) if precision == "fp32" else (BF16_ATOL, BF16_RTOL)
    assert got.shape == ref.shape
    for want in (ref, fix):
        _within(got, want, atol, rtol)


@pytest.mark.parametrize("name", sorted(to.BENCH))
def test_twins_bf16_at_config_size(lib, name):
    """The two tools/twins_bench.py models at full size (224^2) with stress weights, against the spec and the fixture.  Their
    residual streams reach logits of 13-15, and bf16 storage alone (forward_bf16_storage: the 1x1 and to_kv convolutions'
    operands and results, the stream after every sub-block and the PEG output rounded to bf16, all arithmetic in float64) already
    misses the config-size bound of 6e-2 + 1.5e-2 |ref|, by 0.014 and 0.016 at its worst logit.  So the engine's error is held to
    twice that estimate instead, as for LeViT."""
    cfg = to.make_config(**to.BENCH[name])
    img = to.make_image(cfg, to.BATCH, to.IMAGE_SEED)
    w = to.stress_weights(cfg, to.WEIGHT_SEED)
    got = _model(cfg, w, "bf16")(img).numpy().astype(np.float64)
    ref = to.forward(img, w, cfg)
    fix = np.load(os.path.join(GOLDEN, f"{name}__stress_weights__refshim.npz"))["logits_ref_f32"]
    storage = np.abs(to.forward_bf16_storage(img, w, cfg) - ref)
    err = np.abs(got - ref).max()
    print(f"{name}: bf16 max err {err:.4f}, bf16 storage alone {storage.max():.4f} (|ref| max {np.abs(ref).max():.3f})")
    atol, rtol = BENCH_TOL
    assert not (storage <= atol + rtol * np.abs(ref)).all()
    assert np.isfinite(got).all() and err <= 2.0 * storage.max()
    assert np.abs(got - fix).max() <= 2.0 * storage.max() + np.abs(fix - ref).max()


def _window_attention_ref(qkv, B, H, W, p, heads, dh):
    inner = heads * dh
    x = qkv[:, :3 * inner].astype(np.float64).reshape(B, H // p, p, W // p, p, 3, heads, dh)
    x = x.transpose(5, 0, 1, 3, 6, 2, 4, 7).reshape(3, -1, heads, p * p, dh)    # (q|k|v) (b x y) h (p1 p2) d
    o = to.softmax_attention(x[0], x[1], x[2]) if dh == to.DIM_HEAD else None
    if o is None:
        s = x[0] @ np.swapaxes(x[1], -1, -2) * dh ** -0.5
        a = np.exp(s - s.max(-1, keepdims=True))
        o = (a / a.sum(-1, keepdims=True)) @ x[2]
    return o.reshape(B, H // p, W // p, heads, p, p, dh).transpose(0, 1, 4, 2, 5, 3, 6).reshape(B * H * W, inner)


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("p,gy,gx", [(2, 3, 5), (4, 2, 1), (7, 2, 3), (8, 1, 2), (9, 2, 1)])
def test_op_window_attention_against_numpy(lib, precision, p, gy, gx):
    """Windows of 4, 16, 49, 64 and 81 tokens (81: two query tiles and two key blocks) on non-square window grids; the q|k|v rows
    are read in place (pitch wider than q|k|v), the output rows written pixel-major.  bf16 runs the windowed flash kernel, fp32
    the permuted materialised-scores path."""
    from vit_tensorflow_b200 import _lib
    B, heads, dh = 2, 2, 64
    H, W = gy * p, gx * p
    rng = np.random.default_rng(p * 100 + gy * 10 + gx)
    qkv = rng.standard_normal((B * H * W, 3 * heads * dh + 64)).astype(np.float32)
    _lib.last_attention_path()
    got, _ = _lib.op_window_attention(qkv, H, W, p, heads, dh, precision=precision)
    assert _lib.last_attention_path() == ("flash" if precision == "bf16" else "simt")
    ref = _window_attention_ref(qkv, B, H, W, p, heads, dh)
    atol, rtol = (1e-4, 1e-4) if precision == "fp32" else (2e-2, 2e-2)
    _within(got.astype(np.float64), ref, atol, rtol)


def test_op_window_attention_fallback_in_bf16(lib):
    """A head width the flash kernel refuses (32) takes the permuted materialised-scores path in bf16 too."""
    from vit_tensorflow_b200 import _lib
    B, p, H, W, heads, dh = 1, 3, 6, 9, 2, 32
    qkv = np.random.default_rng(5).standard_normal((B * H * W, 3 * heads * dh)).astype(np.float32)
    got, _ = _lib.op_window_attention(qkv, H, W, p, heads, dh, precision="bf16")
    assert _lib.last_attention_path() != "flash"
    _within(got.astype(np.float64), _window_attention_ref(qkv, B, H, W, p, heads, dh), 2e-2, 2e-2)


@pytest.mark.parametrize("name", ["twins_p9_wide", "twins_p7"])
def test_twins_bf16_profile_flash_and_no_fallbacks(lib, name):
    """One profiled bf16 forward: one flash launch per local and per global attention (the materialised-scores paths launch three
    and more), the only launches of the "other" class are the four PEGs (a GEMM on the SIMT fallback or a window permutation would
    be counted there too, for widths 40 / 72 as well), and one LayerNorm-folded GELU fc1 per MLP."""
    from vit_tensorflow_b200 import _lib
    cfg = to.make_config(**to.SMALL[name])
    w = to.stress_weights(cfg, to.WEIGHT_SEED)
    img = to.make_image(cfg, to.BATCH, to.IMAGE_SEED)
    m = _model(cfg, w, "bf16")
    m(img)
    m.profile(True)
    m.profile_read(reset=True)
    _lib.last_attention_path()
    got = m(img).numpy().astype(np.float64)
    prof = m.profile_read(reset=True)
    m.profile(False)
    layers = [(st < 3) for st in range(4) for _ in to.layer_prefixes(cfg, st)]
    n_local, n_global = sum(layers), len(layers)
    assert _lib.last_attention_path() == "flash"
    assert prof["attention"]["launches"] == n_local + n_global, prof
    assert prof["other"]["launches"] == 4, prof
    assert prof["gemm_wgmma_gelu"]["launches"] == n_local + n_global, prof
    _within(got, to.forward(img, w, cfg), BF16_ATOL, BF16_RTOL)


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_twins_image_sizes_and_refusals(lib, precision):
    """One handle serves 224^2, 448^2 and 224 x 448 images (its arena grows; no position embedding limits it).  Sizes that break
    a shape rule raise ValueError naming the stage and the sizes (stage 4 keeps its 14 x 14 map at 224^2 and a global_k of 10,
    so that a small image can break the VALID rule)."""
    cfg = to.make_config(image_size=224, num_classes=7, s1_emb_dim=64, s2_emb_dim=64, s3_emb_dim=128, s3_depth=1, s4_emb_dim=128,
                         s4_depth=1, s4_patch_size=1, s4_global_k=10)
    w = to.stress_weights(cfg, 3)
    m = _model(cfg, w, precision)
    atol, rtol = (FP32_ATOL, FP32_RTOL) if precision == "fp32" else (BF16_ATOL, BF16_RTOL)
    for h, wd, batch in ((224, 224, 2), (448, 448, 1), (224, 448, 2), (224, 224, 1)):
        img = to.make_image(cfg, batch, h + wd, h, wd)
        got = m(img)
        assert got.shape == (batch, 7)
        _within(np.asarray(got, np.float64), to.forward(img, w, cfg), atol, rtol)
    for h, wd, msg in ((230, 224, "stage 1: the 230 x 224 map is not divisible by patch_size 4"),
                       (220, 224, "stage 1: the 55 x 56 map is not divisible by local_patch_size 7"),
                       (112, 224, "stage 4: the 7 x 14 map is smaller than global_k 10")):
        with pytest.raises(ValueError, match=msg):
            m(to.make_image(cfg, 1, 0, h, wd))


def test_twins_training_and_dropout_rule(lib):
    """No BatchNorm: with dropout = 0 training=True computes what training=False does; with dropout > 0 only training=True is
    refused, as for ViT."""
    from vit_tensorflow_b200 import _lib
    cfg = to.make_config(**to.SMALL["twins_small"])
    w = to.stress_weights(cfg, 2)
    img = to.make_image(cfg, 2, 3)
    m = _model(cfg, w, "bf16")
    assert np.array_equal(m(img), m(img, training=False)) and np.array_equal(m(img, training=True, mask=None), m(img))
    md = _model(cfg, w, "bf16", dropout=0.1)
    with pytest.raises(NotImplementedError):
        md(img)
    assert np.array_equal(md(img, training=False), m(img))
    with pytest.raises(_lib.VbError, match="whole forward only"):
        m.forward_head(np.zeros((1, 4, 128), np.float32))
    with pytest.raises(_lib.VbError):
        m.forward_embed(img)


def test_twins_graph_replay_and_batch_independence(lib):
    import torch
    cfg = to.make_config(**to.BENCH["twins_readme"])
    w = to.stress_weights(cfg, 7)
    m = _model(cfg, w, "bf16")
    B = 8
    img = torch.from_numpy(to.make_image(cfg, B, 8)).cuda()
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

"""NesT (reference nest.py) on the H100 engine: fp32 and bf16 against the float64 spec and the reference-code fixtures
(tests/golden/nest_*__refshim.npz, tests/golden/make_nest_golden.py), the two tools/nest_bench.py configurations at their own size,
vb_op_block_attention and vb_op_nest_aggregate against numpy, the kernel classes of a profiled forward, one handle over several
image sizes and the refused ones, the training / dropout rule, graph replay and batch independence."""
import os

import numpy as np
import pytest

import nest_oracle as no

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
FP32_RTOL, FP32_ATOL = 1e-3, 1e-4
BF16_RTOL, BF16_ATOL = 4e-2, 6e-2            # the bf16 bound of test_gpu_models.py


def _model(cfg, w, precision, **kw):
    from vit_tensorflow_b200 import NesT
    m = NesT(**{**no.ctor_kwargs(cfg), **kw}, precision=precision)
    m.set_weights_dict(w)
    return m


def _within(got, want, atol, rtol):
    err = np.abs(got - want)
    assert np.isfinite(got).all() and (err <= atol + rtol * np.abs(want)).all(), f"max err {err.max():.3g}"


@pytest.mark.parametrize("gen", ["init_weights", "stress_weights"])
@pytest.mark.parametrize("name", sorted(no.SMALL))
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_nest_small_vs_spec_and_reference_fixture(lib, precision, name, gen):
    cfg = no.make_config(**no.SMALL[name])
    w = getattr(no, gen)(cfg, no.WEIGHT_SEED)
    img = no.make_image(cfg, no.BATCH, no.IMAGE_SEED)
    got = np.asarray(_model(cfg, w, precision)(img), np.float64)
    ref = no.forward(img, w, cfg)
    fix = np.load(os.path.join(GOLDEN, f"{name}__{gen}__refshim.npz"))["logits_ref_f64"]
    atol, rtol = (FP32_ATOL, FP32_RTOL) if precision == "fp32" else (BF16_ATOL, BF16_RTOL)
    assert got.shape == ref.shape
    for want in (ref, fix):
        _within(got, want, atol, rtol)


@pytest.mark.parametrize("name", sorted(no.BENCH))
def test_nest_bf16_at_config_size(lib, name):
    """The two tools/nest_bench.py models at full size (224^2) with stress weights, against the spec and the fixture.  The logits
    are held to the config-size bound where bf16 storage alone meets it, and otherwise to twice what bf16 storage alone costs
    (forward_bf16_storage: the convolutions' operands and results, the attention output and the stream after every sub-block
    rounded to bf16, all arithmetic in float64), as for Twins-SVT and LeViT."""
    cfg = no.make_config(**no.BENCH[name])
    img = no.make_image(cfg, no.BATCH, no.IMAGE_SEED)
    w = no.stress_weights(cfg, no.WEIGHT_SEED)
    got = _model(cfg, w, "bf16")(img).numpy().astype(np.float64)
    ref = no.forward(img, w, cfg)
    fix = np.load(os.path.join(GOLDEN, f"{name}__stress_weights__refshim.npz"))["logits_ref_f32"]
    storage = np.abs(no.forward_bf16_storage(img, w, cfg) - ref)
    err = np.abs(got - ref)
    print(f"{name}: bf16 max err {err.max():.4f}, bf16 storage alone {storage.max():.4f} (|ref| max {np.abs(ref).max():.3f})")
    assert np.isfinite(got).all()
    if (storage <= BF16_ATOL + BF16_RTOL * np.abs(ref)).all():
        _within(got, ref, BF16_ATOL, BF16_RTOL)
    else:
        assert err.max() <= 2.0 * storage.max()
    assert np.abs(got - fix).max() <= max(2.0 * storage.max(), BF16_ATOL + BF16_RTOL * np.abs(ref).max()) + np.abs(fix - ref).max()


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("dh", [32, 64, 24])
@pytest.mark.parametrize("bh,bw,gy,gx", [(2, 2, 3, 5), (7, 7, 2, 3), (8, 8, 1, 2), (9, 9, 2, 1), (14, 14, 2, 2), (14, 7, 1, 3)])
def test_op_block_attention_against_numpy(lib, precision, dh, bh, bw, gy, gx):
    """Blocks of 4, 49 and 64 tokens (one query tile), 81 and 196 (two and four query tiles and key blocks) and a rectangular 14 x 7
    block of 98, on non-square block grids; the q|k|v rows are read in place (pitch wider than q|k|v), the output rows written
    pixel-major.  bf16 with head width 32 or 64 runs the windowed flash kernel; head width 24 and every fp32 call the permuted
    materialised-scores path."""
    from vit_tensorflow_b200 import _lib
    B, heads = 2, 3
    H, W = gy * bh, gx * bw
    rng = np.random.default_rng(bh * 1000 + bw * 100 + gy * 10 + gx + dh)
    qkv = rng.standard_normal((B * H * W, 3 * heads * dh + 64)).astype(np.float32)
    _lib.last_attention_path()
    got, _ = _lib.op_block_attention(qkv, H, W, bh, bw, heads, dh, precision=precision)
    path = _lib.last_attention_path()
    if precision == "fp32":
        assert path == "simt"
    elif dh in (32, 64):
        assert path == "flash"
    else:
        assert path != "flash"
    ref = no.block_attention(qkv.astype(np.float64).reshape(B, H, W, -1), heads, dh, bh, bw).reshape(B * H * W, heads * dh)
    atol, rtol = (1e-4, 1e-4) if precision == "fp32" else (2e-2, 2e-2)
    _within(got.astype(np.float64), ref, atol, rtol)


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("H,W,C,blocks", [(14, 14, 192, (7, 7)), (28, 28, 96, (7, 7)), (8, 12, 40, (2, 3)), (7, 5, 64, None)])
def test_op_nest_aggregate_against_numpy(lib, precision, H, W, C, blocks):
    """LayerNorm on load (a large beta and negative gammas: the order of LayerNorm and max matters), the 3 x 3 stride-2 SAME max
    with the bottom / right pad (and both pads on odd sizes), the next level's position scalar on the true channels only; bf16 also
    returns the stored rows' statistics, which must be those of the stored values."""
    from vit_tensorflow_b200 import _lib
    B = 2
    rng = np.random.default_rng(H * 100 + W + C)
    x = (rng.standard_normal((B, H, W, C)) * 2.0 + 0.5).astype(np.float32)
    g = (1.0 + 0.3 * rng.standard_normal(C)).astype(np.float32)
    g[::3] *= -1.0
    b = (3.0 + 0.5 * rng.standard_normal(C)).astype(np.float32)
    pos = bh = bw = None
    if blocks is not None:
        bh, bw = blocks
        pos = rng.standard_normal(bh * bw).astype(np.float32)
    out, stats, _ = _lib.op_nest_aggregate(x, g, b, pos, bh or 1, bw or 1, precision=precision)
    xin = x.astype(np.float64) if precision == "fp32" else no.bf16_round(x.astype(np.float64))
    ref = no.aggregate_tail(xin, g.astype(np.float64), b.astype(np.float64), pos, bh or 1, bw or 1)
    assert out.shape == ref.shape
    atol, rtol = (1e-4, 1e-4) if precision == "fp32" else (5e-2, 2e-2)
    _within(out.astype(np.float64), ref, atol, rtol)
    if precision == "bf16":
        rows = out.reshape(-1, C).astype(np.float64)
        parts = np.zeros((-(-C // 64), rows.shape[0], 2))
        for j in range(parts.shape[0]):
            chunk = rows[:, 64 * j:64 * (j + 1)]
            parts[j, :, 0], parts[j, :, 1] = chunk.sum(1), (chunk * chunk).sum(1)
        _within(stats.astype(np.float64), parts, 1e-2, 1e-4)


@pytest.mark.parametrize("name", ["nest_readme_small", "nest_dh64"])
def test_nest_bf16_profile_flash_and_no_fallbacks(lib, name):
    """One profiled bf16 forward: exactly one flash attention launch per Transformer block and no window permutation, no GEMM on the
    SIMT fallback (either would add to the "other" class, which holds just the level-0 position add and one aggregation tail per
    Aggregate), and one LayerNorm-folded GELU fc1 per MLP."""
    from vit_tensorflow_b200 import _lib
    cfg = no.make_config(**no.SMALL[name])
    w = no.stress_weights(cfg, no.WEIGHT_SEED)
    img = no.make_image(cfg, no.BATCH, no.IMAGE_SEED)
    m = _model(cfg, w, "bf16")
    m(img)
    m.profile(True)
    m.profile_read(reset=True)
    _lib.last_attention_path()
    got = m(img).numpy().astype(np.float64)
    prof = m.profile_read(reset=True)
    m.profile(False)
    levels = no.plan(cfg)["levels"]
    blocks = sum(lv["depth"] for lv in levels)
    assert blocks > 0
    assert _lib.last_attention_path() == "flash"
    assert prof["attention"]["launches"] == blocks, prof
    assert prof["other"]["launches"] == 1 + sum(lv["aggregate"] for lv in levels), prof
    assert prof["gemm_wgmma_gelu"]["launches"] == blocks, prof
    _within(got, no.forward(img, w, cfg), BF16_ATOL, BF16_RTOL)


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_nest_image_sizes_and_refusals(lib, precision):
    """One handle serves 224^2, 192^2 and 224 x 112 images (rectangular 14 x 7 blocks at the first level; its arena grows).  Sizes
    that break a shape rule raise ValueError naming the level, the map and the rule."""
    cfg = no.make_config(image_size=224, patch_size=4, dim=64, heads=2, num_hierarchies=3, block_repeats=1, num_classes=7)
    w = no.stress_weights(cfg, 3)
    m = _model(cfg, w, precision)
    atol, rtol = (FP32_ATOL, FP32_RTOL) if precision == "fp32" else (BF16_ATOL, BF16_RTOL)
    for h, wd, batch in ((224, 224, 2), (192, 192, 1), (224, 112, 2), (224, 224, 1)):
        img = no.make_image(cfg, batch, h + wd, h, wd)
        got = m(img)
        assert got.shape == (batch, 7)
        _within(np.asarray(got, np.float64), no.forward(img, w, cfg), atol, rtol)
    for h, wd, msg in ((226, 224, "NesT: the 226 x 224 image is not divisible by patch_size 4"),
                       (224, 216, "NesT level 0: the 56 x 54 map is not divisible into 4 x 4 blocks"),
                       (256, 256, "NesT level 0: the 64 x 64 map has blocks of 16 x 16 tokens, more than seq_len 196 positions")):
        with pytest.raises(ValueError, match=msg):
            m(no.make_image(cfg, 1, 0, h, wd))


def test_nest_training_and_dropout_rule(lib):
    """No BatchNorm: with dropout = 0 training=True computes what training=False does; with dropout > 0 only training=True is
    refused, as for Twins-SVT.  The stage entries refuse a NesT handle."""
    from vit_tensorflow_b200 import _lib
    cfg = no.make_config(**no.SMALL["nest_readme_small"])
    w = no.stress_weights(cfg, 2)
    img = no.make_image(cfg, 2, 3)
    m = _model(cfg, w, "bf16")
    assert np.array_equal(m(img), m(img, training=False)) and np.array_equal(m(img, training=True, mask=None), m(img))
    md = _model(cfg, w, "bf16", dropout=0.1)
    with pytest.raises(NotImplementedError):
        md(img)
    assert np.array_equal(md(img, training=False), m(img))
    with pytest.raises(_lib.VbError, match="whole forward only"):
        m.forward_head(np.zeros((1, 4, m._cfg.dim), np.float32))
    with pytest.raises(_lib.VbError):
        m.forward_embed(img)


def test_nest_graph_replay_and_batch_independence(lib):
    import torch
    cfg = no.make_config(**no.BENCH["nest_readme"])
    w = no.stress_weights(cfg, 7)
    m = _model(cfg, w, "bf16")
    B = 8
    img = torch.from_numpy(no.make_image(cfg, B, 8)).cuda()
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

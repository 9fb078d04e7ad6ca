"""CvT (reference cvt.py) on the H100 engine: fp32 and bf16 against the float64 spec and the reference-code fixtures
(tests/golden/cvt_*__refshim.npz, tests/golden/make_cvt_golden.py), the two tools/cvt_bench.py configurations at their own size,
vb_op_dwconv against numpy, the kernel classes of a profiled forward, one handle over several image sizes, the training=False
rule, the stage refusals, graph replay and batch independence."""
import os

import numpy as np
import pytest

import cvt_oracle as co

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
FP32_RTOL, FP32_ATOL = 1e-3, 1e-4
BF16_RTOL, BF16_ATOL = 4e-2, 6e-2            # the bf16 bound of test_gpu_models.py
BENCH_TOL = (6.0e-2, 1.5e-2)                 # (atol, rtol): the config-size bound of test_gpu_cct.py


def _model(cfg, w, precision):
    from vit_tensorflow_b200 import from_config
    m = from_config(cfg, precision=precision)
    m.set_weights_dict(w)
    return m


def _blocks(cfg):
    return sum(st["depth"] for st in co.stages(cfg))


@pytest.mark.parametrize("gen", ["init_weights", "stress_weights"])
@pytest.mark.parametrize("name", sorted(co.SMALL))
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_cvt_small_vs_spec_and_reference_fixture(lib, precision, name, gen):
    cfg = co.make_config(**co.SMALL[name])
    w = getattr(co, gen)(cfg, co.WEIGHT_SEED)
    img = co.make_image(cfg, co.BATCH, co.IMAGE_SEED)
    got = np.asarray(_model(cfg, w, precision)(img, training=False), np.float64)
    ref = co.forward(img, w, cfg)
    fix = np.load(os.path.join(GOLDEN, f"{name}__{gen}__refshim.npz"))["logits_ref_f64"]
    atol, rtol = (FP32_ATOL, FP32_RTOL) if precision == "fp32" else (BF16_ATOL, BF16_RTOL)
    assert got.shape == ref.shape and np.isfinite(got).all()
    for want in (ref, fix):
        assert (np.abs(got - want) <= atol + rtol * np.abs(want)).all(), f"max err {np.abs(got - want).max():.3g}"


@pytest.mark.parametrize("name", sorted(co.BENCH))
def test_cvt_bf16_at_config_size(lib, name):
    """The two tools/cvt_bench.py models at full size (224^2) with stress weights, against the spec and the fixture."""
    cfg = co.make_config(**co.BENCH[name])
    img = co.make_image(cfg, co.BATCH, co.IMAGE_SEED)
    w = co.stress_weights(cfg, co.WEIGHT_SEED)
    got = _model(cfg, w, "bf16")(img, training=False).numpy().astype(np.float64)
    ref = co.forward(img, w, cfg)
    fix = np.load(os.path.join(GOLDEN, f"{name}__stress_weights__refshim.npz"))["logits_ref_f32"]
    atol, rtol = BENCH_TOL
    err = np.abs(got - ref)
    print(f"{name}: bf16 max err {err.max():.4f} (|ref| max {np.abs(ref).max():.3f})")
    assert np.isfinite(got).all() and (err <= atol + rtol * np.abs(ref)).all(), f"max err {err.max():.3g}"
    assert (np.abs(got - fix) <= atol + rtol * np.abs(fix)).all()


def _dwconv_ref(x, g, b, wq, bnq, wkv, bnkv, s):
    y = co.layer_norm(x, g, b)
    bn = lambda t, p: (t - p[2]) / np.sqrt(p[3] + co.BN_EPS) * p[0] + p[1]   # noqa: E731
    return bn(co.dwconv_same(y, wq, 1), bnq), bn(co.dwconv_same(y, wkv, s), bnkv)


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("k", [1, 3, 5, 7])
@pytest.mark.parametrize("s", [1, 2])
@pytest.mark.parametrize("H,W,C", [(13, 9, 40), (14, 16, 64), (8, 7, 72)])
def test_op_dwconv_against_numpy(lib, precision, k, s, H, W, C):
    """The LayerNorm applied on load (bf16: from the rows' statistics; fp32: a separate LayerNorm), both depthwise convolutions with
    their BatchNormalizations folded, and the SAME halo: the padding is zeros of the NORMALISED map (a large LayerNorm beta makes
    LN(0) != 0 visible at every border)."""
    from vit_tensorflow_b200 import _lib
    rng = np.random.default_rng(k * 100 + s * 10 + H)
    B = 2
    x = (rng.standard_normal((B, H, W, C)) * 2 + 0.5).astype(np.float32)
    g = (1 + 0.2 * rng.standard_normal(C)).astype(np.float32)
    b = (1.5 + 0.2 * rng.standard_normal(C)).astype(np.float32)
    wq, wkv = (rng.standard_normal((k, k, 1, C)).astype(np.float32) / k for _ in range(2))
    bnq, bnkv = (np.stack([1 + 0.2 * rng.standard_normal(C), 0.2 * rng.standard_normal(C), 0.2 * rng.standard_normal(C),
                           rng.uniform(0.5, 2.0, C)]).astype(np.float32) for _ in range(2))
    q, kv, _ = _lib.op_dwconv(x, g, b, wq, bnq, wkv, bnkv, s, precision=precision)
    rq, rkv = _dwconv_ref(*(a.astype(np.float64) for a in (x, g, b, wq, bnq, wkv, bnkv)), s)
    assert q.shape == rq.shape and kv.shape == rkv.shape == (B, -(-H // s), -(-W // s), C)
    atol, rtol = (1e-4, 1e-4) if precision == "fp32" else (3e-2, 2e-2)
    for got, ref in ((q, rq), (kv, rkv)):
        assert (np.abs(got - ref) <= atol + rtol * np.abs(ref)).all(), f"max err {np.abs(got - ref).max():.3g}"


@pytest.mark.parametrize("name", ["cvt_widths", "cvt_odd52"])
def test_cvt_bf16_profile_flash_dwconv_and_fc1(lib, name):
    """One profiled bf16 forward: one flash attention launch per block (the materialised-scores paths launch three), the only
    launches of the "other" class are the depthwise convolutions, one per block (a GEMM that fell back to the SIMT kernel would be
    counted there too, for widths like 40 / 72 as well), and one LayerNorm-folded GELU fc1 per block."""
    from vit_tensorflow_b200 import _lib
    cfg = co.make_config(**co.SMALL[name])
    w = co.stress_weights(cfg, co.WEIGHT_SEED)
    img = co.make_image(cfg, co.BATCH, co.IMAGE_SEED)
    m = _model(cfg, w, "bf16")
    m(img, training=False)
    m.profile(True)
    m.profile_read(reset=True)
    _lib.last_attention_path()
    got = m(img, training=False).numpy().astype(np.float64)
    prof = m.profile_read(reset=True)
    m.profile(False)
    blocks = _blocks(cfg)
    assert _lib.last_attention_path() == "flash"
    assert prof["attention"]["launches"] == blocks, prof
    assert prof["other"]["launches"] == blocks, prof
    assert prof["gemm_wgmma_gelu"]["launches"] == blocks, prof
    ref = co.forward(img, w, cfg)
    assert (np.abs(got - ref) <= BF16_ATOL + BF16_RTOL * np.abs(ref)).all(), f"max err {np.abs(got - ref).max():.3g}"


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_cvt_image_sizes_training_rule_and_refusals(lib, precision):
    """One handle serves a 224^2 image and then a non-square 200 x 232 one (its arena grows, no position embedding limits it)."""
    from vit_tensorflow_b200 import _lib
    cfg = co.make_config(image_size=224, num_classes=7, s1_emb_dim=64, s1_depth=1, s2_emb_dim=64, s2_heads=2, s2_depth=1,
                         s3_emb_dim=128, s3_heads=2, s3_depth=1)
    w = co.stress_weights(cfg, 3)
    m = _model(cfg, w, precision)
    atol, rtol = (FP32_ATOL, FP32_RTOL) if precision == "fp32" else (BF16_ATOL, BF16_RTOL)
    for h, wd, batch in ((224, 224, 2), (200, 232, 3), (224, 224, 1)):
        img = co.make_image(cfg, batch, h + wd, h, wd)
        got = m(img, training=False)
        ref = co.forward(img, w, cfg)
        assert got.shape == (batch, 7)
        assert (np.abs(got - ref) <= atol + rtol * np.abs(ref)).all(), f"{h}x{wd}: max err {np.abs(got - ref).max():.3g}"
    for training in (True, None):
        with pytest.raises(NotImplementedError, match="training=False"):
            m(img, training=training)
    with pytest.raises(_lib.VbError, match="whole forward only"):
        m.forward_head(np.zeros((1, 4, 128), np.float32))
    with pytest.raises(_lib.VbError):
        m.forward_embed(img)


def test_cvt_graph_replay_and_batch_independence(lib):
    import torch
    cfg = co.make_config(**co.BENCH["cvt_readme"])
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
    single = m(img[:1].cpu().numpy(), training=False)
    assert np.array_equal(single, outs[0][:1].cpu().numpy())
    half = m(img[3:7].cpu().numpy(), training=False)
    assert np.array_equal(half, outs[0][3:7].cpu().numpy())

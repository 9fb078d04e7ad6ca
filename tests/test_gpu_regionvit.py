"""RegionViT (reference regionvit.py) on the H100 engine: fp32 and bf16 against the float64 spec and the reference-code fixtures
(tests/golden/regionvit_*__refshim.npz, tests/golden/make_regionvit_golden.py), the two tools/regionvit_bench.py configurations at
their own size, vb_op_r2l_attention against numpy, the kernel classes of a profiled forward, one handle over several image sizes
and the refused ones, the training / dropout rule, graph replay and batch independence."""
import os

import numpy as np
import pytest

import regionvit_oracle as ro

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
FP32_RTOL, FP32_ATOL = 1e-3, 1e-4
BF16_RTOL, BF16_ATOL = 4e-2, 6e-2            # the bf16 bound of test_gpu_models.py


def _model(cfg, w, precision, **kw):
    from vit_tensorflow_b200 import RegionViT
    m = RegionViT(**{**ro.ctor_kwargs(cfg), **kw}, precision=precision)
    m.set_weights_dict(w)
    return m


def _within(got, want, atol, rtol):
    err = np.abs(got - want)
    assert np.isfinite(got).all() and (err <= atol + rtol * np.abs(want)).all(), f"max err {err.max():.3g}"


@pytest.mark.parametrize("gen", ["init_weights", "stress_weights"])
@pytest.mark.parametrize("name", sorted(ro.SMALL))
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_regionvit_small_vs_spec_and_reference_fixture(lib, precision, name, gen):
    cfg = ro.make_config(**ro.SMALL[name])
    w = getattr(ro, gen)(cfg, ro.WEIGHT_SEED)
    img = ro.make_image(cfg, ro.BATCH, ro.IMAGE_SEED)
    got = np.asarray(_model(cfg, w, precision)(img), np.float64)
    ref = ro.forward(img, w, cfg)
    fix = np.load(os.path.join(GOLDEN, f"{name}__{gen}__refshim.npz"))["logits_ref_f64"]
    atol, rtol = (FP32_ATOL, FP32_RTOL) if precision == "fp32" else (BF16_ATOL, BF16_RTOL)
    assert got.shape == ref.shape
    for want in (ref, fix):
        _within(got, want, atol, rtol)


@pytest.mark.parametrize("name", sorted(ro.BENCH))
def test_regionvit_bf16_at_config_size(lib, name):
    """The two tools/regionvit_bench.py models at full size (224^2) with stress weights, against the spec and the fixture: held to
    the config-size bound where bf16 storage alone meets it, and otherwise to twice what bf16 storage alone costs
    (forward_bf16_storage), as for NesT."""
    cfg = ro.make_config(**ro.BENCH[name])
    img = ro.make_image(cfg, ro.BATCH, ro.IMAGE_SEED)
    w = ro.stress_weights(cfg, ro.WEIGHT_SEED)
    got = _model(cfg, w, "bf16")(img).numpy().astype(np.float64)
    ref = ro.forward(img, w, cfg)
    fix = np.load(os.path.join(GOLDEN, f"{name}__stress_weights__refshim.npz"))["logits_ref_f32"]
    storage = np.abs(ro.forward_bf16_storage(img, w, cfg) - ref)
    err = np.abs(got - ref)
    print(f"{name}: bf16 max err {err.max():.4f}, bf16 storage alone {storage.max():.4f} (|ref| max {np.abs(ref).max():.3f})")
    assert np.isfinite(got).all()
    if (storage <= BF16_ATOL + BF16_RTOL * np.abs(ref)).all():
        _within(got, ref, BF16_ATOL, BF16_RTOL)
    else:
        assert err.max() <= 2.0 * storage.max()
    assert np.abs(got - fix).max() <= max(2.0 * storage.max(), BF16_ATOL + BF16_RTOL * np.abs(ref).max()) + np.abs(fix - ref).max()


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("ws,wh,ww,rh,rw", [(7, 7, 7, 2, 3), (14, 14, 14, 1, 2), (7, 4, 7, 2, 1), (7, 2, 2, 3, 2), (7, 1, 1, 2, 2),
                                           (14, 7, 7, 1, 1), (40, 2, 3, 1, 2)])
def test_op_r2l_attention_against_numpy(lib, precision, ws, wh, ww, rh, rw):
    """Windows of 7 x 7 (50 tokens: one query tile), 14 x 14 (197: four query tiles and key blocks), rectangular 4 x 7, 2 x 2 and
    1 x 1 with the table of pitch 13, a 7 x 7 window under window_size 14's table, on non-square region grids; the q|k|v rows are
    read in place at a pitch wider than q|k|v and the output written at a pitch wider than the heads.  bf16 runs the R2L flash
    kernel; every fp32 call, and window_size 40 (a (2 ws - 1)^2 table past the kernel's shared-memory table), gather the windows
    and run the materialised-scores path."""
    from vit_tensorflow_b200 import _lib
    B, heads, dh = 2, 4, 32
    lh, lw = rh * wh, rw * ww
    rng = np.random.default_rng(ws * 1000 + wh * 100 + ww * 10 + rh + rw)
    rows = B * (lh * lw + rh * rw)
    qkv = rng.standard_normal((rows, 3 * heads * dh + 64)).astype(np.float32)
    table = rng.standard_normal(((2 * ws - 1) ** 2, heads)).astype(np.float32)
    _lib.last_attention_path()
    got, _ = _lib.op_r2l_attention(qkv, B, lh, lw, rh, rw, heads, dh, table, ws, precision=precision, ldo=heads * dh + 32)
    path = _lib.last_attention_path()
    assert path == ("flash" if precision == "bf16" and ws < 33 else "simt"), path
    q64 = qkv.astype(np.float64)
    Ml = B * lh * lw
    ol, orr = ro.r2l_attention(q64[:Ml].reshape(B, lh, lw, -1), q64[Ml:].reshape(B, rh, rw, -1), heads, dh, table.astype(np.float64), ws)
    ref = np.concatenate([ol.reshape(Ml, -1), orr.reshape(-1, heads * dh)], 0)
    atol, rtol = (1e-4, 1e-4) if precision == "fp32" else (2e-2, 2e-2)
    _within(got[:, :heads * dh].astype(np.float64), ref, atol, rtol)
    assert not got[:, heads * dh:].any()                                 # columns past the heads are left as they were


@pytest.mark.parametrize("name", ["regionvit_readme_small", "regionvit_3conv_peg"])
def test_regionvit_bf16_profile_flash_and_no_fallbacks(lib, name):
    """One profiled bf16 forward: exactly two flash attention launches per R2L layer (the regional one and the R2L one), no window
    gather or scatter and no GEMM on the SIMT fallback (either would add to the "other" class, which holds just one PEG per stage
    that has one), and one LayerNorm-folded GELU fc1 per layer (the 3-conv tokenizer's GELU is applied on load, not by a GEMM)."""
    from vit_tensorflow_b200 import _lib
    cfg = ro.make_config(**ro.SMALL[name])
    w = ro.stress_weights(cfg, ro.WEIGHT_SEED)
    img = ro.make_image(cfg, ro.BATCH, ro.IMAGE_SEED)
    m = _model(cfg, w, "bf16")
    m(img)
    m.profile(True)
    m.profile_read(reset=True)
    _lib.last_attention_path()
    got = m(img).numpy().astype(np.float64)
    prof = m.profile_read(reset=True)
    m.profile(False)
    layers = sum(ro.depths(cfg))
    assert layers > 0
    assert _lib.last_attention_path() == "flash"
    assert prof["attention"]["launches"] == 2 * layers, prof
    assert prof["other"]["launches"] == (3 if cfg["use_peg"] else 0), prof
    assert prof["gemm_wgmma_gelu"]["launches"] == layers, prof
    _within(got, ro.forward(img, w, cfg), BF16_ATOL, BF16_RTOL)


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_regionvit_image_sizes_and_refusals(lib, precision):
    """One handle serves 224^2, 112^2, 56^2, 448^2 and 28 x 56 images (windows from 7 x 7 down to 1 x 1, and 4 x 7; its arena
    grows).  Sizes the reference cannot run raise its assert messages, or ValueError naming the stage, both maps and the rule."""
    cfg = ro.make_config(dim=(32, 64, 64, 96), depth=1, num_classes=7)
    w = ro.stress_weights(cfg, 3)
    m = _model(cfg, w, precision)
    atol, rtol = (FP32_ATOL, FP32_RTOL) if precision == "fp32" else (BF16_ATOL, BF16_RTOL)
    for h, wd, batch in ((224, 224, 2), (112, 112, 1), (56, 56, 2), (448, 448, 1), (28, 56, 2), (224, 224, 1)):
        img = ro.make_image(cfg, batch, h + wd, h, wd)
        got = m(img)
        assert got.shape == (batch, 7)
        _within(np.asarray(got, np.float64), ro.forward(img, w, cfg), atol, rtol)
    with pytest.raises(AssertionError, match="^height and width must be divisible by region patch size$"):
        m(ro.make_image(cfg, 1, 0, 224, 220))
    with pytest.raises(ValueError, match=r"^RegionViT stage 3: the 11 x 11 local map and the 2 x 2 region map do not make whole "
                                         r"windows \(the local map must be the region map times the window\)$"):
        m(ro.make_image(cfg, 1, 0, 168, 168))
    cfg8 = ro.make_config(dim=(32, 64, 64, 96), depth=1, num_classes=7, local_patch_size=8)
    m8 = _model(cfg8, ro.init_weights(cfg8, 3), precision)
    with pytest.raises(ValueError, match=r"^RegionViT stage 1: the 56 x 56 local map and the 4 x 4 region map make 14 x 14 windows, "
                                         r"larger than window_size 7"):
        m8(ro.make_image(cfg, 1, 0, 224, 224))


def test_regionvit_engine_size_check_matches_the_host(lib):
    """The engine checks the same rules itself (vb_forward below the host class), with the same words."""
    from vit_tensorflow_b200 import _lib
    cfg = ro.make_config(dim=(32, 64, 64, 96), depth=1, num_classes=7)
    m = _model(cfg, ro.init_weights(cfg, 1), "bf16")
    img = ro.make_image(cfg, 1, 0, 168, 168)
    out = np.empty((1, 7), np.float32)
    with pytest.raises(_lib.VbError, match=r"RegionViT stage 3: the 11 x 11 local map and the 2 x 2 region map do not make whole"):
        m.forward_raw(img.ctypes.data, _lib.MEM_HOST, 1, 168, 168, out.ctypes.data, _lib.MEM_HOST, None)


def test_regionvit_training_and_dropout_rule(lib):
    """No BatchNorm: training=True computes what training=False does; attn_dropout builds nothing in the reference and runs; with
    ff_dropout > 0 only training=True is refused.  The stage entries refuse a RegionViT handle."""
    from vit_tensorflow_b200 import _lib
    cfg = ro.make_config(**ro.SMALL["regionvit_readme_small"])
    w = ro.stress_weights(cfg, 2)
    img = ro.make_image(cfg, 2, 3)
    m = _model(cfg, w, "bf16")
    assert np.array_equal(m(img), m(img, training=False)) and np.array_equal(m(img, training=True, mask=None), m(img))
    ma = _model(cfg, w, "bf16", attn_dropout=0.3)
    assert np.array_equal(ma(img), m(img))
    md = _model(cfg, w, "bf16", ff_dropout=0.1)
    with pytest.raises(NotImplementedError):
        md(img)
    assert np.array_equal(md(img, training=False), m(img))
    with pytest.raises(_lib.VbError, match="whole forward only"):
        m.forward_head(np.zeros((1, 4, m._cfg.dim), np.float32))
    with pytest.raises(_lib.VbError):
        m.forward_embed(img)


def test_regionvit_graph_replay_and_batch_independence(lib):
    import torch
    cfg = ro.make_config(**ro.BENCH["regionvit_readme"])
    w = ro.stress_weights(cfg, 7)
    m = _model(cfg, w, "bf16")
    B = 8
    img = torch.from_numpy(ro.make_image(cfg, B, 8)).cuda()
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

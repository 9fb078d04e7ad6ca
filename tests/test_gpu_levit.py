"""LeViT (reference levit.py) on the H100 engine: fp32 and bf16 against the float64 spec and the reference-code fixtures
(tests/golden/levit_*__refshim.npz, tests/golden/make_levit_golden.py), the two tools/levit_bench.py configurations at their own
size, vb_op_attention_bias on the flash and materialised-scores branches, the distillation tuple, non-square images and the
refused sizes, the training=False rule, the stage refusals, graph replay and batch independence."""
import ctypes as C
import os

import numpy as np
import pytest

import levit_oracle as lo

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


def _split(out):
    return out if isinstance(out, tuple) else (out,)


@pytest.mark.parametrize("gen", ["init_weights", "stress_weights"])
@pytest.mark.parametrize("name", sorted(lo.SMALL))
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_levit_small_vs_spec_and_reference_fixture(lib, precision, name, gen):
    cfg = lo.make_config(**lo.SMALL[name])
    w = getattr(lo, gen)(cfg, lo.WEIGHT_SEED)
    img = lo.make_image(cfg, lo.BATCH, lo.IMAGE_SEED)
    got = [np.asarray(g, np.float64) for g in _split(_model(cfg, w, precision)(img, training=False))]
    ref = _split(lo.forward(img, w, cfg))
    z = np.load(os.path.join(GOLDEN, f"{name}__{gen}__refshim.npz"))
    fix = [z["logits_ref_f64"]] + ([z["distill_ref_f64"]] if "distill_ref_f64" in z.files else [])
    assert len(got) == len(ref) == len(fix)
    atol, rtol = (FP32_ATOL, FP32_RTOL) if precision == "fp32" else (BF16_ATOL, BF16_RTOL)
    for g, r, f in zip(got, ref, fix):
        assert g.shape == r.shape and np.isfinite(g).all()
        for want in (r, f):
            assert (np.abs(g - want) <= atol + rtol * np.abs(want)).all(), f"max err {np.abs(g - want).max():.3g}"


@pytest.mark.parametrize("name", sorted(lo.BENCH))
def test_levit_bf16_at_config_size(lib, name):
    """The two tools/levit_bench.py models at full size.  With to_out gammas of 0.2 x (1 + 0.2 N) the bf16 logits meet the
    config-size bound.  With the full stress weights (to_out gammas around 1) the stream of these 16- and 12-block models grows to
    logits of 20-40, and bf16 storage alone (forward_bf16_storage: only the 1x1 convolutions' operands and results rounded)
    already misses that bound; there the engine's error is held to twice that estimate instead."""
    cfg = lo.make_config(**lo.BENCH[name])
    img = lo.make_image(cfg, lo.BATCH, lo.IMAGE_SEED)
    w = lo.stress_weights(cfg, lo.WEIGHT_SEED, to_out_gamma=0.2)
    got = _model(cfg, w, "bf16")(img, training=False).numpy().astype(np.float64)
    ref = lo.forward(img, w, cfg)
    atol, rtol = BENCH_TOL
    err = np.abs(got - ref)
    print(f"{name}: to_out gamma 0.2: bf16 max err {err.max():.4f} (|ref| max {np.abs(ref).max():.3f})")
    assert np.isfinite(got).all() and (err <= atol + rtol * np.abs(ref)).all(), f"max err {err.max():.3g}"
    w = lo.stress_weights(cfg, lo.WEIGHT_SEED)
    got = _model(cfg, w, "bf16")(img, training=False).numpy().astype(np.float64)
    ref = lo.forward(img, w, cfg)
    err = np.abs(got - ref).max()
    storage = np.abs(lo.forward_bf16_storage(img, w, cfg) - ref).max()
    print(f"{name}: to_out gamma 1: bf16 max err {err:.4f}, bf16 storage alone {storage:.4f} (|ref| max {np.abs(ref).max():.3f})")
    assert np.isfinite(got).all() and err <= 2.0 * storage


@pytest.mark.parametrize("name", ["levit_odd", "levit_192"])
def test_levit_bf16_widths_off_64_run_every_gemm_on_wgmma(lib, name):
    """Channel widths that are not multiples of 64 (40 / 56, 192 / 288) are carried zero-padded to them, so every GEMM of the
    forward runs on the wgmma kernel: the only launches of the profile's "other" class are the shrink blocks' even-pixel gathers
    (a GEMM that fell back to the SIMT kernel would be counted there too)."""
    cfg = lo.make_config(**lo.SMALL[name])
    w = lo.stress_weights(cfg, lo.WEIGHT_SEED)
    img = lo.make_image(cfg, lo.BATCH, lo.IMAGE_SEED)
    m = _model(cfg, w, "bf16")
    m(img, training=False)
    m.profile(True)
    m.profile_read(reset=True)
    got = m(img, training=False).numpy().astype(np.float64)
    prof = m.profile_read(reset=True)
    m.profile(False)
    shrinks = cfg["stages"] - 1
    assert prof["other"]["launches"] == shrinks, prof
    blocks = len(lo.blocks(cfg))
    assert prof["gemm_wgmma_gelu"]["launches"] == blocks                 # fc1 (hard-swish epilogue) of every block
    ref = lo.forward(img, w, cfg)
    assert (np.abs(got - ref) <= BF16_ATOL + BF16_RTOL * np.abs(ref)).all(), f"max err {np.abs(got - ref).max():.3g}"


def _attention_ref(q, k, v, table, heads, dh, fmap, step, scale, gelu):
    """float64: softmax(q k^T * scale + table[idx] / scale) v, GELU; q [B, nq, heads*dh] etc."""
    from oracle import spec_numpy
    B, nq = q.shape[:2]
    qh = q.reshape(B, nq, heads, dh).transpose(0, 2, 1, 3)
    kh = k.reshape(B, -1, heads, dh).transpose(0, 2, 1, 3)
    vh = v.reshape(B, -1, heads, dh).transpose(0, 2, 1, 3)
    s = qh @ kh.transpose(0, 1, 3, 2) * scale + table[lo.pos_indices(fmap, step == 2)].transpose(2, 0, 1)[None] / scale
    p = np.exp(s - s.max(-1, keepdims=True))
    o = ((p / p.sum(-1, keepdims=True)) @ vh).transpose(0, 2, 1, 3).reshape(B, nq, heads * dh)
    return spec_numpy.gelu(o) if gelu else o


@pytest.mark.parametrize("precision,dh,path", [("bf16", 64, "flash"), ("bf16", 32, "mid_fused"), ("bf16", 48, "mid_fused"),
                                               ("fp32", 64, "simt"), ("fp32", 20, "simt")])
@pytest.mark.parametrize("fmap,step", [(14, 1), (14, 2), (7, 2), (9, 1), (4, 2)])
def test_op_attention_bias_branches(lib, precision, dh, path, fmap, step):
    from vit_tensorflow_b200 import _lib
    rng = np.random.default_rng(fmap * 10 + step + dh)
    B, heads = 3, 4
    nk, nq = fmap * fmap, (-(-fmap // step)) ** 2
    q, k, v = (rng.standard_normal((B, n, heads * dh)).astype(np.float32) for n in (nq, nk, nk))
    table = rng.standard_normal((nk, heads)).astype(np.float32)
    scale = 16 ** -0.5
    q *= 0.5
    _lib.last_attention_path()
    for gelu in (True, False):
        got, _ = _lib.op_attention_bias(q, k, v, table, heads, dh, fmap, step, scale, np.zeros((B, nq, heads * dh), np.float32),
                                        gelu_out=gelu, precision=precision)
        assert _lib.last_attention_path() == path
        ref = _attention_ref(*(x.astype(np.float64) for x in (q, k, v, table)), heads, dh, fmap, step, scale, gelu)
        atol, rtol = (1e-4, 1e-3) if precision == "fp32" else (3e-2, 3e-2)
        assert (np.abs(got - ref) <= atol + rtol * np.abs(ref)).all(), f"max err {np.abs(got - ref).max():.3g}"


def test_levit_distill_tuple_non_square_image_and_refusals(lib):
    from vit_tensorflow_b200 import LeViT, _lib
    cfg = lo.make_config(image_size=224, num_classes=9, dim=(64, 128), depth=1, heads=(2, 2), mlp_mult=2, stages=2,
                         num_distill_classes=4)
    w = lo.stress_weights(cfg, 3)
    m = _model(cfg, w, "fp32")
    img = lo.make_image(cfg, 2, 4, 210, 216)                           # the stem gives 14 x 14 for both
    out, dist = m(img, training=False)
    ref, rdist = lo.forward(img, w, cfg)
    assert out.shape == (2, 9) and dist.shape == (2, 4)
    np.testing.assert_allclose(out, ref, rtol=FP32_RTOL, atol=FP32_ATOL)
    np.testing.assert_allclose(dist, rdist, rtol=FP32_RTOL, atol=FP32_ATOL)
    with pytest.raises(_lib.VbError, match="14 x 14"):
        m(lo.make_image(cfg, 1, 5, 224, 240), training=False)
    for training in (True, None):
        with pytest.raises(NotImplementedError, match="training=False"):
            m(img, training=training)
    with pytest.raises(ValueError, match="image_size // 16"):
        LeViT(image_size=200, num_classes=3, dim=64, depth=1, heads=2, mlp_mult=2)
    with pytest.raises(_lib.VbError, match="whole forward only"):
        m.forward_head(np.zeros((1, 4, 128), np.float32))
    with pytest.raises(_lib.VbError):
        m.forward_embed(img)
    tok = np.zeros(128, np.float32)
    rc = m._lib.vb_forward_distill(m._h, img.ctypes.data_as(C.c_void_p), 0, 2, 210, 216, tok.ctypes.data_as(C.c_void_p),
                                   out.ctypes.data_as(C.c_void_p), dist.ctypes.data_as(C.c_void_p), 0, None)
    assert rc != 0 and b"no distillation token" in m._lib.vb_last_error(m._h)


def test_levit_graph_replay_and_batch_independence(lib):
    import torch
    cfg = lo.make_config(**lo.BENCH["levit_128s"])
    w = lo.stress_weights(cfg, 7)
    m = _model(cfg, w, "bf16")
    B = 8
    img = torch.from_numpy(lo.make_image(cfg, B, 8)).cuda()
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

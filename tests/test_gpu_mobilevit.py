"""MobileViT (reference mobile_vit.py) on the H100 engine: fp32 and bf16 against the float64 spec and the reference-code fixtures
(tests/golden/mobilevit_*__refshim.npz, tests/golden/make_mobilevit_golden.py), the README XS model and XXS at 256^2, batch 8;
vb_op_mv2_dwconv, the SiLU GEMM epilogue and vb_op_patch_attention against numpy; the training=False rule, the refused sizes and
stage entries, graph replay and batch independence."""
import os

import numpy as np
import pytest

import mobilevit_oracle as mo
from levit_oracle import bf16_round

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
# The whole-model bounds are relative to each case's own logit scale s = max |ref|: with the Keras initial weights the signal shrinks
# by orders of magnitude through the stem and the small cases' logits are 1.5e-5 to 4e-2, so an absolute bound would pass an all-zero
# output.  Measured on an H100 over the SMALL cases: fp32 at most 2.1e-6 s; bf16 at most 1.6 % of s with the initial weights and
# 0.3 % with the stress weights (bf16 rounds every stored activation by up to 2^-9 = 0.2 %, through ~30 layers in sequence).  The
# bounds are about five and three times those: max |err| <= 1e-5 s (fp32), 5e-2 s (bf16).  A case whose logits fall below
# SCALE_FLOOR fails instead of passing on a vanishing signal.
FP32_REL, BF16_REL = 1e-5, 5e-2
SCALE_FLOOR = 1e-6
# At config size (XS / XXS, 256^2) the logits pass through ~40 bf16-stored activations and ~30 folded BatchNorms in sequence.
# Measured on an H100: 2.4 % (XS) and 1.2 % (XXS) of max |ref| with the initial weights, at most 0.4 % with the stress weights; the
# bound is 8 %, about three times the largest.
BENCH_REL = 8e-2


def _model(cfg, w, precision):
    from vit_tensorflow_b200 import from_config
    m = from_config(cfg, precision=precision)
    m.set_weights_dict(w)
    return m


def _within(got, want, atol, rtol):
    err = np.abs(got - want)
    assert np.isfinite(got).all() and (err <= atol + rtol * np.abs(want)).all(), f"max err {err.max():.3g}"


@pytest.mark.parametrize("gen", ["init_weights", "stress_weights"])
@pytest.mark.parametrize("name", sorted(mo.SMALL))
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_mobilevit_small_vs_spec_and_reference_fixture(lib, precision, name, gen):
    cfg = mo.make_config(**mo.SMALL[name])
    w = getattr(mo, gen)(cfg, mo.WEIGHT_SEED)
    img = mo.make_image(cfg, mo.BATCH, mo.IMAGE_SEED)
    got = _model(cfg, w, precision)(img, training=False).numpy().astype(np.float64)
    ref = mo.forward(img, w, cfg)
    fix = np.load(os.path.join(GOLDEN, f"{name}__{gen}__refshim.npz"))["logits_ref_f64"]
    scale = np.abs(ref).max()
    bound = (FP32_REL if precision == "fp32" else BF16_REL) * scale
    print(f"{name} {gen} {precision}: max err {np.abs(got - ref).max():.3g} ({np.abs(got - ref).max() / scale:.2e} of |ref| max {scale:.3g})")
    assert scale >= SCALE_FLOOR, f"the case's logits ({scale:.3g}) are too small to test against"
    assert got.shape == ref.shape and np.isfinite(got).all()
    for want in (ref, fix):
        assert np.abs(got - want).max() <= bound, f"max err {np.abs(got - want).max():.3g} > {bound:.3g}"


@pytest.mark.parametrize("name", ["mobilevit_xs", "mobilevit_xxs"])
def test_mobilevit_bf16_at_config_size(lib, name):
    cfg = mo.make_config(**mo.BENCH[name])
    img = mo.make_image(cfg, 8, mo.IMAGE_SEED)
    for gen in (mo.init_weights, mo.stress_weights):
        w = gen(cfg, mo.WEIGHT_SEED)
        got = _model(cfg, w, "bf16")(img, training=False).numpy().astype(np.float64)
        ref = mo.forward(img, w, cfg)
        err, scale = np.abs(got - ref).max(), np.abs(ref).max()
        print(f"{name} {gen.__name__}: bf16 max err {err:.4g}, |ref| max {scale:.4g} ({err / scale:.2%})")
        assert scale >= SCALE_FLOOR and np.isfinite(got).all() and err <= BENCH_REL * scale


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("H,W,C,stride", [(9, 7, 16, 1), (9, 7, 16, 2), (8, 12, 72, 2), (16, 16, 384, 1), (5, 6, 384, 2), (32, 33, 72, 1)])
def test_op_mv2_dwconv_against_numpy(lib, precision, H, W, C, stride):
    """Odd and even maps, stride 1 and 2 (TF SAME pads the smaller half first), C off a multiple of 64 (pad channels written as
    zero in bf16) and a BatchNorm far from the identity."""
    from vit_tensorflow_b200 import _lib
    rng = np.random.default_rng(H * 1000 + W * 10 + C + stride)
    x = (1.5 * rng.standard_normal((2, H, W, C))).astype(np.float32)
    k = (rng.standard_normal((3, 3, 1, C)) / 3).astype(np.float32)
    bn = np.stack([1 + 0.3 * rng.standard_normal(C), 0.5 * rng.standard_normal(C), 0.5 * rng.standard_normal(C),
                   rng.uniform(0.3, 3.0, C)]).astype(np.float32)
    out, _ = _lib.op_mv2_dwconv(x, k, bn, stride, precision=precision)
    xin = x.astype(np.float64) if precision == "fp32" else bf16_round(x)
    w = {"b.gamma": bn[0], "b.beta": bn[1], "b.moving_mean": bn[2], "b.moving_variance": bn[3]}
    ref = mo.silu(mo._bn(mo._dwconv(xin, k.astype(np.float64), stride), {n: v.astype(np.float64) for n, v in w.items()}, "b"))
    assert out.shape[:3] == ref.shape[:3] == (2, -(-H // stride), -(-W // stride), C)[:3]
    if precision == "bf16":
        assert out.shape[3] == -(-C // 64) * 64 and (out[..., C:] == 0).all()
    atol, rtol = (1e-5, 1e-5) if precision == "fp32" else (2e-2, 1e-2)
    _within(out[..., :C].astype(np.float64), ref, atol, rtol)


@pytest.mark.parametrize("N", [256, 1536])
@pytest.mark.parametrize("folded", [False, True])
def test_silu_gemm_epilogue_against_numpy(lib, N, folded):
    """The wgmma GEMM's SiLU epilogue after the bias and after the folded LayerNorm (eps 1e-3), on the 128-wide tile (N = 256) and
    the 192-wide one (N = 1536)."""
    from vit_tensorflow_b200 import _lib
    M, K = 300, 192
    rng = np.random.default_rng(N + folded)
    a = bf16_round((rng.standard_normal((M, K)) + 0.5).astype(np.float32))
    wt = bf16_round((rng.standard_normal((N, K)) / np.sqrt(K)).astype(np.float32))
    bias = (0.5 * rng.standard_normal(N)).astype(np.float32)
    acc = a @ wt.T.astype(np.float64)
    if folded:
        ch = a.reshape(M, K // 64, 64).transpose(1, 0, 2)
        stats = np.stack([ch.sum(-1), (ch ** 2).sum(-1)], -1).astype(np.float32)
        c1 = wt.astype(np.float64).sum(1)
        mu = a.mean(1, keepdims=True)
        rstd = 1.0 / np.sqrt((a * a).mean(1, keepdims=True) - mu * mu + 1e-3)
        pre = rstd * (acc - mu * c1) + bias
        out, _, _ = _lib.op_gemm(a, wt, N, K, np.zeros((M, N), np.float32), bias=bias, ln_stats=stats, ln_c1=c1.astype(np.float32), silu=True)
    else:
        pre = acc + bias
        out, _, _ = _lib.op_gemm(a, wt, N, K, np.zeros((M, N), np.float32), bias=bias, silu=True)
    _within(out.astype(np.float64), mo.silu(pre), 1e-2, 1e-2)


def _patch_attention_ref(qkv, B, H, W, ph, pw, heads, dh, scale):
    x = qkv.astype(np.float64).reshape(B, H // ph, ph, W // pw, pw, -1).transpose(0, 2, 4, 1, 3, 5).reshape(B, ph * pw, -1, qkv.shape[1])
    HD = heads * dh
    q, k, v = (x[..., i * HD:(i + 1) * HD].reshape(B, ph * pw, -1, heads, dh).transpose(0, 1, 3, 2, 4) for i in range(3))
    s = q @ k.transpose(0, 1, 2, 4, 3) * scale
    p = np.exp(s - s.max(-1, keepdims=True))
    o = (p / p.sum(-1, keepdims=True)) @ v
    o = o.transpose(0, 1, 3, 2, 4).reshape(B, ph, pw, H // ph, W // pw, HD).transpose(0, 3, 1, 4, 2, 5)
    return o.reshape(B * H * W, HD)


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("H,W,ph,pw", [(4, 4, 2, 2), (8, 16, 2, 4), (16, 16, 2, 2), (24, 12, 2, 2), (64, 64, 2, 2), (32, 128, 2, 4)])
def test_op_patch_attention_against_numpy(lib, precision, H, W, ph, pw):
    """Groups of 4, 16, 64, 72, 1,024 and 512 tokens (one to sixteen query tiles), square and rectangular patches, 4 heads of 8
    widened to 32 with zero columns and scale 8^-0.5 as the engine runs them.  bf16 runs the windowed flash kernel on the dilated
    window; fp32 the permuted materialised-scores path."""
    from vit_tensorflow_b200 import _lib
    B, heads, dh, dm = 2, 4, 32, 8
    rng = np.random.default_rng(H * 100 + W + ph)
    qkv = np.zeros((B * H * W, 3 * heads * dh + 64), np.float32)
    for g in range(3):
        for h in range(heads):
            qkv[:, g * heads * dh + h * dh:g * heads * dh + h * dh + dm] = rng.standard_normal((B * H * W, dm))
    if precision == "bf16":
        qkv = bf16_round(qkv).astype(np.float32)
    _lib.last_attention_path()
    got, _ = _lib.op_patch_attention(qkv, H, W, ph, pw, heads, dh, scale=dm ** -0.5, precision=precision)
    assert _lib.last_attention_path() == ("flash" if precision == "bf16" else "simt")
    ref = _patch_attention_ref(qkv, B, H, W, ph, pw, heads, dh, dm ** -0.5)
    atol, rtol = (1e-4, 1e-4) if precision == "fp32" else (2e-2, 2e-2)
    _within(got.astype(np.float64), ref, atol, rtol)


def test_mobilevit_refusals(lib):
    from vit_tensorflow_b200 import _lib
    cfg = mo.make_config(**mo.SMALL["mobilevit_sq"])
    w = mo.stress_weights(cfg, 3)
    m = _model(cfg, w, "fp32")
    img = mo.make_image(cfg, 2, 4, 128, 64)                            # any size whose trunk maps divide by the patch runs
    ref = mo.forward(img, w, cfg)
    assert np.abs(m(img, training=False) - ref).max() <= FP32_REL * np.abs(ref).max()
    for training in (True, None):
        with pytest.raises(NotImplementedError, match="training=False"):
            m(img, training=training)
    with pytest.raises(ValueError, match="MobileViT stage 3"):
        m(mo.make_image(cfg, 1, 5, 96, 64), training=False)
    rc = m._lib.vb_forward(m._h, img.ctypes.data, 0, 1, 96, 64, np.zeros((1, 10), np.float32).ctypes.data, 0, None)
    assert rc != 0 and b"MobileViT stage 3" in m._lib.vb_last_error(m._h)
    with pytest.raises(_lib.VbError, match="whole forward only"):
        m.forward_head(np.zeros((1, 4, 96), np.float32))
    with pytest.raises(_lib.VbError, match="whole forward only"):
        m.forward_embed(img)


def test_mobilevit_graph_replay_and_batch_independence(lib):
    import torch
    cfg = mo.make_config(**mo.BENCH["mobilevit_xxs"])
    w = mo.stress_weights(cfg, 7)
    m = _model(cfg, w, "bf16")
    B = 8
    img = torch.from_numpy(mo.make_image(cfg, B, 8)).cuda()
    out = torch.empty((B, cfg["num_classes"]), dtype=torch.float32, device="cuda")
    s = torch.cuda.Stream()
    outs = []
    with torch.cuda.stream(s):
        for _ in range(4):                                              # eager, capture, replay, replay
            m.forward_raw(img.data_ptr(), 1, B, 256, 256, out.data_ptr(), 1, s.cuda_stream)
            s.synchronize()
            outs.append(out.clone())
    st = m.graph_stats()
    assert st["captures"] == 1 and st["replays"] == 2 and st["failures"] == 0, st
    for o in outs[1:]:
        assert torch.equal(o, outs[0])
    single = m(img[:1].cpu().numpy(), training=False)
    assert np.array_equal(single, outs[0][:1].cpu().numpy())
    part = m(img[3:7].cpu().numpy(), training=False)
    assert np.array_equal(part, outs[0][3:7].cpu().numpy())

"""ScalableViT (reference scalable_vit.py) on the H100 engine: fp32 and bf16 against the float64 spec and the reference-code fixtures
(tests/golden/scalable_vit_*__refshim.npz, tests/golden/make_scalable_vit_golden.py), the README model at 256^2, batch 8; plain
attention at head width 32 through vb_op_attention_ex against numpy; the refused sizes, the training rule and the stage entries;
graph replay and batch independence."""
import os

import numpy as np
import pytest

import scalable_vit_oracle as so
from levit_oracle import bf16_round

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
# The whole-model bounds are relative to each case's own logit scale s = max |ref| (0.9 to 2.8 on the SMALL cases).  Measured on an
# H100 over the SMALL cases: fp32 at most 8.4e-7 s, bf16 at most 2.1e-2 s (initial weights; 0.9e-2 s with the stress weights).  The
# bounds are about 4.8 and 3.8 times those.  A case whose logits fall below SCALE_FLOOR fails instead of passing on a vanishing signal.
FP32_REL, BF16_REL = 4e-6, 8e-2
SCALE_FLOOR = 1e-3
# The README model at 256^2: 26 blocks of bf16-stored activations in sequence.  Measured on an H100: 0.67 % of max |ref| (stress
# weights, batch 8); the bound is about 4.5 times that.
README_REL = 3e-2


def _model(cfg, w, precision):
    from vit_tensorflow_b200 import from_config
    m = from_config(cfg, precision=precision)
    m.set_weights_dict(w)
    return m


def _spec(img, w, cfg):
    return np.concatenate([so.forward(img[i:i + 1], w, cfg) for i in range(img.shape[0])])


@pytest.mark.parametrize("gen", ["init_weights", "stress_weights"])
@pytest.mark.parametrize("name", sorted(so.SMALL))
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_scalable_vit_small_vs_spec_and_reference_fixture(lib, precision, name, gen):
    cfg = so.make_config(**so.SMALL[name])
    w = getattr(so, gen)(cfg, so.WEIGHT_SEED)
    img = so.make_image(cfg, so.BATCH, so.IMAGE_SEED)
    got = _model(cfg, w, precision)(img, training=False).numpy().astype(np.float64)
    ref = so.forward(img, w, cfg)
    fix = np.load(os.path.join(GOLDEN, f"{name}__{gen}__refshim.npz"))["logits_ref_f64"]
    scale = np.abs(ref).max()
    bound = (FP32_REL if precision == "fp32" else BF16_REL) * scale
    print(f"{name} {gen} {precision}: max err {np.abs(got - ref).max():.3g} ({np.abs(got - ref).max() / scale:.2e} of |ref| max {scale:.3g})")
    assert scale >= SCALE_FLOOR, f"the case's logits ({scale:.3g}) are too small to test against"
    assert got.shape == ref.shape and np.isfinite(got).all()
    for want in (ref, fix):
        assert np.abs(got - want).max() <= bound, f"max err {np.abs(got - want).max():.3g} > {bound:.3g}"


def test_scalable_vit_readme_model_bf16(lib):
    cfg = so.make_config(**so.BENCH["scalable_vit_readme"])
    img = so.make_image(cfg, 8, so.IMAGE_SEED)
    w = so.stress_weights(cfg, so.WEIGHT_SEED)
    got = _model(cfg, w, "bf16")(img, training=False).numpy().astype(np.float64)
    ref = _spec(img, w, cfg)
    err, scale = np.abs(got - ref).max(), np.abs(ref).max()
    print(f"README model stress_weights: bf16 max err {err:.4g}, |ref| max {scale:.4g} ({err / scale:.2%})")
    assert scale >= SCALE_FLOOR and np.isfinite(got).all() and err <= README_REL * scale


def _attention_ref(q, k, v, heads, dh, scale):
    B, nq, _ = q.shape
    nk = k.shape[1]
    Q, K, V = (t.astype(np.float64).reshape(B, -1, heads, dh).transpose(0, 2, 1, 3) for t in (q, k, v))
    s = Q @ K.transpose(0, 1, 3, 2) * scale
    p = np.exp(s - s.max(-1, keepdims=True))
    o = (p / p.sum(-1, keepdims=True)) @ V
    assert o.shape == (B, heads, nq, dh) and K.shape[2] == nk
    return o.transpose(0, 2, 1, 3).reshape(B, nq, heads * dh)


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("B,nq,nk,heads,scale", [(2, 4096, 64, 2, 40 ** -0.5), (3, 100, 25, 4, 0.0), (2, 130, 130, 3, 0.0), (1, 37, 37, 5, 0.2),
                                                  (2, 65, 257, 2, 0.0), (4, 49, 9, 8, 24 ** -0.5), (1, 2, 1, 1, 0.0)])
def test_plain_attention_head_width_32(lib, precision, B, nq, nk, heads, scale):
    """SSA's shapes: q from every pixel against the r x r reduced keys (nq != nk; nk under, at and over one 64-key block), and
    nq == nk; odd query and key counts (partial query tiles and key blocks); explicit scales (the widened heads' dim_key^-0.5).
    k | v are the fused to_k | to_v rows, as the engine lays them out.  bf16 runs the streaming flash kernel at head width 32."""
    from vit_tensorflow_b200 import _lib
    dh = 32
    HD = heads * dh
    rng = np.random.default_rng(nq * 7 + nk + heads)
    rnd = bf16_round if precision == "bf16" else (lambda t: t)
    q = rnd(rng.standard_normal((B, nq, HD)).astype(np.float32)).astype(np.float32)
    kv = rnd(rng.standard_normal((B, nk, 2 * HD)).astype(np.float32)).astype(np.float32)
    _lib.last_attention_path()
    out, _ = _lib.op_attention_ex(q, heads, dh, np.zeros((B, nq, HD), np.float32), kv=kv, k_off=0, v_off=HD, scale=scale,
                                  precision=precision)
    path = _lib.last_attention_path()
    ref = _attention_ref(q, kv[..., :HD], kv[..., HD:], heads, dh, scale if scale > 0 else dh ** -0.5)
    err = np.abs(out - ref)
    print(f"B{B} nq{nq} nk{nk} h{heads} {precision}: path {path}, max err {err.max():.3g}")
    if precision == "bf16":
        assert path == "flash" or (nq == 1 and path == "cls")
        assert np.isfinite(out).all() and (err <= 1e-2 + 1e-2 * np.abs(ref)).all()
    else:
        assert path == "simt"
        assert (err <= 1e-5 + 1e-5 * np.abs(ref)).all()


def test_head_width_64_attention_dispatch_unchanged(lib):
    """dim_head 64 keeps the resident kernel (nk <= 256) and the streaming one above it: both report the flash path."""
    from vit_tensorflow_b200 import _lib
    rng = np.random.default_rng(3)
    for nk in (197, 300):
        q = bf16_round(rng.standard_normal((2, nk, 3 * 128)).astype(np.float32)).astype(np.float32)
        _lib.last_attention_path()
        out, _ = _lib.op_attention_ex(q, 2, 64, np.zeros((2, nk, 128), np.float32), k_off=128, v_off=256)
        assert _lib.last_attention_path() == "flash"
        ref = _attention_ref(q[..., :128], q[..., 128:256], q[..., 256:], 2, 64, 0.125)
        assert (np.abs(out - ref) <= 1e-2 + 1e-2 * np.abs(ref)).all()


def test_scalable_vit_refusals_and_training_rule(lib):
    from vit_tensorflow_b200 import _lib, ScalableViT
    cfg = so.make_config(**so.SMALL["scalable_vit_rect_odd"])
    w = so.stress_weights(cfg, 3)
    m = _model(cfg, w, "fp32")
    img = so.make_image(cfg, 2, 4)
    ref = so.forward(img, w, cfg)
    # no BatchNorm and dropout 0: training=True computes what training=False does
    assert np.array_equal(m(img), m(img, training=False))
    assert np.abs(m(img) - ref).max() <= FP32_REL * np.abs(ref).max()
    other = so.make_image(cfg, 1, 5, 36, 20)                             # maps 9 x 5 (r = 2) and 5 x 3: no window of 2 divides
    with pytest.raises(AssertionError, match=r"stage 2: height \(5\) or width \(3\) of feature map is not divisible by the window size \(2, 2\)"):
        m(other)
    rc = m._lib.vb_forward(m._h, other.ctypes.data, 0, 1, 36, 20, np.zeros((1, 7), np.float32).ctypes.data, 0, None)
    assert rc != 0 and b"ScalableViT stage 2: height (5) or width (3)" in m._lib.vb_last_error(m._h)
    with pytest.raises(ValueError, match=r"ScalableViT stage 1: the 1 x 3 map is smaller than reduction_factor 2"):
        m(so.make_image(cfg, 1, 6, 4, 12))
    with pytest.raises(ValueError, match="channels=3"):
        m(np.zeros((1, 60, 44, 4), np.float32))
    with pytest.raises(_lib.VbError, match="whole forward only"):
        m.forward_embed(img)
    with pytest.raises(_lib.VbError, match="whole forward only"):
        m.forward_head(np.zeros((1, 4, 48), np.float32))
    d = ScalableViT(**so.ctor_kwargs({**cfg, "dropout": 0.1}), precision="fp32")
    d.set_weights_dict(w)
    with pytest.raises(NotImplementedError, match="training=False"):
        d(img)
    assert np.array_equal(d(img, training=False), m(img, training=False))


def test_scalable_vit_graph_replay_and_batch_independence(lib):
    import torch
    cfg = so.make_config(**{**so.SMALL["scalable_vit_s2_win10"], "image_size": (160, 160)})
    w = so.stress_weights(cfg, 7)
    m = _model(cfg, w, "bf16")
    B = 8
    img = torch.from_numpy(so.make_image(cfg, B, 8)).cuda()
    out = torch.empty((B, cfg["num_classes"]), dtype=torch.float32, device="cuda")
    s = torch.cuda.Stream()
    outs = []
    with torch.cuda.stream(s):
        for _ in range(4):                                              # eager, capture, replay, replay
            m.forward_raw(img.data_ptr(), 1, B, 160, 160, out.data_ptr(), 1, s.cuda_stream)
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

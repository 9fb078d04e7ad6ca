"""PiT (reference pit.py) on the H100 engine: every small case in fp32 and bf16 against the float64 spec and the reference-code
fixtures (tests/golden/pit_*__refshim.npz, tests/golden/make_pit_golden.py), the README model at 224^2, batch 4, in bf16; call-time
images smaller than image_size, rectangular ones included; the engine's weight names against the oracle's; the refusals, the
stage entries and the training rule; graph replay and batch independence.

Tolerances per logit are the small-dataset ViT's (test_gpu_small_vit.py): fp32 1e-4 + 1e-3 |ref|, bf16 6e-2 + 4e-2 |ref|."""
import ctypes as C
import os

import numpy as np
import pytest

import pit_oracle as po

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
CASES = [(n, g) for n in sorted(po.SMALL) for g in po.WEIGHTS]
# The README model at 224^2 (n = 962, nine layers of bf16-stored activations), stress weights, batch 4.  Measured on an H100 80GB
# HBM3: a max error of 0.572 % of max |ref| (0.0137 against 2.39); the bound is five times that.
README_MEASURED = 5.72e-3
README_REL = 5 * README_MEASURED


def fp32_tol(ref):
    return 1e-4 + 1e-3 * np.abs(ref)


def bf16_tol(ref):
    return 6e-2 + 4e-2 * np.abs(ref)


def _model(cfg, w, precision):
    from vit_tensorflow_b200 import from_config
    m = from_config(cfg, precision=precision)
    m.set_weights_dict(w)
    return m


@pytest.mark.parametrize("gen", po.WEIGHTS)
@pytest.mark.parametrize("name", sorted(po.SMALL))
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_pit_small_vs_spec_and_reference_fixture(lib, precision, name, gen):
    cfg = po.make_config(**po.SMALL[name])
    w = getattr(po, gen)(cfg, po.WEIGHT_SEED)
    img = po.make_image(cfg, po.BATCH, po.IMAGE_SEED)
    m = _model(cfg, w, precision)
    assert list(m.weight_specs().items()) == [(k, v[0]) for k, v in po.weight_specs(cfg).items()]
    got = np.asarray(m(img, training=False), np.float64)
    ref = po.forward(img, w, cfg)
    with np.load(os.path.join(GOLDEN, po.fixture_name(name, gen))) as z:
        fix = z["logits_ref_f64"]
    tol = fp32_tol(ref) if precision == "fp32" else bf16_tol(ref)
    err = np.abs(got - ref)
    print(f"{name} {gen} {precision}: max err {err.max():.3g} ({err.max() / np.abs(ref).max():.2e} of |ref| max), "
          f"worst err / tol {(err / tol).max():.3f}")
    assert got.shape == ref.shape and np.isfinite(got).all()
    for want in (ref, fix):
        assert (np.abs(got - want) <= tol).all(), np.abs(got - want).max()


def test_pit_readme_model_bf16(lib):
    cfg = po.make_config(**po.README)
    w = po.stress_weights(cfg, po.WEIGHT_SEED)
    img = po.make_image(cfg, 4, po.IMAGE_SEED)
    got = np.asarray(_model(cfg, w, "bf16")(img, training=False), np.float64)
    ref = po.forward(img, w, cfg)
    err, scale = np.abs(got - ref).max(), np.abs(ref).max()
    print(f"README model stress_weights: bf16 max err {err:.4g}, |ref| max {scale:.4g} ({err / scale:.3%}); "
          f"worst err / per-logit bf16 tol {(np.abs(got - ref) / bf16_tol(ref)).max():.3f}")
    assert np.isfinite(got).all() and err <= README_REL * scale
    assert (np.abs(got - ref) <= bf16_tol(ref)).all()


@pytest.mark.parametrize("hw", [(36, 36), (30, 30), (20, 32), (36, 4), (4, 4)])
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_pit_call_time_images_up_to_the_table(lib, precision, hw):
    """pit_stream is built for 36^2 (289 patches); smaller and rectangular images read the first n + 1 rows of pos_embedding."""
    cfg = po.make_config(**po.SMALL["pit_stream"])
    w = po.stress_weights(cfg, 5)
    img = po.make_image(cfg, 3, 7, *hw)
    got = np.asarray(_model(cfg, w, precision)(img, training=False), np.float64)
    ref = po.forward(img, w, cfg)
    tol = fp32_tol(ref) if precision == "fp32" else bf16_tol(ref)
    assert (np.abs(got - ref) <= tol).all(), np.abs(got - ref).max()


def test_pit_refusals_and_training_rule(lib):
    from vit_tensorflow_b200 import PiT, _lib
    cfg = po.make_config(**po.SMALL["pit_p8"])
    w = po.stress_weights(cfg, 3)
    m = _model(cfg, w, "fp32")
    img = po.make_image(cfg, 2, 4)
    with pytest.raises(ValueError, match=r"the 40 x 32 image gives 63 patches but pos_embedding has rows for 49"):
        m(po.make_image(cfg, 1, 0, 40, 32))
    with pytest.raises(ValueError, match=r"a 7 x 32 image is smaller than one 8 x 8 patch"):
        m(po.make_image(cfg, 1, 0, 7, 32))
    with pytest.raises(ValueError, match=r"NHWC"):
        m(np.zeros((1, 32, 32, 4), np.float32))
    out = np.zeros((1, 5), np.float32)
    m.build()                                                           # vb_finalize, which the raw entry expects
    for h, wd, msg in ((40, 32, b"gives 63 patches but pos_embedding has rows for 49"), (32, 7, b"smaller than one 8 x 8 patch")):
        big = po.make_image(cfg, 1, 0, h, wd)                            # the engine refuses them on its own too
        rc = m._lib.vb_forward(m._h, big.ctypes.data, 0, 1, h, wd, out.ctypes.data, 0, None)
        assert rc != 0 and msg in m._lib.vb_last_error(m._h)
    msg = "PiT runs as a whole forward only"
    for call in (lambda: m.forward_embed(img), lambda: m.forward_tokens(np.zeros((2, 50, 64), np.float32)),
                 lambda: m.forward_head(np.zeros((2, 50, 64), np.float32)), lambda: m.to_patch(img),
                 lambda: m.patch_to_emb(np.zeros((2, 192), np.float32))):
        with pytest.raises(_lib.VbError, match=msg):
            call()
    buf = np.zeros(256, np.float32)
    rc = m._lib.vb_forward_distill(m._h, img.ctypes.data_as(C.c_void_p), _lib.MEM_HOST, 2, 32, 32, buf.ctypes.data_as(C.c_void_p),
                                   buf.ctypes.data_as(C.c_void_p), buf.ctypes.data_as(C.c_void_p), _lib.MEM_HOST, None)
    assert rc != 0 and msg.encode() in m._lib.vb_last_error(m._h)
    assert not hasattr(m, "transformer")
    # dropout 0: training=True computes what training=False does; dropout > 0 needs training=False
    assert np.array_equal(m(img), m(img, training=False))
    for kw in (dict(dropout=0.1), dict(emb_dropout=0.1)):
        d = PiT(**po.ctor_kwargs({**cfg, **kw}), precision="fp32")
        d.set_weights_dict(w)
        with pytest.raises(NotImplementedError, match="training=False"):
            d(img)
        assert np.array_equal(d(img, training=False), m(img, training=False))


@pytest.mark.parametrize("name", ["pit_unfold_fold", "pit_fold_unfold_fold"])
def test_pit_folded_layer_after_an_unfolded_one_reads_its_own_statistics(lib, name):
    """In bf16 a stage with heads * dim_head off a multiple of 64 runs its LayerNorms unfolded, and the folded stage after it must
    recompute the row statistics of its input.  The unfolded stage's fc2 is scaled by 8 so that its output moves the rows far from
    the statistics an earlier layer left: folding with those (stale) statistics puts the logits 4 to 17 times the bf16 tolerance
    off the spec (restated in float64 on the CPU), while the bf16 engine stays well inside it."""
    cfg = po.make_config(**po.SMALL[name])
    w = po.stress_weights(cfg, po.WEIGHT_SEED)
    for L, _, heads, _ in po.layer_plan(cfg):
        if heads * cfg["dim_head"] % 64:
            for k in ("fc2.kernel", "fc2.bias"):
                w[f"layers.{L}.{k}"] = w[f"layers.{L}.{k}"] * np.float32(8)
    img = po.make_image(cfg, po.BATCH, po.IMAGE_SEED)
    got = np.asarray(_model(cfg, w, "bf16")(img, training=False), np.float64)
    ref = po.forward(img, w, cfg)
    err = np.abs(got - ref)
    print(f"{name} (unfolded fc2 x 8) bf16: max err {err.max():.3g}, worst err / tol {(err / bf16_tol(ref)).max():.3f}")
    assert (err <= bf16_tol(ref)).all(), err.max()


def test_pit_zero_stages_runs_embedding_and_head(lib):
    """heads=() leaves no (depth, heads) pair: the reference builds no Transformer and classifies the embedded cls row."""
    cfg = po.make_config(**{**po.SMALL["pit_p8"], "heads": ()})
    w = po.stress_weights(cfg, 2)
    assert not any(k.startswith("layers.") for k in w)
    img = po.make_image(cfg, 2, 3)
    for precision in ("fp32", "bf16"):
        got = np.asarray(_model(cfg, w, precision)(img, training=False), np.float64)
        ref = po.forward(img, w, cfg)
        assert (np.abs(got - ref) <= (fp32_tol(ref) if precision == "fp32" else bf16_tol(ref))).all()


def test_pit_graph_replay_and_batch_independence(lib):
    import torch
    cfg = po.make_config(**po.SMALL["pit_p5_odd"])
    w = po.stress_weights(cfg, 7)
    m = _model(cfg, w, "bf16")
    B = 8
    img = torch.from_numpy(po.make_image(cfg, B, 8)).cuda()
    out = torch.empty((B, cfg["num_classes"]), dtype=torch.float32, device="cuda")
    s = torch.cuda.Stream()
    outs = []
    with torch.cuda.stream(s):
        for _ in range(4):                                              # eager, capture, replay, replay
            m.forward_raw(img.data_ptr(), 1, B, 30, 30, out.data_ptr(), 1, s.cuda_stream)
            s.synchronize()
            outs.append(out.clone())
    st = m.graph_stats()
    assert st["captures"] == 1 and st["replays"] == 2 and st["failures"] == 0, st
    for o in outs[1:]:
        assert torch.equal(o, outs[0])
    eager = m(img.cpu().numpy(), training=False)
    assert np.array_equal(eager, outs[0].cpu().numpy())
    single = m(img[:1].cpu().numpy(), training=False)
    assert np.array_equal(single, outs[0][:1].cpu().numpy())
    part = m(img[3:7].cpu().numpy(), training=False)
    assert np.array_equal(part, outs[0][3:7].cpu().numpy())

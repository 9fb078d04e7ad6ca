"""DistillWrapper on the H100 (distill.py:87-134): the fp32 and bf16 engines against every fixture of the reference run over the
numpy stand-in, an engine teacher against a host callable returning its logits, captured and replayed calls bit for bit (with T,
alpha, student and teacher weights changing between them), the loss kernels on their own against float64, and the refusals.

Tolerances.  Logits: fp32 rtol 1e-3 / atol 1e-4 (the distillation students' fp32 gate); bf16 test_gpu_models' BF16_ATOL /
BF16_RTOL, which the same ViT / T2TViT paths are held to.  Loss: the first-order bound of the measured logit errors, doubled --
ce[i] moves by at most 2 max|d student_logits| per unit of label mass, and q[j] by at most 2 (max|d teacher_logits| / |T|)
(ln(1 / 1e-7) + 1), scaled by alpha T^2 -- plus 1e-6 of the loss for its float32 rounding.
"""
import ctypes as C
import os

import numpy as np
import pytest

import distill_wrapper_oracle as o
from test_gpu_models import BF16_ATOL, BF16_RTOL

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")


def _build(name, gen, precision, host_teacher=False):
    import vit_tensorflow_b200 as vb
    student, inp = o.engine_student(name, gen, precision)
    teacher = o.engine_teacher(name, inp, precision)
    if host_teacher and inp["fixed"] is None:
        eng = teacher
        teacher = lambda x, training=True: eng(x, training=training)                     # noqa: E731
    w = vb.DistillWrapper(teacher, student, temperature=inp["T"], alpha=inp["alpha"])
    w.set_weights_dict(inp["own"])
    return w, inp


def loss_tol(inp, d_student, d_teacher, loss, T=None, alpha=None):
    T = inp["T"] if T is None else T
    a = inp["alpha"] if alpha is None else alpha
    mass = float(np.abs(inp["labels"]).sum(-1).max())
    bound = (1 - a) * 2 * d_student * mass + a * T * T * 2 * (d_teacher / abs(T)) * (np.log(1e7) + 1)
    return 2 * bound + 1e-6 * float(np.abs(loss).max())


def _check(w, inp, z, atol, rtol):
    loss, sl, dl, tl = w.forward_distill_loss([inp["img"], inp["labels"]])
    errs = {}
    for got, k in ((sl, "student_logits"), (dl, "distill_logits"), (tl, "teacher_logits")):
        ref = z[k]
        err = np.abs(got - ref)
        assert np.isfinite(got).all()
        assert (err <= atol + rtol * np.abs(ref)).all(), f"{k}: max err {err.max():.4g}"
        errs[k] = float(err.max())
    tol = loss_tol(inp, errs["student_logits"], errs["teacher_logits"], z["loss_ref_f64"])
    lerr = float(np.abs(loss - z["loss_ref_f64"]).max())
    assert loss.dtype == np.float32 and lerr <= tol, f"loss err {lerr:.4g} > {tol:.4g} (logit errors {errs})"
    print(f"logit errors {errs}, loss err {lerr:.3g} (tolerance {tol:.3g})")


@pytest.mark.parametrize("gen", o.WEIGHTS)
@pytest.mark.parametrize("name", list(o.CASES))
def test_fp32_engine_matches_every_fixture(name, gen):
    w, inp = _build(name, gen, "fp32")
    _check(w, inp, np.load(os.path.join(GOLDEN, o.fixture_name(name, gen))), 1e-4, 1e-3)


@pytest.mark.parametrize("gen", o.WEIGHTS)
@pytest.mark.parametrize("name", list(o.CASES))
def test_bf16_engine_matches_every_fixture(name, gen):
    w, inp = _build(name, gen, "bf16")
    _check(w, inp, np.load(os.path.join(GOLDEN, o.fixture_name(name, gen))), BF16_ATOL, BF16_RTOL)


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("name", ["vit_cls", "t2t_mean"])
def test_engine_teacher_and_host_callable_give_the_same_bits(name, precision):
    w_dev, inp = _build(name, "stress", precision)
    w_host, _ = _build(name, "stress", precision, host_teacher=True)
    assert w_dev._engine_teacher() and not w_host._engine_teacher()
    x = [inp["img"], inp["labels"]]
    a, b = w_dev(x, training=False), w_host(x, training=False)
    assert np.array_equal(a, b)
    assert np.array_equal(w_dev.forward_distill_loss(x)[3], w_host.forward_distill_loss(x)[3])


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_graph_replays_are_bit_identical_and_follow_every_change(precision):
    import torch
    from vit_tensorflow_b200 import _lib
    w, inp = _build("vit_cls", "stress", precision)
    b, h, wd, _ = inp["img"].shape
    img = torch.from_numpy(inp["img"]).cuda()
    labels = torch.from_numpy(inp["labels"]).cuda()
    loss = torch.empty(b, device="cuda")
    s = torch.cuda.Stream()
    torch.cuda.synchronize()

    def call(T, alpha):
        w.forward_raw(img.data_ptr(), _lib.MEM_DEVICE, b, h, wd, labels.data_ptr(), _lib.MEM_DEVICE, T, alpha, loss.data_ptr(),
                      _lib.MEM_DEVICE, s.cuda_stream, teacher=w.teacher)
        s.synchronize()
        return loss.cpu().numpy().copy()

    first = call(3.0, 0.5)
    runs = [call(3.0, 0.5) for _ in range(4)]
    for r in runs:
        assert np.array_equal(r, first)
    st = w.graph_stats()
    assert st["captures"] >= 1 and st["replays"] >= 2 and st["failures"] == 0, st
    assert np.array_equal(w([inp["img"], inp["labels"]], training=False), first)         # eager, host buffers, default stream
    for T, alpha in ((1.0, 0.5), (3.0, 0.25), (20.0, 1.0)):
        got = [call(T, alpha) for _ in range(3)]
        assert all(np.array_equal(g, got[0]) for g in got)
        want = o.forward_wrapper(inp, T=T, alpha=alpha)["loss"]
        assert np.abs(got[0] - want).max() <= 1e-3 * np.abs(want).max() and not np.array_equal(got[0], first)
    assert np.array_equal(call(3.0, 0.5), first)
    # a student weight, then a teacher weight: the next call reads each
    bias = inp["w"]["head.bias"] + np.arange(10, dtype=np.float32)
    w.student.set_weights_dict({"head.bias": bias})
    moved = call(3.0, 0.5)
    want = o.forward_wrapper(dict(inp, w=dict(inp["w"], **{"head.bias": bias})))["loss"]
    assert not np.array_equal(moved, first) and np.abs(moved - want).max() <= 1e-2 * np.abs(want).max()
    assert np.array_equal(call(3.0, 0.5), moved)
    tbias = inp["tw"]["head.bias"] + 3.0 * np.arange(10, dtype=np.float32)
    w.teacher.set_weights_dict({"head.bias": tbias})
    moved_t = call(3.0, 0.5)
    inp2 = dict(inp, w=dict(inp["w"], **{"head.bias": bias}), tw=dict(inp["tw"], **{"head.bias": tbias}))
    want = o.forward_wrapper(inp2)["loss"]
    assert not np.array_equal(moved_t, moved) and np.abs(moved_t - want).max() <= 1e-2 * np.abs(want).max()
    assert np.array_equal(call(3.0, 0.5), moved_t)


OP_SHAPES = [(1, 10), (256, 10), (4096, 10), (1, 1000), (256, 1000), (4096, 1000), (1, 1001), (256, 1001), (4096, 1001),
             (1, 21843), (256, 21843)]


@pytest.mark.parametrize("B,K", OP_SHAPES)
def test_op_loss_against_float64(B, K):
    """Logits of magnitude ~100, one-hot and soft labels, edge temperatures and alphas: relative 1e-6 (values below 1 compared at
    absolute 1e-6)."""
    from vit_tensorflow_b200 import _lib
    rng = np.random.default_rng(B * 7 + K)
    s = (100.0 * rng.standard_normal((B, K))).astype(np.float32)
    t = (100.0 * rng.standard_normal((B, K))).astype(np.float32)
    onehot = np.eye(K, dtype=np.float32)[rng.integers(0, K, B)]
    soft = rng.uniform(0, 1, (B, K)).astype(np.float32)
    for labels, T, alpha in ((onehot, 1.0, 0.5), (soft, 0.01, 0.0), (onehot, 100.0, 1.0), (soft, 3.0, 0.3), (onehot, -2.0, 0.5)):
        got = _lib.op_distill_loss(s, labels, t, T, alpha)
        want = o.wrapper_loss(s, labels, t, T, alpha, eps=float(np.float32(1e-7)))
        assert got.dtype == np.float32 and np.isfinite(got).all()
        np.testing.assert_array_less(np.abs(got - want), 1e-6 * np.maximum(np.abs(want), 1.0))


def test_refusals():
    import vit_tensorflow_b200 as vb
    from vit_tensorflow_b200 import _lib
    w, inp = _build("vit_cls", "init", "fp32")
    x = [inp["img"], inp["labels"]]
    with pytest.raises(ValueError, match="temperature 0"):
        w(x, temperature=0.0, training=False)
    with pytest.raises(_lib.VbError, match="temperature 0"):
        _lib.op_distill_loss(inp["labels"], inp["labels"], inp["labels"], 0.0, 0.5)
    with pytest.raises(ValueError, match="incompatible"):
        w([inp["img"], inp["labels"][:, :4]], training=False)
    with pytest.raises(ValueError, match="expected \\[b, num_classes\\]"):
        vb.DistillWrapper(lambda img, training=True: np.zeros((3, 4), np.float32), w.student)(x, training=False)
    other = vb.ViT(**dict(o.teacher_kwargs("vit_cls"), num_classes=7), precision="fp32")
    with pytest.raises(_lib.VbError, match="the teacher logits must be \\[b, num_classes\\]"):
        vb.DistillWrapper(other, w.student)(x, training=False)
    for b in (1, 3):
        hard = vb.DistillWrapper(w.teacher, w.student, hard=True)
        with pytest.raises(ValueError, match=f"Shapes \\({b},\\) and \\({b}, 10\\) are incompatible"):
            hard([inp["img"][:b], inp["labels"][:b]], training=False)
    _, skw = o.student_kwargs("vit_cls")
    with pytest.raises(NotImplementedError):
        vb.DistillWrapper(w.teacher, vb.DistillableViT(**skw, dropout=0.1, precision="fp32"))(x)
    with pytest.raises(NotImplementedError):
        vb.DistillWrapper(vb.ViT(**o.teacher_kwargs("vit_cls"), emb_dropout=0.1, precision="fp32"), w.student)(x)
    import vit_tensorflow_b200.models as models
    eff = vb.DistillableEfficientViT(image_size=32, patch_size=16, num_classes=10, dim=32, transformer=lambda t, training=True: t)
    with pytest.raises(AttributeError, match="no attribute 'dropout'"):
        vb.DistillWrapper(w.teacher, eff)(x, training=False)
    import distill_oracle as do
    kw = {k: v for k, v in do.CASES["t2t_distill_cls"].items() if k != "kind"}
    with pytest.raises(NotImplementedError, match="injected transformer"):
        vb.DistillWrapper(w.teacher, vb.DistillableT2TViT(**kw, transformer=lambda t, training=True: t))
    # vb_create_distill refuses every kind but ViT and T2TViT, and a depth-0 T2TViT
    lib = _lib.load()
    for name, kind in _lib.KIND.items():
        if kind in (_lib.KIND["vit"], _lib.KIND["t2t_vit"]):
            continue
        cfg = _lib.VbConfig.from_buffer_copy(w.student._cfg)
        cfg.kind = kind
        h = C.c_void_p()
        assert lib.vb_create_distill(C.byref(cfg), 0, C.byref(h)) != 0, name
        assert b"supports ViT and T2TViT (distill.py:47, :61)" in lib.vb_last_error(None), name
    assert models.DistillWrapper is vb.DistillWrapper

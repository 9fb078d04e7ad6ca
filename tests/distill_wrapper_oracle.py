"""Test oracle of DistillWrapper (reference distill.py:87-134), kept beside the tests that use it.

  * CASES: a distillable student (ViT or T2TViT), a teacher (an oracle ViT, or fixed logits large enough that the teacher's
    softmax underflows below 1e-7 and Keras' clip engages), T, alpha, the labels (one-hot or soft rows that do not sum to 1) and
    the batch;
  * forward_wrapper: the float64 restatement of DistillWrapper.call as include/vitb200.h reads it -- distill_oracle's student,
    distill_mlp (LayerNormalization eps 1e-3 + Dense) on the token's row, ce from the student logits and the KL term from the
    teacher alone (Keras' KLDivergence clips y_pred = log_softmax(...) <= 0 to 1e-7);
  * reference_wrapper: the reference's own distill.DistillWrapper run unmodified over the numpy stand-in (oracle/tf_shim.py), with
    its token and distill_mlp set to the case's weights;
  * FakeLib / fake_installed: distill_oracle's C-ABI double, answering vb_create_distill, vb_forward_distill_loss and
    vb_op_distill_loss as well.
"""
from __future__ import annotations

import collections
import contextlib

import numpy as np

import distill_oracle as do
import fake_engine
import oracle
from oracle import ref_bind, tf_shim

WEIGHT_SEED, TEACHER_SEED, OWN_SEED, IMAGE_SEED, LABEL_SEED = 21, 22, 23, 24, 25
WEIGHTS = ("init", "stress")
EPS = 1e-7                                          # keras.backend.epsilon(), KLDivergence's clip

_VIT = dict(kind="vit", image_size=32, patch_size=8, num_classes=10, dim=64, depth=2, heads=4, mlp_dim=128, dim_head=16)
_T2T = dict(do.CASES["t2t_distill_cls"])
CASES = {
    "vit_cls": dict(student=_VIT, teacher="vit", T=3.0, alpha=0.5, labels="onehot", batch=3),
    "vit_mean": dict(student=dict(_VIT, pool="mean"), teacher="vit", T=1.0, alpha=0.5, labels="onehot", batch=3),
    # dim 50: not a multiple of 64, so the bf16 engine runs the transformer's LayerNorms unfolded
    "vit_dim50": dict(student=dict(_VIT, dim=50, heads=2, dim_head=24, mlp_dim=70), teacher="vit", T=0.5, alpha=0.0,
                      labels="onehot", batch=3),
    "vit_k1001": dict(student=dict(_VIT, num_classes=1001), teacher="vit", T=20.0, alpha=1.0, labels="onehot", batch=3),
    "vit_batch1": dict(student=_VIT, teacher="vit", T=3.0, alpha=0.5, labels="onehot", batch=1),
    "vit_soft": dict(student=dict(_VIT, pool="mean"), teacher="vit", T=3.0, alpha=0.5, labels="soft", batch=3),
    "vit_clip": dict(student=_VIT, teacher="fixed", T=1.0, alpha=0.5, labels="soft", batch=3),
    "t2t_cls": dict(student=_T2T, teacher="vit", T=3.0, alpha=0.5, labels="onehot", batch=2),
    "t2t_mean": dict(student=dict(_T2T, pool="mean"), teacher="vit", T=0.5, alpha=1.0, labels="soft", batch=2),
}


def fixture_name(name, gen):
    return f"distill_wrapper_{name}__{gen}__refshim.npz"


def student_kwargs(name):
    kw = dict(CASES[name]["student"])
    return kw.pop("kind"), kw


def teacher_kwargs(name):
    """A small ViT teacher on the student's image with the student's classes."""
    s = CASES[name]["student"]
    return dict(image_size=s["image_size"], patch_size=8, num_classes=s["num_classes"], dim=32, depth=1, heads=2, mlp_dim=64,
                dim_head=16)


def own_weights(dim, num_classes, gen, seed=OWN_SEED):
    """The wrapper's own weights: distillation_token N(0, 1) (distill.py:101) and distill_mlp (:103-106) at Keras' defaults
    (init) or with non-trivial LayerNorm affine and Dense bias (stress)."""
    rng = np.random.default_rng(seed)
    lim = np.sqrt(6.0 / (dim + num_classes))
    w = collections.OrderedDict([("distillation_token", rng.standard_normal((1, 1, dim))),
                                 ("distill_mlp.0.gamma", np.ones(dim)), ("distill_mlp.0.beta", np.zeros(dim)),
                                 ("distill_mlp.1.kernel", rng.uniform(-lim, lim, (dim, num_classes))),
                                 ("distill_mlp.1.bias", np.zeros(num_classes))])
    if gen == "stress":
        w["distill_mlp.0.gamma"] = 1.0 + 0.2 * rng.standard_normal(dim)
        w["distill_mlp.0.beta"] = 0.2 * rng.standard_normal(dim)
        w["distill_mlp.1.bias"] = 0.2 * rng.standard_normal(num_classes)
    return collections.OrderedDict((k, v.astype(np.float32)) for k, v in w.items())


def make_labels(kind, b, K, seed=LABEL_SEED):
    rng = np.random.default_rng(seed)
    if kind == "onehot":
        return np.eye(K, dtype=np.float32)[rng.integers(0, K, b)]
    return rng.uniform(0.0, 1.0, (b, K)).astype(np.float32)           # soft rows, not normalised


def inputs(name, gen):
    """Everything a case's call reads, regenerated from the seeds the fixtures were made with."""
    c = CASES[name]
    kind, kw = student_kwargs(name)
    cfg = oracle.make_config(kind, **kw)
    make = oracle.init_weights if gen == "init" else oracle.stress_weights
    K, b = cfg["num_classes"], c["batch"]
    tcfg = oracle.make_config("vit", **teacher_kwargs(name))
    fixed = 25.0 * np.random.default_rng(TEACHER_SEED).standard_normal((b, K)).astype(np.float32) if c["teacher"] == "fixed" else None
    return dict(cfg=cfg, w=make(cfg, WEIGHT_SEED), own=own_weights(cfg["dim"], K, gen), tcfg=tcfg, tw=make(tcfg, TEACHER_SEED),
                fixed=fixed, img=oracle.make_image(cfg, b, IMAGE_SEED), labels=make_labels(c["labels"], b, K), T=c["T"],
                alpha=c["alpha"])


def teacher_logits(inp, dtype=np.float64):
    if inp["fixed"] is not None:
        return inp["fixed"].astype(dtype)
    return oracle.forward_numpy(inp["img"], inp["tw"], inp["tcfg"], dtype)


def log_softmax(x):
    s = x - x.max(-1, keepdims=True)
    return s - np.log(np.exp(s).sum(-1, keepdims=True))


def wrapper_loss(student_logits, labels, teacher, T, alpha, eps=EPS):
    """distill.py:119-134 as include/vitb200.h reads it: out[i] = (1 - alpha) ce[i] + alpha T^2 mean_j q[j]."""
    s, y, t = (np.asarray(a, np.float64) for a in (student_logits, labels, teacher))
    ce = -(y * log_softmax(s)).sum(-1)
    p = np.clip(np.exp(log_softmax(t / T)), eps, 1.0)
    q = (p * (np.log(p) - np.log(eps))).sum(-1)
    return (1 - alpha) * ce + alpha * T ** 2 * q.sum() / q.shape[0]


def distill_mlp(tokens, own):
    """Sequential([LayerNormalization(), Dense(num_classes)]) (distill.py:103-106) in float64."""
    x = np.asarray(tokens, np.float64)
    mu = x.mean(-1, keepdims=True)
    var = ((x - mu) ** 2).mean(-1, keepdims=True)
    x = (x - mu) / np.sqrt(var + 1e-3) * own["distill_mlp.0.gamma"] + own["distill_mlp.0.beta"]
    return x @ own["distill_mlp.1.kernel"].astype(np.float64) + own["distill_mlp.1.bias"]


def forward_wrapper(inp, T=None, alpha=None):
    """DistillWrapper.call in float64 -> dict(loss [b], student_logits, distill_logits, teacher_logits)."""
    T = inp["T"] if T is None else T
    alpha = inp["alpha"] if alpha is None else alpha
    sl, dt = do.forward_distill(inp["img"], inp["own"]["distillation_token"], inp["w"], inp["cfg"])
    tl = teacher_logits(inp)
    return dict(loss=wrapper_loss(sl, inp["labels"], tl, T, alpha), student_logits=sl, distill_logits=distill_mlp(dt, inp["own"]),
                teacher_logits=tl)


@contextlib.contextmanager
def keras_shape_check():
    """categorical_crossentropy as Keras runs it: labels whose shape is not the logits' raise ValueError (the stand-in would
    broadcast them instead).  Made inside this context only, so oracle/ stays as it is."""
    saved = tf_shim._categorical_crossentropy

    def checked(y_true, y_pred, from_logits=False, **kw):
        a, b = np.shape(y_true), np.shape(y_pred)
        if a != b:
            raise ValueError(f"Shapes {a} and {b} are incompatible")
        return saved(y_true, y_pred, from_logits=from_logits, **kw)

    tf_shim._categorical_crossentropy = checked
    try:
        yield
    finally:
        tf_shim._categorical_crossentropy = saved


def reference_wrapper(ref_dir, name, gen, dtype=np.float64, T=None, alpha=None, own=None, hard=False):
    """The reference's distill.DistillWrapper over the stand-in in `dtype`, its token and distill_mlp set to the case's (or `own`)
    weights -> dict(loss, student_logits, distill_logits, teacher_logits)."""
    inp = inputs(name, gen)
    own = inp["own"] if own is None else own
    T = inp["T"] if T is None else T
    alpha = inp["alpha"] if alpha is None else alpha
    kind, kw = student_kwargs(name)
    cast = lambda a: np.asarray(a, dtype=dtype)
    img = cast(inp["img"])
    tf_shim.set_dtype(dtype)
    try:
        with keras_shape_check(), tf_shim.installed(ref_dir):
            import distill
            cls = distill.DistillableViT if kind == "vit" else distill.DistillableT2TViT
            student = ref_bind.build_model(kind, kw, {k: cast(v) for k, v in inp["w"].items()}, img, cls=cls)
            if inp["fixed"] is not None:
                fixed = cast(inp["fixed"])
                teacher = lambda x, training=True: fixed                                   # noqa: E731
            else:
                teacher = ref_bind.build_model("vit", teacher_kwargs(name), {k: cast(v) for k, v in inp["tw"].items()}, img)
            wrapper = distill.DistillWrapper(teacher=teacher, student=student, temperature=T, alpha=alpha, hard=hard)
            wrapper.distillation_token.assign(cast(own["distillation_token"]))
            wrapper.distill_mlp(np.zeros((1, inp["cfg"]["dim"]), dtype))                   # builds the lazily created variables
            wrapper.distill_mlp.layers[0].set_weights([cast(own["distill_mlp.0.gamma"]), cast(own["distill_mlp.0.beta"])])
            wrapper.distill_mlp.layers[1].set_weights([cast(own["distill_mlp.1.kernel"]), cast(own["distill_mlp.1.bias"])])
            loss = wrapper([img, cast(inp["labels"])], training=False)
            sl, dt = student(img, distill_token=wrapper.distillation_token, training=False)
            return dict(loss=ref_bind.to_numpy(loss), student_logits=ref_bind.to_numpy(sl),
                        distill_logits=ref_bind.to_numpy(wrapper.distill_mlp(dt)), teacher_logits=ref_bind.to_numpy(teacher(img)))
    finally:
        tf_shim.set_dtype(np.float32)


# ------------------------------------------------------------------------------------------ the C-ABI double


class FakeLib(do.FakeLib):
    """distill_oracle's C-ABI double with DistillWrapper's entries, computing with this oracle (host buffers only)."""

    def vb_create_distill(self, cfg_ref, device, handle_ref):
        c = cfg_ref._obj
        if c.kind not in (0, 6):
            self.err = b"vb_create_distill supports ViT and T2TViT (distill.py:47, :61)"
            return 1
        rc = self.vb_create(cfg_ref, device, handle_ref)
        if rc == 0:
            st = self._h(handle_ref._obj.value)
            d, K = st["cfg"]["dim"], st["cfg"]["num_classes"]
            st["specs"] += [("distillation_token", ((1, 1, d), None)), ("distill_mlp.0.gamma", ((d,), None)),
                            ("distill_mlp.0.beta", ((d,), None)), ("distill_mlp.1.kernel", ((d, K), None)),
                            ("distill_mlp.1.bias", ((K,), None))]
            self.calls[-1] = ("vb_create_distill", st["cfg"]["kind"])
        return rc

    def vb_forward_distill_loss(self, h, img, img_mem, b, hh, ww, labels, teacher, tlog, in_mem, T, alpha, loss, sl, dl, tlo, out_mem,
                                stream):
        st = self._ready(h)
        cfg, w = st["cfg"], st["w"]
        K = cfg["num_classes"]
        x = fake_engine._f32(img, (b, hh, ww, 3))
        logits, tokens = do.forward_distill(x, w["distillation_token"], w, cfg)
        if teacher is not None:
            ts = self._ready(teacher)
            tl = oracle.forward_numpy(x, ts["w"], ts["cfg"])
        else:
            tl = fake_engine._f32(tlog, (b, K)).astype(np.float64)
        fake_engine._f32(loss, (b,))[:] = wrapper_loss(logits, fake_engine._f32(labels, (b, K)), tl, T, alpha)
        for ptr, v in ((sl, logits), (dl, distill_mlp(tokens, w)), (tlo, tl)):
            if ptr is not None:
                fake_engine._f32(ptr, (b, K))[:] = v
        self.calls.append(("vb_forward_distill_loss", "teacher" if teacher is not None else "teacher_logits", T, alpha))
        return 0

    def vb_op_distill_loss(self, sl, labels, tl, B, K, T, alpha, out):
        fake_engine._f32(out, (B,))[:] = wrapper_loss(*(fake_engine._f32(p, (B, K)) for p in (sl, labels, tl)), T, alpha)
        self.calls.append(("vb_op_distill_loss", (B, K)))
        return 0


@contextlib.contextmanager
def fake_installed():
    """`vit_tensorflow_b200._lib.load()` returns this module's FakeLib inside the block."""
    from vit_tensorflow_b200 import _lib
    fake = FakeLib()
    saved_load, saved_cached = _lib.load, _lib._lib
    _lib.load = lambda: fake
    try:
        yield fake
    finally:
        _lib.load, _lib._lib = saved_load, saved_cached


def engine_student(name, gen, precision="fp32", seed=None):
    """The case's student on the engine (or the double), with the case's weights; -> (student, inputs)."""
    import vit_tensorflow_b200 as vb
    inp = inputs(name, gen)
    kind, kw = student_kwargs(name)
    cls = vb.DistillableViT if kind == "vit" else vb.DistillableT2TViT
    student = cls(**kw, precision=precision, seed=seed)
    student.set_weights_dict(inp["w"])
    return student, inp


def engine_teacher(name, inp, precision="fp32"):
    """The case's teacher as the engine runs it: an engine ViT with the case's weights, or a host callable of the fixed logits."""
    import vit_tensorflow_b200 as vb
    if inp["fixed"] is not None:
        fixed = inp["fixed"]
        return lambda x, training=True: fixed
    t = vb.ViT(**teacher_kwargs(name), precision=precision)
    t.set_weights_dict(inp["tw"])
    return t

"""DistillWrapper (reference distill.py:87-134) checked against the reference's own code without a GPU.

* LIVE (skipped where the reference checkout is absent): the unmodified reference DistillWrapper over the numpy stand-in equals
  distill_wrapper_oracle.forward_wrapper to ~1e-12 in float64 on every case, at every T and alpha; its loss does not move when
  distill_mlp's weights change and does move with the distillation token (the KL reading of include/vitb200.h); the constructor and
  call signatures and the errors equal the reference's.
* FIXTURES (always): tests/golden/distill_wrapper_*__refshim.npz equal the restatement; the GPU tests compare the engine with them.
* HOST LOGIC over the C-ABI double (always): marshalling, the teacher dispatch, the weight push, the refusals, the ABI.
"""
import inspect
import os
import re

import numpy as np
import pytest

import distill_wrapper_oracle as o
from oracle import tf_shim

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
REF_DIR = os.environ.get("VB_REFERENCE_DIR", "/root/reference/vit_tensorflow")    # the reference checkout (absent on the GPU box)
live = pytest.mark.skipif(not os.path.isdir(REF_DIR), reason="reference checkout not present (GPU box): fixtures cover it")
HEADER = os.path.join(os.path.dirname(__file__), "..", "include", "vitb200.h")


def _close(a, b, rel):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    np.testing.assert_allclose(a, b, rtol=0, atol=rel * max(1.0, float(np.abs(b).max())))


# ------------------------------------------------------------------------------------------ the restatement vs the reference
@live
@pytest.mark.parametrize("gen", o.WEIGHTS)
@pytest.mark.parametrize("name", list(o.CASES))
def test_live_reference_equals_the_restatement(name, gen):
    r = o.reference_wrapper(REF_DIR, name, gen)
    f = o.forward_wrapper(o.inputs(name, gen))
    assert r["loss"].shape == (o.CASES[name]["batch"],)
    for k in f:
        _close(r[k], f[k], 1e-12)


@live
@pytest.mark.parametrize("T", [0.5, 1.0, 3.0, 20.0])
@pytest.mark.parametrize("alpha", [0.0, 0.5, 1.0])
def test_live_reference_at_every_temperature_and_alpha(T, alpha):
    r = o.reference_wrapper(REF_DIR, "vit_soft", "stress", T=T, alpha=alpha)
    _close(r["loss"], o.forward_wrapper(o.inputs("vit_soft", "stress"), T=T, alpha=alpha)["loss"], 1e-12)


@live
def test_live_clip_engages_on_the_fixed_teacher():
    """The fixed teacher's softmax falls below 1e-7 for most classes, so the clip of y_true matters."""
    inp = o.inputs("vit_clip", "init")
    p = np.exp(o.log_softmax(o.teacher_logits(inp) / inp["T"]))
    assert (p < o.EPS).mean() > 0.5
    r = o.reference_wrapper(REF_DIR, "vit_clip", "init")
    unclipped = o.wrapper_loss(r["student_logits"], inp["labels"], o.teacher_logits(inp), inp["T"], inp["alpha"], eps=1e-300)
    assert np.abs(unclipped - r["loss"]).max() > 1e-3
    _close(r["loss"], o.forward_wrapper(inp)["loss"], 1e-12)


@live
@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_live_kl_term_never_reads_distill_mlp(dtype):
    """Keras' KLDivergence clips y_pred = log_softmax(distill_logits / T) <= 0 to 1e-7: rescaling the Dense kernel and changing the
    LayerNorm leave the reference's loss bit-identical; the distillation token changes it through the student's logits."""
    inp = o.inputs("vit_cls", "stress")
    base = o.reference_wrapper(REF_DIR, "vit_cls", "stress", dtype)["loss"]
    own = dict(inp["own"])
    own["distill_mlp.1.kernel"] = own["distill_mlp.1.kernel"] * 7.0
    own["distill_mlp.0.beta"] = own["distill_mlp.0.beta"] + 1.0
    moved = o.reference_wrapper(REF_DIR, "vit_cls", "stress", dtype, own=own)
    assert np.array_equal(moved["loss"], base)
    assert not np.allclose(moved["distill_logits"], o.reference_wrapper(REF_DIR, "vit_cls", "stress", dtype)["distill_logits"])
    own = dict(inp["own"], distillation_token=-inp["own"]["distillation_token"])
    assert np.abs(o.reference_wrapper(REF_DIR, "vit_cls", "stress", dtype, own=own)["loss"] - base).max() > 1e-4


@pytest.mark.parametrize("gen", o.WEIGHTS)
@pytest.mark.parametrize("name", list(o.CASES))
def test_reference_fixture_equals_the_restatement(name, gen):
    z = np.load(os.path.join(GOLDEN, o.fixture_name(name, gen)))
    f = o.forward_wrapper(o.inputs(name, gen))
    _close(z["loss_ref_f64"], f["loss"], 1e-12)
    _close(z["loss_ref_f32"], f["loss"], 1e-5)
    for k in ("student_logits", "distill_logits", "teacher_logits"):
        _close(z[k], f[k], 1e-12)


# ------------------------------------------------------------------------------------------ the boundary
@live
def test_live_constructor_and_call_signatures_equal_the_reference():
    import vit_tensorflow_b200 as vb
    with tf_shim.installed(REF_DIR):
        import distill
        ref_init, ref_call = inspect.signature(distill.DistillWrapper.__init__), inspect.signature(distill.DistillWrapper.call)
    sig = lambda s: [(p.name, p.kind, p.default) for p in list(s.parameters.values())[1:] if p.kind is not p.KEYWORD_ONLY]
    assert sig(inspect.signature(vb.DistillWrapper.__init__)) == sig(ref_init)
    assert [p.name for p in inspect.signature(vb.DistillWrapper.__init__).parameters.values() if p.kind is p.KEYWORD_ONLY] == ["seed"]
    assert sig(inspect.signature(vb.DistillWrapper.__call__)) == sig(ref_call)
    assert vb.DistillWrapper.call is vb.DistillWrapper.__call__


def _small_vit_student(vb, **kw):
    _, skw = o.student_kwargs("vit_cls")
    return vb.DistillableViT(**{**skw, **kw}, precision="fp32")


@live
def test_live_errors_equal_the_reference():
    """A plain ViT student: AssertionError; hard=True: ValueError at batch 1 and 3 (Keras' shape check of categorical_crossentropy,
    which the oracle's context adds to the stand-in); an EfficientViT student: AttributeError at every call."""
    import vit_tensorflow_b200 as vb
    got = {}
    for label in ("reference", "ours"):
        errs = []
        with o.fake_installed(), o.keras_shape_check(), tf_shim.installed(REF_DIR):
            import distill
            import vit
            mod = distill if label == "reference" else vb
            _, skw = o.student_kwargs("vit_cls")
            with pytest.raises(AssertionError) as e:
                mod.DistillWrapper(teacher=lambda x, training=True: x, student=vit.ViT(**skw) if label == "reference" else vb.ViT(**skw))
            errs.append(str(e.value))
            if label == "reference":
                student = mod.DistillableViT(**skw)
                student(np.zeros((1, 32, 32, 3), np.float32), training=False)
            else:
                student = _small_vit_student(vb)
            for b in (1, 3):
                teacher = lambda x, training=True, b=b: np.zeros((b, 10), np.float32)          # noqa: E731
                w = mod.DistillWrapper(teacher=teacher, student=student, temperature=3, alpha=0.5, hard=True)
                with pytest.raises(ValueError) as e:
                    w([np.zeros((b, 32, 32, 3), np.float32), np.eye(10, dtype=np.float32)[:b]], training=False)
                errs.append(str(e.value))
            tr = vit.Transformer(32, 1, 2, 16, 32)
            eff = mod.DistillableEfficientViT(image_size=32, patch_size=16, num_classes=4, dim=32, transformer=tr)
            w = mod.DistillWrapper(teacher=lambda x, training=True: np.zeros((2, 4), np.float32), student=eff)
            for training in (True, False):
                with pytest.raises(AttributeError) as e:
                    w([np.zeros((2, 32, 32, 3), np.float32), np.eye(4, dtype=np.float32)[:2]], training=training)
                errs.append(str(e.value))
        got[label] = errs
    assert got["ours"] == got["reference"]
    assert got["ours"][:3] == ["student must be a vision transformer", "Shapes (1,) and (1, 10) are incompatible",
                               "Shapes (3,) and (3, 10) are incompatible"]
    assert got["ours"][3] == "'DistillableEfficientViT' object has no attribute 'dropout'"


def test_shim_exports_the_wrapper():
    import vit_tensorflow_b200 as vb
    from vit_tensorflow.distill import DistillableViT, DistillWrapper
    assert (DistillableViT, DistillWrapper) == (vb.DistillableViT, vb.DistillWrapper) and "DistillWrapper" in vb.__all__


# ------------------------------------------------------------------------------------------ host logic over the double
def _wrapper(vb, name="vit_cls", gen="stress", teacher="engine", **kw):
    student, inp = o.engine_student(name, gen)
    if teacher == "engine":
        t = vb.ViT(**o.teacher_kwargs(name), precision="fp32")
        t.set_weights_dict(inp["tw"])
    else:
        logits = o.teacher_logits(inp).astype(np.float32)
        t = lambda x, training=True: logits                                                    # noqa: E731
    w = vb.DistillWrapper(t, student, temperature=inp["T"], alpha=inp["alpha"], **kw)
    w.set_weights_dict(inp["own"])
    return w, inp


@pytest.mark.parametrize("name", ["vit_cls", "t2t_cls", "vit_clip"])
def test_call_over_the_double(name):
    import vit_tensorflow_b200 as vb
    with o.fake_installed() as fake:
        w, inp = _wrapper(vb, name, teacher="host" if name == "vit_clip" else "engine")
        assert w.distillation_token.shape == (1, 1, inp["cfg"]["dim"]) and (w.dim, w.num_classes) == (inp["cfg"]["dim"], inp["cfg"]["num_classes"])
        loss = w([inp["img"], inp["labels"]], training=False)
        f = o.forward_wrapper(inp)
        assert loss.dtype == np.float32 and loss.shape == (o.CASES[name]["batch"],) and hasattr(loss, "numpy")
        _close(loss, f["loss"], 1e-5)
        outs = w.forward_distill_loss([inp["img"], inp["labels"]], temperature=2.0, alpha=0.25)
        _close(outs[0], o.forward_wrapper(inp, T=2.0, alpha=0.25)["loss"], 1e-5)
        for got, k in zip(outs[1:], ("student_logits", "distill_logits", "teacher_logits")):
            _close(got, f[k], 1e-5)
        entry = [c for c in fake.calls if c[0] == "vb_forward_distill_loss"]
        assert entry[-1] == ("vb_forward_distill_loss", "teacher_logits" if name == "vit_clip" else "teacher", 2.0, 0.25)
        assert entry[0][2:] == (inp["T"], inp["alpha"])


def test_weight_names_and_initial_values():
    import vit_tensorflow_b200 as vb
    with o.fake_installed():
        student, inp = o.engine_student("vit_cls", "init")
        w = vb.DistillWrapper(lambda x, training=True: x, student, seed=3)
        own = w.get_weights_dict()
        assert list(own) == ["distillation_token", "distill_mlp.0.gamma", "distill_mlp.0.beta", "distill_mlp.1.kernel", "distill_mlp.1.bias"]
        assert np.array_equal(own["distill_mlp.0.gamma"], np.ones(64)) and not own["distill_mlp.1.bias"].any()
        assert np.abs(own["distill_mlp.1.kernel"]).max() <= np.sqrt(6.0 / 74) and own["distillation_token"].std() > 0.5
        assert np.array_equal(vb.DistillWrapper(lambda x, training=True: x, student, seed=3).distillation_token, w.distillation_token)
        with pytest.raises(KeyError, match="belongs to the student: set it with student.set_weights_dict"):
            w.set_weights_dict({"head.bias": np.zeros(10, np.float32)})


def test_student_and_teacher_weight_changes_reach_the_next_call():
    import vit_tensorflow_b200 as vb
    with o.fake_installed():
        w, inp = _wrapper(vb)
        x = [inp["img"], inp["labels"]]
        before = w(x, training=False)
        w.student.set_weights_dict({"head.bias": inp["w"]["head.bias"] + np.arange(10, dtype=np.float32)})
        after = w(x, training=False)
        assert np.abs(after - before).max() > 1e-3
        w.teacher.set_weights_dict({"head.bias": inp["tw"]["head.bias"] + 5.0 * np.arange(10, dtype=np.float32)})
        assert np.abs(w(x, training=False) - after).max() > 1e-3


@pytest.mark.parametrize("cls_name", ["ViT", "DeepViT", "CaiT", "T2TViT", "DistillableViT", "PatchMergerViT"])
def test_engine_teachers_run_on_their_handle(cls_name):
    """Each listed engine class goes through the teacher handle; a subclass, a plain callable or an injected-transformer T2TViT is
    called on the host."""
    import vit_tensorflow_b200 as vb
    from vit_tensorflow_b200 import models
    assert getattr(vb, cls_name) in models._ENGINE_TEACHERS
    with o.fake_installed():
        student, _ = o.engine_student("vit_cls", "init")
        kind = {"ViT": "vit", "DeepViT": "deepvit", "CaiT": "cait", "T2TViT": "t2t_vit", "DistillableViT": "vit",
                "PatchMergerViT": "patch_merger_vit"}[cls_name]
        import cases
        kw = dict(cases.SMALL[{"vit": "vit_small", "deepvit": "deepvit_small", "cait": "cait_small", "t2t_vit": "t2t_small",
                               "patch_merger_vit": "merger_small"}[kind]])
        kw.pop("kind")
        teacher = getattr(vb, cls_name)(**kw, precision="fp32")
        assert vb.DistillWrapper(teacher, student)._engine_teacher()
        sub = type("Sub", (getattr(vb, cls_name),), {})(**kw, precision="fp32")
        assert not vb.DistillWrapper(sub, student)._engine_teacher()
        assert not vb.DistillWrapper(lambda x, training=True: x, student)._engine_teacher()
        if cls_name == "T2TViT":
            inj = vb.T2TViT(**{**kw, "transformer": lambda x, training=True: x}, precision="fp32")
            assert not vb.DistillWrapper(inj, student)._engine_teacher()


def test_refusals_over_the_double():
    import vit_tensorflow_b200 as vb
    with o.fake_installed():
        w, inp = _wrapper(vb)
        x = [inp["img"], inp["labels"]]
        with pytest.raises(ValueError, match="temperature 0"):
            w(x, temperature=0, training=False)
        with pytest.raises(ValueError, match=re.escape("Shapes (3, 9) and (3, 10) are incompatible")):
            w([inp["img"], inp["labels"][:, :9]], training=False)
        bad = vb.DistillWrapper(lambda img, training=True: np.zeros((3, 9), np.float32), w.student)
        with pytest.raises(ValueError, match="expected \\[b, num_classes\\]"):
            bad(x, training=False)
        dropout, _ = o.engine_student("vit_cls", "init")
        _, skw = o.student_kwargs("vit_cls")
        dropout = vb.DistillableViT(**skw, dropout=0.1, precision="fp32")
        with pytest.raises(NotImplementedError):
            vb.DistillWrapper(w.teacher, dropout)(x)
        teacher = vb.ViT(**o.teacher_kwargs("vit_cls"), emb_dropout=0.1, precision="fp32")
        with pytest.raises(NotImplementedError):
            vb.DistillWrapper(teacher, w.student)(x)
        import distill_oracle as do
        kw = {k: v for k, v in do.CASES["t2t_distill_cls"].items() if k != "kind"}
        inj = vb.DistillableT2TViT(**kw, transformer=lambda t, training=True: t, precision="fp32")
        with pytest.raises(NotImplementedError, match="injected transformer"):
            vb.DistillWrapper(w.teacher, inj)


def test_op_distill_loss_marshalling():
    from vit_tensorflow_b200 import _lib
    rng = np.random.default_rng(0)
    s, y, t = (rng.standard_normal((4, 7)).astype(np.float32) for _ in range(3))
    with o.fake_installed() as fake:
        _close(_lib.op_distill_loss(s, y, t, 2.0, 0.3), o.wrapper_loss(s, y, t, 2.0, 0.3), 1e-6)
        assert fake.calls[-1] == ("vb_op_distill_loss", (4, 7))
        with pytest.raises(ValueError, match="alike"):
            _lib.op_distill_loss(s, y[:, :6], t, 2.0, 0.3)


def test_abi_declares_and_binds_the_new_entries():
    from vit_tensorflow_b200 import _lib
    src = open(HEADER).read()
    for name, nargs in (("vb_create_distill", 3), ("vb_forward_distill_loss", 18), ("vb_op_distill_loss", 8)):
        m = re.search(r"VB_API int " + name + r"\(([^)]*)\)", src)
        assert m, name
        assert len(m.group(1).split(",")) == nargs == len(_lib.SIGNATURES[name][1])


def test_vb_create_distill_refuses_other_kinds_over_the_double():
    import vit_tensorflow_b200 as vb
    with o.fake_installed():
        teacher = vb.ViT(**o.teacher_kwargs("vit_cls"), precision="fp32")
        student = vb.DistillableViT(**o.student_kwargs("vit_cls")[1], precision="fp32")
        student._cfg.kind = 2                                                 # as a CaiT config reaches vb_create_distill
        with pytest.raises(_lib_error(), match=re.escape("supports ViT and T2TViT (distill.py:47, :61)")):
            vb.DistillWrapper(teacher, student)


def _lib_error():
    from vit_tensorflow_b200 import _lib
    return _lib.VbError


def test_readme_example_runs_over_the_double():
    """The README's DistillWrapper example, run as written (a host teacher, training=False): a float32 loss vector [2]."""
    src = open(os.path.join(os.path.dirname(__file__), "..", "README.md")).read()
    block = next(b for b in re.findall(r"```python\n(.*?)```", src, re.S) if "DistillWrapper" in b)
    with o.fake_installed() as fake:
        scope = {}
        exec(compile(block, "README.md", "exec"), scope)
        loss = scope["loss"]
        assert loss.shape == (2,) and loss.dtype == np.float32 and np.isfinite(loss).all() and hasattr(loss, "numpy")
        assert [c[1] for c in fake.calls if c[0] == "vb_forward_distill_loss"] == ["teacher_logits"]

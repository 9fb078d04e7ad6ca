"""Test oracle of the distillation students (reference distill.py), kept beside the tests that use it.

  * CASES: DistillableT2TViT configurations, in the reference's constructor kwargs (tests/cases.py's spelling, with `kind`);
  * forward_distill: the float64 numpy restatement of DistillMixin.call with a token (distill.py:17-45) on any model whose
    `call` up to the transformer is spec_numpy.embed_tokens (ViT's patch embedding, or T2T's soft splits, t2t.py:58-74): cls and
    positions, the token appended as the last row, the Transformer over n + 2 rows, then pool + mlp_head on x[:, :-1] and x[:, -1];
  * reference_distill: the reference's own distill.DistillableT2TViT run unmodified over the numpy stand-in (oracle/tf_shim.py),
    with the oracle's weights set by attribute path;
  * FakeLib / fake_installed: tests/fake_engine.py's C-ABI double, answering vb_forward_distill for a T2TViT handle too.
"""
from __future__ import annotations

import contextlib

import numpy as np

import fake_engine
import oracle
from oracle import ref_bind, spec_numpy, tf_shim

WEIGHT_SEED, IMAGE_SEED, TOKEN_SEED, BATCH = 11, 12, 13, 2
WEIGHTS = ("init_weights", "stress_weights")

_SMALL = dict(kind="t2t_vit", image_size=32, num_classes=10, dim=64, depth=2, heads=4, mlp_dim=128, dim_head=16,
              t2t_layers=((3, 2), (3, 2)))
CASES = {
    "t2t_distill_cls": _SMALL,
    "t2t_distill_mean": dict(_SMALL, pool="mean"),
    # dim 50: not a multiple of 64, so the bf16 engine runs the transformer's LayerNorms unfolded
    "t2t_distill_dim50": dict(_SMALL, dim=50, heads=2, dim_head=24, mlp_dim=70, pool="mean", t2t_layers=((5, 2), (3, 2))),
    # one t2t layer: the soft split feeds the Dense directly, with no soft-split transformer
    "t2t_distill_1layer": dict(_SMALL, t2t_layers=((4, 4),)),
    # four t2t layers: soft-split transformers of widths 27, 27 and 108 (k = 1 and an even k with asymmetric SAME padding)
    "t2t_distill_4layers": dict(_SMALL, t2t_layers=((3, 2), (1, 1), (2, 1), (3, 2))),
    # the reference README's T2TViT (README.md:208-216) at its own size
    "t2t_distill_readme": dict(kind="t2t_vit", image_size=224, num_classes=1000, dim=512, depth=5, heads=8, mlp_dim=512,
                               t2t_layers=((7, 4), (3, 2), (3, 2))),
}
SMALL = tuple(n for n in CASES if n != "t2t_distill_readme")


def fixture_name(name, gen):
    return f"{name}__{gen}__refshim.npz"


def config(name):
    c = dict(CASES[name])
    return oracle.make_config(c.pop("kind"), **c)


def make_token(dim, seed=TOKEN_SEED):
    """A distillation token [1, 1, dim] (DistillWrapper's tf.random.normal Variable, distill.py:101)."""
    return np.random.default_rng(seed).standard_normal((1, 1, dim)).astype(np.float32)


def inputs(name, gen):
    """(cfg, weights, image, token) of a fixture case, from the seeds the fixtures were made with."""
    cfg = config(name)
    return cfg, getattr(oracle, gen)(cfg, WEIGHT_SEED), oracle.make_image(cfg, BATCH, IMAGE_SEED), make_token(cfg["dim"])


def forward_distill(img, distill_token, weights, cfg, dtype=np.float64):
    """DistillMixin.call with a distillation token (distill.py:17-45) -> (logits, distill_tokens)."""
    x = spec_numpy.embed_tokens(img, weights, cfg, dtype)                                  # :19-24
    b, _, d = x.shape
    tok = np.broadcast_to(np.asarray(distill_token, dtype=dtype).reshape(1, 1, d), (b, 1, d))
    x = np.concatenate([x, tok], axis=1)                                                   # :26-28
    x = spec_numpy.transformer_tokens(x, weights, cfg, dtype)                              # :30 (_attend, dropout 0)
    return spec_numpy.head_logits(x[:, :-1], weights, cfg, dtype), x[:, -1]                # :32-43


def reference_distill(ref_dir, name_or_case, weights, img, token, dtype=np.float64, img_call=None):
    """The reference's distill.DistillableT2TViT over the stand-in in `dtype`: -> (logits, distill_tokens, plain logits) for
    `img_call` (default `img`, which also builds the variables)."""
    case = CASES[name_or_case] if isinstance(name_or_case, str) else name_or_case
    kind, kw = ref_bind.ctor_kwargs(case)
    w = {k: np.asarray(v, dtype=dtype) for k, v in weights.items()}
    x = np.asarray(img if img_call is None else img_call, dtype=dtype)
    tf_shim.set_dtype(dtype)
    try:
        with tf_shim.installed(ref_dir):
            import distill
            model = ref_bind.build_model(kind, kw, w, np.asarray(img, dtype=dtype), cls=distill.DistillableT2TViT)
            logits, dist = model(x, distill_token=np.asarray(token, dtype=dtype), training=False)
            plain = model(x, training=False)
            return ref_bind.to_numpy(logits), ref_bind.to_numpy(dist), ref_bind.to_numpy(plain)
    finally:
        tf_shim.set_dtype(np.float32)


class FakeLib(fake_engine.FakeLib):
    """The C-ABI double, with vb_forward_distill answered for a T2TViT handle as well as a ViT one."""

    def vb_forward_distill(self, h, img, mem_in, b, hh, ww, tok, logits, dist, mem_out, stream):
        st = self._ready(h)
        if st["cfg"]["kind"] != "t2t_vit":
            return super().vb_forward_distill(h, img, mem_in, b, hh, ww, tok, logits, dist, mem_out, stream)
        d = st["cfg"]["dim"]
        if st["cfg"]["depth"] == 0:
            self.err = b"vb_forward_distill: this T2TViT was built for an injected transformer (depth 0)"
            return 1
        lo, di = forward_distill(fake_engine._f32(img, (b, hh, ww, 3)), fake_engine._f32(tok, (d,)), st["w"], st["cfg"])
        fake_engine._f32(logits, lo.shape)[:] = lo
        fake_engine._f32(dist, di.shape)[:] = di
        self.calls.append(("vb_forward_distill", (b, hh, ww)))
        return 0


@contextlib.contextmanager
def fake_installed():
    """`vit_tensorflow_b200._lib.load()` returns a FakeLib inside the block (as fake_engine.installed)."""
    from vit_tensorflow_b200 import _lib
    fake = FakeLib()
    saved_load, saved_cached = _lib.load, _lib._lib
    _lib.load = lambda: fake
    try:
        yield fake
    finally:
        _lib.load, _lib._lib = saved_load, saved_cached


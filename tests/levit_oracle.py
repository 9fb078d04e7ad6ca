"""Test oracle of LeViT (reference levit.py), kept beside the tests that use it.

  * make_config / weight_specs / init_weights / stress_weights: configs and seeded weights in the engine's names (SURVEY.md
    App. B: the reference's attribute paths), the reference's initial distributions;
  * forward: the float64 numpy restatement of LeViT.call (levit.py:214-226) with inference BatchNormalization;
  * forward_torch: an independent PyTorch restatement (conv2d with explicit asymmetric SAME padding, F.batch_norm);
  * installed(): cct_oracle's stand-in plus what levit.py calls beyond it (BatchNormalization with its training and inference
    branches, GlobalAvgPool2D, tf.nn.relu6, meshgrid / stack / unstack), so that the reference's levit.py runs unmodified --
    including the usage block it executes on import (levit.py:228-242); build_reference loads the oracle's weights by attribute path.

The TensorFlow semantics restated here (third-party, public API documentation): BatchNormalization normalises with the batch's
mean and biased variance over every axis but the last when training, and with moving_mean / moving_variance otherwise, then
applies gamma and beta; epsilon is added to the variance.  A 1x1 Conv2D with stride 2 and 'valid' padding reads the pixels
(2r, 2c).  Embedding initialises uniform(-0.05, 0.05).
"""
from __future__ import annotations

import collections
import contextlib
import math
import random
import sys

import numpy as np

import cct_oracle
from oracle import spec_numpy, tf_shim
from vit_tensorflow_b200.models import LEVIT_CTOR_KEYS, levit_cast_tuple

LEVIT_DEFAULTS = dict(stages=3, dim_key=32, dim_value=64, dropout=0.0, num_distill_classes=None)   # levit.py:165-177
BN_EPS = 1e-5
BN_LEAVES = ("gamma", "beta", "moving_mean", "moving_variance")


def make_config(**kw) -> dict:
    cfg = dict(LEVIT_DEFAULTS)
    cfg.update(kw)
    cfg["kind"] = "levit"
    s = cfg["stages"]
    cfg["dims"], cfg["depths"], cfg["layer_heads"] = (levit_cast_tuple(cfg[k], s) for k in ("dim", "depth", "heads"))
    return cfg


def ctor_kwargs(cfg) -> dict:
    return {k: cfg[k] for k in LEVIT_CTOR_KEYS if k in cfg}


def blocks(cfg):
    """(attribute-path prefix, dim, dim_out, heads, fmap, mlp_mult, downsample) of every block in backbone order (levit.py:194-204)."""
    out, fmap, t = [], cfg["image_size"] // 16, 0
    for ind in range(cfg["stages"]):
        d, n, h = cfg["dims"][ind], cfg["depths"][ind], cfg["layer_heads"][ind]
        out += [(f"backbone.{t}.layers.{L}.", d, d, h, fmap, cfg["mlp_mult"], False) for L in range(n)]
        t += 1
        if ind != cfg["stages"] - 1:
            out.append((f"backbone.{t}.layers.0.", d, cfg["dims"][ind + 1], 2 * h, fmap, 2, True))
            t += 1
            fmap = math.ceil(fmap / 2)
    return out


def weight_specs(cfg):
    s = collections.OrderedDict()
    cin = 3
    for i, cout in enumerate((32, 64, 128, cfg["dims"][0])):
        s[f"conv_embedding.{i}.kernel"], s[f"conv_embedding.{i}.bias"] = ((3, 3, cin, cout), "glorot"), ((cout,), "zeros")
        cin = cout
    dk, dv = cfg["dim_key"], cfg["dim_value"]
    for pre, d, dout, h, fmap, mult, _ in blocks(cfg):
        a = pre + "0."
        for n, w in (("to_q", h * dk), ("to_k", h * dk), ("to_v", h * dv)):
            s[a + n + ".0.kernel"] = ((1, 1, d, w), "glorot")
            for leaf in BN_LEAVES:
                s[a + n + ".1." + leaf] = ((w,), leaf)
        s[a + "pos_bias.embeddings"] = ((fmap * fmap, h), "embedding")
        s[a + "to_out.1.kernel"], s[a + "to_out.1.bias"] = ((1, 1, h * dv, dout), "glorot"), ((dout,), "zeros")
        for leaf in BN_LEAVES:
            s[a + "to_out.2." + leaf] = ((dout,), "zeros" if leaf == "gamma" else leaf)     # gamma_initializer='zeros' (:91)
        s[pre + "1.net.0.kernel"], s[pre + "1.net.0.bias"] = ((1, 1, dout, dout * mult), "glorot"), ((dout * mult,), "zeros")
        s[pre + "1.net.3.kernel"], s[pre + "1.net.3.bias"] = ((1, 1, dout * mult, dout), "glorot"), ((dout,), "zeros")
    dl = cfg["dims"][-1]
    s["mlp_head.kernel"], s["mlp_head.bias"] = ((dl, cfg["num_classes"]), "glorot"), ((cfg["num_classes"],), "zeros")
    if cfg["num_distill_classes"] is not None:
        n = cfg["num_distill_classes"]
        s["distill_head.kernel"], s["distill_head.bias"] = ((dl, n), "glorot"), ((n,), "zeros")
    return s


def init_weights(cfg, seed=0):
    rng = np.random.default_rng(seed)
    out = collections.OrderedDict()
    for name, (shape, init) in weight_specs(cfg).items():
        if init == "glorot":
            rf = int(np.prod(shape[:-2]))
            lim = math.sqrt(6.0 / (rf * (shape[-2] + shape[-1])))
            a = rng.uniform(-lim, lim, size=shape)
        elif init in ("zeros", "beta", "moving_mean"):
            a = np.zeros(shape)
        elif init in ("gamma", "moving_variance"):
            a = np.ones(shape)
        elif init == "embedding":
            a = rng.uniform(-0.05, 0.05, size=shape)
        else:
            raise AssertionError(init)
        out[name] = np.ascontiguousarray(a, dtype=np.float32)
    return out


def stress_weights(cfg, seed=1, to_out_gamma=1.0):
    """init_weights with what the Keras defaults hide: non-zero biases, betas and moving means, gammas (the to_out ones included)
    around 1, moving variances in [0.5, 2] and a position bias of O(1).  to_out_gamma scales the to_out gammas (the attention
    branches' share of the stream): at 1 a 16-block model's stream grows to logits of O(40)."""
    rng = np.random.default_rng(seed)
    out = init_weights(cfg, seed)
    for name, (shape, init) in weight_specs(cfg).items():
        if name.endswith(".gamma"):                       # the to_out gammas too, whose Keras initial value is 0
            a = (1.0 + 0.2 * rng.standard_normal(shape)) * (to_out_gamma if ".to_out." in name else 1.0)
        elif init in ("zeros", "beta", "moving_mean"):
            a = 0.2 * rng.standard_normal(shape)
        elif init == "moving_variance":
            a = rng.uniform(0.5, 2.0, size=shape)
        elif init == "embedding":
            a = rng.standard_normal(shape)
        else:
            continue
        out[name] = a.astype(np.float32)
    return out


def make_image(cfg, batch, seed=0, h=None, w=None):
    rng = np.random.default_rng(seed)
    return rng.standard_normal((batch, h or cfg["image_size"], w or cfg["image_size"], 3), dtype=np.float32)


# ------------------------------------------------------------------------------------------------ float64 spec
def pos_indices(fmap, downsample):
    """levit.py:102-112: |dr| * fmap + |dc| between the query grid (step 2 when downsampling) and the key grid."""
    qr = np.arange(0, fmap, 2 if downsample else 1)
    kr = np.arange(fmap)
    q = np.stack(np.meshgrid(qr, qr, indexing="ij"), -1).reshape(-1, 2)
    k = np.stack(np.meshgrid(kr, kr, indexing="ij"), -1).reshape(-1, 2)
    rel = np.abs(q[:, None] - k[None])
    return rel[..., 0] * fmap + rel[..., 1]


def _bn(x, w, n):
    return (x - w[n + ".moving_mean"]) / np.sqrt(w[n + ".moving_variance"] + BN_EPS) * w[n + ".gamma"] + w[n + ".beta"]


def _conv1x1(x, w, n, bias=True):
    k = w[n + ".kernel"]
    y = x @ k.reshape(k.shape[-2], k.shape[-1])
    return y + w[n + ".bias"] if bias else y


def attention(x, w, a, heads, dk, dv, fmap, downsample):
    """Attention.call (levit.py:119-139), inference BatchNormalization.  x [b, H, W, C] -> [b, y, y, dim_out]."""
    b = x.shape[0]
    xq = x[:, ::2, ::2] if downsample else x
    y = xq.shape[1]
    q = _bn(_conv1x1(xq, w, a + "to_q.0", False), w, a + "to_q.1").reshape(b, -1, heads, dk).transpose(0, 2, 1, 3)
    k = _bn(_conv1x1(x, w, a + "to_k.0", False), w, a + "to_k.1").reshape(b, -1, heads, dk).transpose(0, 2, 1, 3)
    v = _bn(_conv1x1(x, w, a + "to_v.0", False), w, a + "to_v.1").reshape(b, -1, heads, dv).transpose(0, 2, 1, 3)
    scale = dk ** -0.5
    dots = q @ k.transpose(0, 1, 3, 2) * scale
    bias = w[a + "pos_bias.embeddings"][pos_indices(fmap, downsample)].transpose(2, 0, 1)[None]
    dots = dots + bias / scale
    attn = np.exp(dots - dots.max(-1, keepdims=True))
    attn = attn / attn.sum(-1, keepdims=True)
    o = (attn @ v).transpose(0, 2, 1, 3).reshape(b, y, y, heads * dv)
    o = spec_numpy.gelu(o)
    return _bn(_conv1x1(o, w, a + "to_out.1"), w, a + "to_out.2")


def hard_swish(x):
    return x * np.clip(x + 3.0, 0.0, 6.0) / 6.0


def forward(img, weights, cfg, dtype=np.float64):
    """LeViT.call(img, training=False): logits, or (logits, distill) with a distillation head."""
    w = {k: np.asarray(v, dtype=dtype) for k, v in weights.items()}
    x = np.asarray(img, dtype=dtype)
    for i in range(4):                                                              # conv_embedding :187-192
        kern = w[f"conv_embedding.{i}.kernel"]
        x = spec_numpy.extract_patches_same(x, 3, 2) @ kern.reshape(-1, kern.shape[-1]) + w[f"conv_embedding.{i}.bias"]
    for pre, d, dout, h, fmap, mult, down in blocks(cfg):                           # Transformer.call :156-162
        res = x if (not down and d == dout) else 0
        x = attention(x, w, pre + "0.", h, cfg["dim_key"], cfg["dim_value"], fmap, down) + res
        x = _conv1x1(hard_swish(_conv1x1(x, w, pre + "1.net.0")), w, pre + "1.net.3") + x
    z = x.mean(axis=(1, 2))                                                         # GlobalAvgPool2D :206-208
    out = spec_numpy.dense(z, w, "mlp_head")
    if cfg["num_distill_classes"] is not None:
        return out, spec_numpy.dense(z, w, "distill_head")
    return out


def bf16_round(x):
    """Round to the nearest bfloat16 (ties to even), returned as float64."""
    a = np.asarray(x, np.float32).view(np.uint32).astype(np.uint64)
    a = ((a + 0x7FFF + ((a >> 16) & 1)) & 0xFFFF0000).astype(np.uint32)
    return a.view(np.float32).astype(np.float64)


def forward_bf16_storage(img, weights, cfg):
    """forward() with the operands and results of every 1x1 convolution (the folded BatchNorm applied in float64 after it) rounded
    to bfloat16, everything else in float64: a lower estimate of what storing activations and weights in bf16 alone costs."""
    global _conv1x1
    exact = _conv1x1

    def rounded(x, w, n, bias=True):
        k = w[n + ".kernel"]
        y = bf16_round(x) @ bf16_round(k.reshape(k.shape[-2], k.shape[-1]))
        return bf16_round(y + w[n + ".bias"] if bias else y)
    _conv1x1 = rounded
    try:
        return forward(img, weights, cfg)
    finally:
        _conv1x1 = exact


def forward_torch(img, weights, cfg):
    """The same model restated in PyTorch (float64): F.conv2d with the SAME padding spelled out, F.batch_norm in inference mode,
    F.hardswish, torch.nn.functional.gelu (exact)."""
    import torch
    import torch.nn.functional as F
    t = {k: torch.from_numpy(np.asarray(v, np.float64)) for k, v in weights.items()}
    x = torch.from_numpy(np.asarray(img, np.float64)).permute(0, 3, 1, 2)

    def conv(x, n, stride=1, bias=True):
        k = t[n + ".kernel"]
        return F.conv2d(x, k.permute(3, 2, 0, 1), t[n + ".bias"] if bias else None, stride=stride)

    def bn(x, n):
        return F.batch_norm(x, t[n + ".moving_mean"], t[n + ".moving_variance"], t[n + ".gamma"], t[n + ".beta"], False, 0.0, BN_EPS)

    for i in range(4):
        H, W = x.shape[-2:]
        ph, pw = max((-(-H // 2) - 1) * 2 + 3 - H, 0), max((-(-W // 2) - 1) * 2 + 3 - W, 0)
        x = conv(F.pad(x, (pw // 2, pw - pw // 2, ph // 2, ph - ph // 2)), f"conv_embedding.{i}", 2)
    dk, dv = cfg["dim_key"], cfg["dim_value"]
    for pre, d, dout, h, fmap, mult, down in blocks(cfg):
        a = pre + "0."
        b = x.shape[0]
        q = bn(conv(x, a + "to_q.0", 2 if down else 1, False), a + "to_q.1")
        k, v = bn(conv(x, a + "to_k.0", 1, False), a + "to_k.1"), bn(conv(x, a + "to_v.0", 1, False), a + "to_v.1")
        y = q.shape[-1]
        q, k, v = (z.flatten(2).unflatten(1, (h, -1)).transpose(-1, -2) for z in (q, k, v))    # b h n d
        bias = t[a + "pos_bias.embeddings"][torch.from_numpy(pos_indices(fmap, down))].permute(2, 0, 1)
        attn = torch.softmax(q @ k.transpose(-1, -2) * dk ** -0.5 + bias / dk ** -0.5, dim=-1)
        o = (attn @ v).transpose(-1, -2).reshape(b, h * dv, y, y)
        o = bn(conv(F.gelu(o), a + "to_out.1"), a + "to_out.2")
        x = o + (x if (not down and d == dout) else 0)
        x = conv(F.hardswish(conv(x, pre + "1.net.0")), pre + "1.net.3") + x
    z = x.mean(dim=(2, 3))
    out = (z @ t["mlp_head.kernel"] + t["mlp_head.bias"]).numpy()
    if cfg["num_distill_classes"] is not None:
        return out, (z @ t["distill_head.kernel"] + t["distill_head.bias"]).numpy()
    return out


# ------------------------------------------------------------------------------------------------ the reference's levit.py
def _shim_layers():
    _arr = tf_shim._arr

    class BatchNormalization(tf_shim._Weighted):
        _order = ("gamma", "beta", "moving_mean", "moving_variance")

        def __init__(self, axis=-1, momentum=0.99, epsilon=1e-3, gamma_initializer='ones', name=None, **kwargs):
            super().__init__(name=name)
            if axis != -1:
                raise NotImplementedError("BatchNormalization: only axis=-1 is used by levit.py")
            self.momentum, self.epsilon, self.gamma_initializer = momentum, epsilon, gamma_initializer
            self.gamma = self.beta = self.moving_mean = self.moving_variance = None

        def call(self, inputs, training=None):
            x = _arr(inputs)
            c = x.shape[-1]
            if self.gamma is None:
                self.gamma = tf_shim.Variable(np.ones(c) if self.gamma_initializer == 'ones' else np.zeros(c))
                self.beta, self.moving_mean = tf_shim.Variable(np.zeros(c)), tf_shim.Variable(np.zeros(c))
                self.moving_variance = tf_shim.Variable(np.ones(c))
            if training:                                  # batch statistics; the moving averages follow them
                axes = tuple(range(x.ndim - 1))
                mean, var = x.mean(axis=axes), x.var(axis=axes)
                m = self.momentum
                self.moving_mean.assign(m * self.moving_mean.view(np.ndarray) + (1 - m) * mean)
                self.moving_variance.assign(m * self.moving_variance.view(np.ndarray) + (1 - m) * var)
            else:
                mean, var = self.moving_mean.view(np.ndarray), self.moving_variance.view(np.ndarray)
            return (x - mean) / np.sqrt(var + self.epsilon) * self.gamma.view(np.ndarray) + self.beta.view(np.ndarray)

    class GlobalAvgPool2D(tf_shim.Layer):
        def call(self, inputs):
            return _arr(inputs).mean(axis=(1, 2))

    return BatchNormalization, GlobalAvgPool2D


@contextlib.contextmanager
def installed(reference_dir):
    """cct_oracle.installed(reference_dir) plus what levit.py needs beyond it; `import levit` inside the block is the reference's
    own file (its import-time usage block included), removed from sys.modules again on exit."""
    saved = sys.modules.pop("levit", None)
    with cct_oracle.installed(reference_dir) as tf:
        BatchNormalization, GlobalAvgPool2D = _shim_layers()
        layers = sys.modules["tensorflow.keras.layers"]
        layers.BatchNormalization, layers.GlobalAvgPool2D = BatchNormalization, GlobalAvgPool2D
        arr = tf_shim._arr
        extra = dict(
            meshgrid=lambda *a, indexing="xy", **_: np.meshgrid(*[arr(x) for x in a], indexing=indexing),
            stack=lambda values, axis=0, **_: np.stack([arr(v) for v in values], axis=axis),
            unstack=lambda value, axis=0, **_: [np.take(arr(value), i, axis=axis) for i in range(arr(value).shape[axis])])
        for k, f in extra.items():
            setattr(tf, k, f)
        tf.nn.relu6 = tf_shim._returns_tensor(lambda x, **_: np.clip(arr(x), 0.0, 6.0))
        try:
            yield tf
        finally:
            sys.modules.pop("levit", None)
            if saved is not None:
                sys.modules["levit"] = saved


def load_weights(model, w):
    """The oracle's weights into a reference LeViT by attribute path (levit.py:187-212)."""
    for i, conv in enumerate(model.conv_embedding.layers):
        conv.set_weights([w[f"conv_embedding.{i}.kernel"], w[f"conv_embedding.{i}.bias"]])
    for t, tr in enumerate(model.backbone.layers):
        for L, (attn, mlp) in enumerate(tr.layers):
            a = f"backbone.{t}.layers.{L}.0."
            for n in ("to_q", "to_k", "to_v"):
                seq = getattr(attn, n).layers
                seq[0].set_weights([w[a + n + ".0.kernel"]])
                seq[1].set_weights([w[a + n + ".1." + leaf] for leaf in BN_LEAVES])
            attn.pos_bias.embeddings.assign(w[a + "pos_bias.embeddings"])
            attn.to_out.layers[1].set_weights([w[a + "to_out.1.kernel"], w[a + "to_out.1.bias"]])
            attn.to_out.layers[2].set_weights([w[a + "to_out.2." + leaf] for leaf in BN_LEAVES])
            m = f"backbone.{t}.layers.{L}.1.net."
            mlp.net.layers[0].set_weights([w[m + "0.kernel"], w[m + "0.bias"]])
            mlp.net.layers[3].set_weights([w[m + "3.kernel"], w[m + "3.bias"]])
    model.mlp_head.set_weights([w["mlp_head.kernel"], w["mlp_head.bias"]])
    if "distill_head.kernel" in w:
        model.distill_head.set_weights([w["distill_head.kernel"], w["distill_head.bias"]])


@contextlib.contextmanager
def reference_module(reference_dir, dtype=np.float64):
    """The reference's levit module over the stand-in in `dtype` (imported once: the import runs its 224^2 usage block)."""
    import importlib
    tf_shim.set_dtype(dtype)
    try:
        with installed(reference_dir):
            yield importlib.import_module("levit")
    finally:
        tf_shim.set_dtype(np.float32)


def reference_logits(mod, cfg, w, img, dtype=np.float64, img_call=None):
    """Build the reference's LeViT for `cfg`, call it once on `img` so that Keras builds every variable (the Embedding is built
    lazily), load `w` and return `model(img_call or img, training=False)` (a tuple with a distillation head)."""
    model = mod.LeViT(**ctor_kwargs(cfg))
    model(np.asarray(img, dtype), training=False)
    load_weights(model, {k: np.asarray(v, dtype) for k, v in w.items()})
    out = model(np.asarray(img if img_call is None else img_call, dtype), training=False)
    if isinstance(out, tuple):
        return tuple(np.asarray(o).view(np.ndarray).copy() for o in out)
    return np.asarray(out).view(np.ndarray).copy()


def random_config(seed):
    """A small random configuration: 1-4 stages, int or short-tuple dims / depths / heads, dim_key below or above dim_value,
    odd widths, with or without a distillation head."""
    r = random.Random(seed)
    stages = r.randint(1, 4)
    image_size = 16 * r.choice([1, 2, 3, 4])

    def spec(lo, hi):
        if r.random() < 0.4:
            return r.randint(lo, hi)
        return tuple(r.randint(lo, hi) for _ in range(r.randint(1, stages)))
    dk, dv = r.choice([(r.randint(3, 9), r.randint(10, 17)), (r.randint(10, 17), r.randint(3, 9)), (8, 8)])
    return make_config(image_size=image_size, num_classes=r.randint(2, 9), dim=spec(5, 24), depth=spec(0, 2), heads=spec(1, 3),
                       mlp_mult=r.randint(1, 3), stages=stages, dim_key=dk, dim_value=dv,
                       num_distill_classes=r.choice([None, r.randint(2, 6)]))


# ------------------------------------------------------------------------------------------------ cases
# small cases (fixtures with float32 and float64 reference logits) and the two configurations tools/levit_bench.py measures
SMALL = {
    "levit_small": dict(image_size=64, num_classes=10, dim=(64, 128), depth=(2, 1), heads=(2, 4), mlp_mult=2, stages=2),
    "levit_small_distill": dict(image_size=48, num_classes=7, dim=64, depth=1, heads=(1, 2, 2), mlp_mult=3, stages=3, dim_key=16,
                                dim_value=32, num_distill_classes=5),
    "levit_odd": dict(image_size=32, num_classes=5, dim=(40, 56), depth=1, heads=3, mlp_mult=1, stages=2, dim_key=20, dim_value=12),
    # the widths of the paper's LeViT-192 (192, 288): 288 is not a multiple of 64
    "levit_192": dict(image_size=64, num_classes=10, dim=(192, 288), depth=1, heads=(3, 5), mlp_mult=2, stages=2),
}
BENCH = {
    "levit_readme": dict(image_size=224, num_classes=1000, dim=(256, 384, 512), depth=4, heads=(4, 6, 8), mlp_mult=2, stages=3),
    "levit_128s": dict(image_size=224, num_classes=1000, dim=(128, 256, 384), depth=(2, 3, 4), heads=(4, 6, 8), mlp_mult=2, stages=3,
                       dim_key=16, dim_value=32),
}
WEIGHT_SEED, IMAGE_SEED, BATCH = 21, 22, 2

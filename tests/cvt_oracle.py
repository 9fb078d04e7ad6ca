"""Test oracle of CvT (reference cvt.py), kept beside the tests that use it.

  * make_config / weight_specs / init_weights / stress_weights: configs and seeded weights in the engine's names (SURVEY.md
    App. B: the reference's attribute paths), the reference's initial distributions;
  * forward: the float64 numpy restatement of CvT.call (cvt.py:200-202) with inference BatchNormalization;
  * forward_torch: an independent PyTorch restatement (conv2d with explicit asymmetric SAME padding and groups=C, F.batch_norm,
    F.layer_norm over the channels at eps 1e-5);
  * installed(): levit_oracle's stand-in plus what cvt.py calls beyond it (Conv2D with groups, tf.math.reduce_variance, tf.sqrt,
    tf.ones), so that the reference's cvt.py runs unmodified; load_weights sets the oracle's weights by attribute path.

The TensorFlow semantics restated here (third-party, public API documentation): a Conv2D with groups == filters == input channels
is a depthwise convolution, kernel [k, k, 1, C], glorot fans k^2 and k^2 * C; 'SAME' gives ceil(in / stride) positions with total
padding max((out - 1) * stride + k - in, 0), the smaller half first; tf.math.reduce_variance is the biased variance.
"""
from __future__ import annotations

import collections
import contextlib
import math
import random
import sys

import numpy as np

import levit_oracle
from oracle import spec_numpy, tf_shim
from vit_tensorflow_b200.models import CVT_CTOR_KEYS, CVT_STAGE_KEYS

CVT_DEFAULTS = dict(s1_emb_dim=64, s1_emb_kernel=7, s1_emb_stride=4, s1_proj_kernel=3, s1_kv_proj_stride=2, s1_heads=1, s1_depth=1,
                    s1_mlp_mult=4, s2_emb_dim=192, s2_emb_kernel=3, s2_emb_stride=2, s2_proj_kernel=3, s2_kv_proj_stride=2, s2_heads=3,
                    s2_depth=2, s2_mlp_mult=4, s3_emb_dim=384, s3_emb_kernel=3, s3_emb_stride=2, s3_proj_kernel=3, s3_kv_proj_stride=2,
                    s3_heads=6, s3_depth=10, s3_mlp_mult=4, dropout=0.0)   # cvt.py:150-177
LN_EPS, BN_EPS, DIM_HEAD = 1e-5, 1e-5, 64
BN_LEAVES = levit_oracle.BN_LEAVES


def make_config(image_size=224, image_w=None, **kw) -> dict:
    """A CvT config: the reference's constructor kwargs (defaults filled in) plus the image size the tests call it with."""
    cfg = dict(CVT_DEFAULTS)
    cfg.update(kw)
    cfg["kind"] = "cvt"
    cfg["image_h"], cfg["image_w"] = image_size, image_w or image_size
    return cfg


def ctor_kwargs(cfg) -> dict:
    return {k: cfg[k] for k in CVT_CTOR_KEYS if k in cfg}


def stages(cfg):
    return [{k: cfg[f"s{i}_{k}"] for k in CVT_STAGE_KEYS} for i in (1, 2, 3)]


def weight_specs(cfg):
    s = collections.OrderedDict()
    cin = 3
    for st, c in enumerate(stages(cfg)):
        p, d, k = f"cvt_layers.{st}.", c["emb_dim"], c["proj_kernel"]
        inner, hidden = DIM_HEAD * c["heads"], d * c["mlp_mult"]
        s[p + "0.kernel"], s[p + "0.bias"] = ((c["emb_kernel"], c["emb_kernel"], cin, d), "glorot"), ((d,), "zeros")
        s[p + "1.g"], s[p + "1.b"] = ((1, 1, 1, d), "ones"), ((1, 1, 1, d), "zeros")
        for L in range(c["depth"]):
            b = f"{p}2.layers.{L}."
            s[b + "0.norm.g"], s[b + "0.norm.b"] = ((1, 1, 1, d), "ones"), ((1, 1, 1, d), "zeros")
            for n, w in (("to_q", inner), ("to_kv", 2 * inner)):
                a = f"{b}0.fn.{n}.net."
                s[a + "0.kernel"] = ((k, k, 1, d), "glorot")
                for leaf in BN_LEAVES:
                    s[a + "1." + leaf] = ((d,), leaf)
                s[a + "2.kernel"] = ((1, 1, d, w), "glorot")
            s[b + "0.fn.to_out.0.kernel"], s[b + "0.fn.to_out.0.bias"] = ((1, 1, inner, d), "glorot"), ((d,), "zeros")
            s[b + "1.norm.g"], s[b + "1.norm.b"] = ((1, 1, 1, d), "ones"), ((1, 1, 1, d), "zeros")
            s[b + "1.fn.net.0.kernel"], s[b + "1.fn.net.0.bias"] = ((1, 1, d, hidden), "glorot"), ((hidden,), "zeros")
            s[b + "1.fn.net.3.kernel"], s[b + "1.fn.net.3.bias"] = ((1, 1, hidden, d), "glorot"), ((d,), "zeros")
        cin = d
    s["cvt_layers.3.1.kernel"], s["cvt_layers.3.1.bias"] = ((cin, cfg["num_classes"]), "glorot"), ((cfg["num_classes"],), "zeros")
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
        elif init in ("ones", "gamma", "moving_variance"):
            a = np.ones(shape)
        else:
            raise AssertionError(init)
        out[name] = np.ascontiguousarray(a, dtype=np.float32)
    return out


def stress_weights(cfg, seed=1):
    """init_weights with what the defaults hide: non-zero biases, betas and moving means, BatchNorm gammas 1 + 0.2 N, moving
    variances in [0.5, 2], LayerNorm g = 1 + 0.2 N and b = 0.2 N."""
    rng = np.random.default_rng(seed)
    out = init_weights(cfg, seed)
    for name, (shape, init) in weight_specs(cfg).items():
        if init in ("ones", "gamma"):
            a = 1.0 + 0.2 * rng.standard_normal(shape)
        elif init in ("zeros", "beta", "moving_mean"):
            a = 0.2 * rng.standard_normal(shape)
        elif init == "moving_variance":
            a = rng.uniform(0.5, 2.0, size=shape)
        else:
            continue
        out[name] = a.astype(np.float32)
    return out


def make_image(cfg, batch, seed=0, h=None, w=None):
    rng = np.random.default_rng(seed)
    return rng.standard_normal((batch, h or cfg["image_h"], w or cfg["image_w"], 3), dtype=np.float32)


# ------------------------------------------------------------------------------------------------ float64 spec
def layer_norm(x, g, b):
    """cvt.py:38-43: over the channels, biased variance, eps 1e-5, g / b [1, 1, 1, dim]."""
    mu = x.mean(-1, keepdims=True)
    var = ((x - mu) ** 2).mean(-1, keepdims=True)
    return (x - mu) / np.sqrt(var + LN_EPS) * g.reshape(-1) + b.reshape(-1)


def dwconv_same(x, kern, stride):
    """Depthwise k x k SAME convolution, no bias: x [b, H, W, C], kern [k, k, 1, C] -> [b, ceil(H/s), ceil(W/s), C]."""
    k, C = kern.shape[0], x.shape[-1]
    p = spec_numpy.extract_patches_same(x, k, stride)
    return (p.reshape(*p.shape[:3], k * k, C) * kern.reshape(k * k, C)).sum(-2)


def batch_norm(x, w, n):
    return (x - w[n + ".moving_mean"]) / np.sqrt(w[n + ".moving_variance"] + BN_EPS) * w[n + ".gamma"] + w[n + ".beta"]


def conv1x1(x, w, n, bias=True):
    k = w[n + ".kernel"]
    y = x @ k.reshape(k.shape[-2], k.shape[-1])
    return y + w[n + ".bias"] if bias else y


def dw_projection(y, w, a, stride):
    """DepthWiseConv2d.call (cvt.py:79-92), inference BatchNormalization: dw (no bias) -> BN -> 1x1 (no bias)."""
    return conv1x1(batch_norm(dwconv_same(y, w[a + "0.kernel"], stride), w, a + "1"), w, a + "2", False)


def attention(y, w, a, heads, kv_stride):
    """Attention.call (cvt.py:111-127) on the normalised map y [b, H, W, dim]."""
    b, H, W, _ = y.shape
    q = dw_projection(y, w, a + "to_q.net.", 1)
    kv = dw_projection(y, w, a + "to_kv.net.", kv_stride)
    inner = heads * DIM_HEAD
    k, v = kv[..., :inner], kv[..., inner:]
    q, k, v = (t.reshape(b, -1, heads, DIM_HEAD).transpose(0, 2, 1, 3) for t in (q, k, v))
    dots = q @ k.transpose(0, 1, 3, 2) * DIM_HEAD ** -0.5
    attn = np.exp(dots - dots.max(-1, keepdims=True))
    attn = attn / attn.sum(-1, keepdims=True)
    o = (attn @ v).transpose(0, 2, 1, 3).reshape(b, H, W, inner)
    return conv1x1(o, w, a + "to_out.0")


def forward(img, weights, cfg, dtype=np.float64):
    """CvT.call(img, training=False) -> logits [b, num_classes]."""
    w = {k: np.asarray(v, dtype=dtype) for k, v in weights.items()}
    x = np.asarray(img, dtype=dtype)
    for st, c in enumerate(stages(cfg)):
        p = f"cvt_layers.{st}."
        kern = w[p + "0.kernel"]
        x = spec_numpy.extract_patches_same(x, c["emb_kernel"], c["emb_stride"]) @ kern.reshape(-1, kern.shape[-1]) + w[p + "0.bias"]
        x = layer_norm(x, w[p + "1.g"], w[p + "1.b"])
        for L in range(c["depth"]):
            b = f"{p}2.layers.{L}."
            x = attention(layer_norm(x, w[b + "0.norm.g"], w[b + "0.norm.b"]), w, b + "0.fn.", c["heads"], c["kv_proj_stride"]) + x
            y = layer_norm(x, w[b + "1.norm.g"], w[b + "1.norm.b"])
            x = conv1x1(spec_numpy.gelu(conv1x1(y, w, b + "1.fn.net.0")), w, b + "1.fn.net.3") + x
    z = x.mean(axis=(1, 2))
    return spec_numpy.dense(z, w, "cvt_layers.3.1")


def forward_torch(img, weights, cfg):
    """The same model restated in PyTorch (float64): F.conv2d with the SAME padding spelled out (groups=C for the depthwise
    convolutions), F.batch_norm in inference mode, F.layer_norm over the channels, exact F.gelu, F.scaled_dot_product_attention."""
    import torch
    import torch.nn.functional as F
    t = {k: torch.from_numpy(np.asarray(v, np.float64)) for k, v in weights.items()}
    x = torch.from_numpy(np.asarray(img, np.float64)).permute(0, 3, 1, 2)

    def same(x, k, s):
        H, W = x.shape[-2:]
        ph, pw = max((-(-H // s) - 1) * s + k - H, 0), max((-(-W // s) - 1) * s + k - W, 0)
        return F.pad(x, (pw // 2, pw - pw // 2, ph // 2, ph - ph // 2))

    def ln(x, n):
        g, b = t[n + ".g"].reshape(-1), t[n + ".b"].reshape(-1)
        return F.layer_norm(x.permute(0, 2, 3, 1), (x.shape[1],), g, b, LN_EPS).permute(0, 3, 1, 2)

    def pw(x, n, bias=True):
        k = t[n + ".kernel"]
        return F.conv2d(x, k.permute(3, 2, 0, 1), t[n + ".bias"] if bias else None)

    def dwp(x, a, s):
        k = t[a + "0.kernel"]
        y = F.conv2d(same(x, k.shape[0], s), k.permute(3, 2, 0, 1), stride=s, groups=x.shape[1])
        y = F.batch_norm(y, t[a + "1.moving_mean"], t[a + "1.moving_variance"], t[a + "1.gamma"], t[a + "1.beta"], False, 0.0, BN_EPS)
        return pw(y, a + "2", False)

    for st, c in enumerate(stages(cfg)):
        p = f"cvt_layers.{st}."
        k = t[p + "0.kernel"]
        x = F.conv2d(same(x, k.shape[0], c["emb_stride"]), k.permute(3, 2, 0, 1), t[p + "0.bias"], stride=c["emb_stride"])
        x = ln(x, p + "1")
        h = c["heads"]
        for L in range(c["depth"]):
            b = f"{p}2.layers.{L}."
            y = ln(x, b + "0.norm")
            q, kv = dwp(y, b + "0.fn.to_q.net.", 1), dwp(y, b + "0.fn.to_kv.net.", c["kv_proj_stride"])
            kk, v = kv.chunk(2, dim=1)
            q, kk, v = (z.flatten(2).unflatten(1, (h, DIM_HEAD)).transpose(-1, -2) for z in (q, kk, v))   # b h n d
            o = F.scaled_dot_product_attention(q, kk, v)
            o = o.transpose(-1, -2).reshape(x.shape[0], h * DIM_HEAD, *x.shape[-2:])
            x = pw(o, b + "0.fn.to_out.0") + x
            x = pw(F.gelu(pw(ln(x, b + "1.norm"), b + "1.fn.net.0")), b + "1.fn.net.3") + x
    z = x.mean(dim=(2, 3))
    return (z @ t["cvt_layers.3.1.kernel"] + t["cvt_layers.3.1.bias"]).numpy()


def bf16_round(x):
    return levit_oracle.bf16_round(x)


# ------------------------------------------------------------------------------------------------ the reference's cvt.py
def _depthwise_conv2d(base):
    _arr = tf_shim._arr

    class Conv2D(base):
        """cct_oracle's Conv2D plus groups: groups == filters == input channels is the depthwise convolution cvt.py:84 builds."""

        def __init__(self, filters, kernel_size, strides=(1, 1), padding='valid', groups=1, use_bias=True, name=None, **kwargs):
            super().__init__(filters, kernel_size, strides=strides, padding=padding, use_bias=use_bias, name=name, **kwargs)
            self.groups = int(groups)

        def call(self, inputs):
            if self.groups == 1:
                return super().call(inputs)
            x = _arr(inputs)
            k, cin = self.k, x.shape[-1]
            if not cin == self.groups == self.filters:
                raise NotImplementedError("Conv2D: only the depthwise grouping (groups == filters == channels) is used by cvt.py")
            if self.kernel is None:                                       # glorot_uniform: fan_in k^2, fan_out k^2 * filters
                lim = math.sqrt(6.0 / (k * k * (1 + self.filters)))
                self.kernel = tf_shim.Variable(tf_shim._RNG[0].uniform(-lim, lim, size=(k, k, 1, self.filters)))
                if self.use_bias:
                    self.bias = tf_shim.Variable(np.zeros(self.filters))
            p = tf_shim._extract_patches(x, [1, k, k, 1], [1, self.s, self.s, 1], [1, 1, 1, 1], self.padding)
            y = (p.reshape(*p.shape[:3], k * k, cin) * self.kernel.view(np.ndarray).reshape(k * k, cin)).sum(-2)
            return y + self.bias.view(np.ndarray) if self.use_bias else y

    return Conv2D


@contextlib.contextmanager
def installed(reference_dir):
    """levit_oracle.installed(reference_dir) plus what cvt.py needs beyond it; `import cvt` inside the block is the reference's own
    file, removed from sys.modules again on exit."""
    saved = sys.modules.pop("cvt", None)
    with levit_oracle.installed(reference_dir) as tf:
        layers = sys.modules["tensorflow.keras.layers"]
        layers.Conv2D = _depthwise_conv2d(layers.Conv2D)
        arr = tf_shim._arr
        tf.math.reduce_variance = tf_shim._returns_tensor(
            lambda input_tensor, axis=None, keepdims=False, **_: arr(input_tensor).var(axis=axis, keepdims=keepdims))
        tf.sqrt = tf_shim._returns_tensor(lambda x, **_: np.sqrt(arr(x)))
        tf.ones = tf_shim._returns_tensor(lambda shape, dtype=None, **_: np.ones(tuple(shape), dtype=dtype or tf_shim.get_dtype()))
        try:
            yield tf
        finally:
            sys.modules.pop("cvt", None)
            if saved is not None:
                sys.modules["cvt"] = saved


def load_weights(model, w):
    """The oracle's weights into a reference CvT by attribute path (cvt.py:182-198)."""
    seqs = model.cvt_layers.layers
    for st in range(3):
        p = f"cvt_layers.{st}."
        conv, ln, tr = seqs[st].layers
        conv.set_weights([w[p + "0.kernel"], w[p + "0.bias"]])
        ln.g.assign(w[p + "1.g"])
        ln.b.assign(w[p + "1.b"])
        for L, (attn, ff) in enumerate(tr.layers):
            b = f"{p}2.layers.{L}."
            attn.norm.g.assign(w[b + "0.norm.g"])
            attn.norm.b.assign(w[b + "0.norm.b"])
            for n in ("to_q", "to_kv"):
                net = getattr(attn.fn, n).net.layers
                a = f"{b}0.fn.{n}.net."
                net[0].set_weights([w[a + "0.kernel"]])
                net[1].set_weights([w[a + "1." + leaf] for leaf in BN_LEAVES])
                net[2].set_weights([w[a + "2.kernel"]])
            attn.fn.to_out.layers[0].set_weights([w[b + "0.fn.to_out.0.kernel"], w[b + "0.fn.to_out.0.bias"]])
            ff.norm.g.assign(w[b + "1.norm.g"])
            ff.norm.b.assign(w[b + "1.norm.b"])
            ff.fn.net.layers[0].set_weights([w[b + "1.fn.net.0.kernel"], w[b + "1.fn.net.0.bias"]])
            ff.fn.net.layers[3].set_weights([w[b + "1.fn.net.3.kernel"], w[b + "1.fn.net.3.bias"]])
    seqs[3].layers[1].set_weights([w["cvt_layers.3.1.kernel"], w["cvt_layers.3.1.bias"]])


@contextlib.contextmanager
def reference_module(reference_dir, dtype=np.float64):
    """The reference's cvt module over the stand-in in `dtype`."""
    import importlib
    tf_shim.set_dtype(dtype)
    try:
        with installed(reference_dir):
            yield importlib.import_module("cvt")
    finally:
        tf_shim.set_dtype(np.float32)


def reference_logits(mod, cfg, w, img, dtype=np.float64, img_call=None):
    """Build the reference's CvT for `cfg`, call it once on `img` so that Keras builds every variable, load `w` and return
    `model(img_call or img, training=False)`."""
    model = mod.CvT(**ctor_kwargs(cfg))
    model(np.asarray(img, dtype), training=False)
    load_weights(model, {k: np.asarray(v, dtype) for k, v in w.items()})
    out = model(np.asarray(img if img_call is None else img_call, dtype), training=False)
    return np.asarray(out).view(np.ndarray).copy()


def random_config(seed):
    """A small random configuration: kernel sizes 1 / 3 / 5 / 7, kv strides 1 and 2, odd map sizes, widths off 64."""
    r = random.Random(seed)
    kw = dict(num_classes=r.randint(2, 9), dropout=0.0)
    for i in (1, 2, 3):
        kw.update({f"s{i}_emb_dim": r.choice([8, 12, 20, 40, 64, 72]), f"s{i}_emb_kernel": r.choice([1, 2, 3, 5]),
                   f"s{i}_emb_stride": r.choice([1, 2, 2, 3]), f"s{i}_proj_kernel": (1, 3, 5, 7)[(seed + i) % 4],
                   f"s{i}_kv_proj_stride": r.choice([1, 2]), f"s{i}_heads": r.randint(1, 3), f"s{i}_depth": r.randint(0, 2),
                   f"s{i}_mlp_mult": r.randint(1, 3)})
    return make_config(image_size=r.choice([9, 13, 16, 21, 24]), image_w=r.choice([11, 16, 19, 24]), **kw)


# ------------------------------------------------------------------------------------------------ cases
def _small(**kw):
    base = dict(num_classes=10, s1_emb_dim=64, s1_emb_kernel=7, s1_emb_stride=4, s1_heads=1, s1_depth=1, s1_mlp_mult=2,
                s2_emb_dim=64, s2_heads=2, s2_depth=1, s2_mlp_mult=2, s3_emb_dim=128, s3_heads=2, s3_depth=1, s3_mlp_mult=2)
    base.update(kw)
    return base


# small cases (fixtures with float32 and float64 reference logits) and the two configurations tools/cvt_bench.py measures
SMALL = {
    "cvt_small": dict(image_size=64, **_small()),
    # a 52^2 image: maps 13 -> 7 -> 4, the asymmetric SAME padding of every stride-2 convolution on an odd map
    "cvt_odd52": dict(image_size=52, **_small(s2_heads=3, s3_heads=4)),
    "cvt_kv1_k5": dict(image_size=48, **_small(s1_kv_proj_stride=1, s2_proj_kernel=5, s3_kv_proj_stride=1, s3_proj_kernel=5)),
    "cvt_widths": dict(image_size=40, image_w=56, **_small(s1_emb_dim=40, s2_emb_dim=72, s3_emb_dim=40, s2_mlp_mult=3, s3_proj_kernel=7)),
}
BENCH = {
    "cvt_readme": dict(image_size=224, num_classes=1000, s3_heads=4),   # the reference README's model
    "cvt_13": dict(image_size=224, num_classes=1000),                   # the constructor defaults: a CvT-13 shape
}
WEIGHT_SEED, IMAGE_SEED, BATCH = 31, 32, 2

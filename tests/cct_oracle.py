"""Test oracle of the Compact Convolutional Transformer (reference cct.py), kept beside the tests that use it.

  * make_config / weight_specs / init_weights / stress_weights: configs and seeded weights in the engine's names
    (SURVEY.md App. B), the reference's initial distributions;
  * forward: the float64 numpy restatement of CCT.call (cct.py:342-345, TransformerClassifier.call :277-305);
  * forward_torch: an independent PyTorch restatement (conv2d / max_pool2d with explicit asymmetric padding);
  * installed(): oracle/tf_shim.py plus the TensorFlow / Keras entry points only cct.py calls (Conv2D and MaxPool2D with
    'SAME' padding, ReLU, pad, tile, squeeze, sin / cos, linspace, random.truncated_normal), so that the reference's cct.py
    runs unmodified; build_reference loads the oracle's weights into it by attribute path.

The TensorFlow semantics restated here (third-party, public API documentation): Conv2D / MaxPool2D 'SAME' give ceil(in / stride)
positions with total padding max((out - 1) * stride + k - in, 0), the smaller half first; a Conv2D kernel is [k, k, cin, cout]
over (row, column, channel) windows, glorot-uniform with fans k*k*cin / k*k*cout; padded max-pool taps never win;
truncated_normal redraws values beyond two standard deviations.
"""
from __future__ import annotations

import collections
import contextlib
import math
import sys

import numpy as np

from oracle import spec_numpy, tf_shim
from vit_tensorflow_b200.models import CCT_CTOR_KEYS, cct_token_grid, sinusoidal_embedding

# defaults of CCT.__init__ (cct.py:308-317) and of the TransformerClassifier kwargs it forwards (:217-230)
CCT_DEFAULTS = dict(img_size=224, embedding_dim=768, n_input_channels=3, n_conv_layers=1, kernel_size=7, stride=2, pooling_kernel_size=3,
                    pooling_stride=2, num_layers=12, num_heads=12, mlp_ratio=4.0, num_classes=1000, positional_embedding='sine')
FACTORIES = {"cct_2": (2, 2, 1, 128), "cct_4": (4, 2, 1, 128), "cct_6": (6, 4, 2, 256), "cct_7": (7, 4, 2, 256), "cct_8": (8, 4, 2, 256),
             "cct_14": (14, 6, 3, 384), "cct_16": (16, 6, 3, 384)}    # (num_layers, num_heads, mlp_ratio, embedding_dim) cct.py:16-48


def factory_kwargs(name, kernel_size=3, stride=None, **kw):
    """The CCT kwargs a cct_N(...) factory call resolves to (cct.py:51-61)."""
    L, h, r, d = FACTORIES[name]
    stride = stride if stride is not None else max(1, (kernel_size // 2) - 1)
    return dict(num_layers=L, num_heads=h, mlp_ratio=r, embedding_dim=d, kernel_size=kernel_size, stride=stride, **kw)


def make_config(**kw) -> dict:
    cfg = dict(CCT_DEFAULTS)
    cfg.update(kw)
    cfg["kind"] = "cct"
    if cfg["positional_embedding"] not in ('sine', 'learnable', 'none'):
        cfg["positional_embedding"] = 'sine'
    ih, iw = cfg["img_size"] if isinstance(cfg["img_size"], tuple) else (cfg["img_size"], cfg["img_size"])
    gh, gw = cct_token_grid(ih, iw, cfg["n_conv_layers"], cfg["stride"], cfg["pooling_stride"])
    cfg.update(image_h=ih, image_w=iw, channels=3, sequence_length=gh * gw, dim=cfg["embedding_dim"],
               mlp_dim=int(cfg["embedding_dim"] * cfg["mlp_ratio"]), heads=cfg["num_heads"], dim_head=cfg["embedding_dim"] // cfg["num_heads"],
               depth=cfg["num_layers"])
    return cfg


def ctor_kwargs(cfg) -> dict:
    return {k: cfg[k] for k in CCT_CTOR_KEYS if k in cfg}


def weight_specs(cfg):
    s = collections.OrderedDict()
    d, k, L = cfg["dim"], cfg["kernel_size"], cfg["n_conv_layers"]
    for i in range(L):
        cin, cout = (3 if i == 0 else 64), (d if i == L - 1 else 64)
        s[f"tokenizer.conv.{i}.kernel"] = ((k, k, cin, cout), "glorot")
    if cfg["positional_embedding"] != "none":
        s["positional_emb"] = ((1, cfg["sequence_length"], d), cfg["positional_embedding"])
    for n in range(cfg["depth"]):
        p = f"layers.{n}."
        s[p + "attn_norm.gamma"], s[p + "attn_norm.beta"] = ((d,), "ones"), ((d,), "zeros")
        s[p + "to_qkv.kernel"] = ((d, 3 * d), "glorot")
        s[p + "to_out.kernel"], s[p + "to_out.bias"] = ((d, d), "glorot"), ((d,), "zeros")
        s[p + "norm1.gamma"], s[p + "norm1.beta"] = ((d,), "ones"), ((d,), "zeros")
        s[p + "fc1.kernel"], s[p + "fc1.bias"] = ((d, cfg["mlp_dim"]), "glorot"), ((cfg["mlp_dim"],), "zeros")
        s[p + "fc2.kernel"], s[p + "fc2.bias"] = ((cfg["mlp_dim"], d), "glorot"), ((d,), "zeros")
    s["norm.gamma"], s["norm.beta"] = ((d,), "ones"), ((d,), "zeros")
    s["attention_pool.kernel"], s["attention_pool.bias"] = ((d, 1), "glorot"), ((1,), "zeros")
    s["head.kernel"], s["head.bias"] = ((d, cfg["num_classes"]), "glorot"), ((cfg["num_classes"],), "zeros")
    return s


def init_weights(cfg, seed=0):
    rng = np.random.default_rng(seed)
    out = collections.OrderedDict()
    for name, (shape, init) in weight_specs(cfg).items():
        if init == "glorot":
            rf = int(np.prod(shape[:-2]))
            lim = math.sqrt(6.0 / (rf * (shape[-2] + shape[-1])))
            a = rng.uniform(-lim, lim, size=shape)
        elif init == "zeros":
            a = np.zeros(shape)
        elif init == "ones":
            a = np.ones(shape)
        elif init == "sine":
            a = sinusoidal_embedding(shape[1], shape[2])
        elif init == "learnable":
            a = rng.standard_normal(shape)
            while (np.abs(a) > 2).any():
                a[np.abs(a) > 2] = rng.standard_normal(int((np.abs(a) > 2).sum()))
            a = 0.2 * a
        else:
            raise AssertionError(init)
        out[name] = np.ascontiguousarray(a, dtype=np.float32)
    return out


def stress_weights(cfg, seed=1):
    """init_weights with non-zero biases and non-unit LayerNorm affines (wiring bugs cannot hide behind the Keras defaults)."""
    rng = np.random.default_rng(seed)
    out = init_weights(cfg, seed)
    for name, (shape, init) in weight_specs(cfg).items():
        if init == "zeros":
            out[name] = (0.2 * rng.standard_normal(shape)).astype(np.float32)
        elif init == "ones":
            out[name] = (1.0 + 0.2 * rng.standard_normal(shape)).astype(np.float32)
    return out


def make_image(cfg, batch, seed=0, h=None, w=None):
    rng = np.random.default_rng(seed)
    return rng.standard_normal((batch, h or cfg["image_h"], w or cfg["image_w"], 3), dtype=np.float32)


# ------------------------------------------------------------------------------------------------ float64 spec
def maxpool_same(x, k, stride):
    """MaxPool2D(k, stride, 'SAME') NHWC: padded taps are -inf (never win)."""
    b, H, W, C = x.shape
    oh, ow = -(-H // stride), -(-W // stride)
    ph, pw = max((oh - 1) * stride + k - H, 0), max((ow - 1) * stride + k - W, 0)
    xp = np.full((b, H + ph, W + pw, C), -np.inf, x.dtype)
    xp[:, ph // 2:ph // 2 + H, pw // 2:pw // 2 + W] = x
    out = np.full((b, oh, ow, C), -np.inf, x.dtype)
    for i in range(k):
        for j in range(k):
            out = np.maximum(out, xp[:, i:i + (oh - 1) * stride + 1:stride, j:j + (ow - 1) * stride + 1:stride])
    return out


def tokens(img, w, cfg):
    """Tokenizer.call (cct.py:211-215) + the 'none' padding and the positional add of TransformerClassifier.call (:278-286)."""
    x = img
    for i in range(cfg["n_conv_layers"]):
        kern = w[f"tokenizer.conv.{i}.kernel"]
        x = spec_numpy.extract_patches_same(x, cfg["kernel_size"], cfg["stride"]) @ kern.reshape(-1, kern.shape[-1])   # Conv2D SAME
        x = maxpool_same(np.maximum(x, 0), cfg["pooling_kernel_size"], cfg["pooling_stride"])                         # ReLU, MaxPool2D
    b, h, ww, c = x.shape
    x = x.reshape(b, h * ww, c)
    if cfg["positional_embedding"] == "none":
        if x.shape[1] < cfg["sequence_length"]:
            x = np.pad(x, ((0, 0), (0, cfg["sequence_length"] - x.shape[1]), (0, 0)))
    else:
        x = x + w["positional_emb"]
    return x


def forward(img, weights, cfg, dtype=np.float64):
    w = {k: np.asarray(v, dtype=dtype) for k, v in weights.items()}
    x = tokens(np.asarray(img, dtype=dtype), w, cfg)
    for n in range(cfg["depth"]):                                                   # TransformerEncoderLayer.call :159-174
        p = f"layers.{n}."
        x = x + spec_numpy.attention_vit(spec_numpy.layer_norm(x, w, p + "attn_norm"), w, p, cfg["heads"], cfg["dim_head"])
        x = spec_numpy.layer_norm(x, w, p + "norm1")
        x = x + spec_numpy.mlp(x, w, p)
    x = spec_numpy.layer_norm(x, w, "norm")                                         # :291
    a = spec_numpy.dense(x, w, "attention_pool")                                    # :295 [b, n, 1]
    a = np.exp(a - a.max(axis=1, keepdims=True))
    a = a / a.sum(axis=1, keepdims=True)                                            # softmax over the tokens :296
    z = (a * x).sum(axis=1)                                                         # :297-299
    return spec_numpy.dense(z, w, "head")                                           # :303


def forward_torch(img, weights, cfg):
    """The same model restated in PyTorch (float64): conv2d / max_pool2d with the SAME padding spelled out (F.pad, -inf for the
    pool), nn.functional.layer_norm / softmax / gelu."""
    import torch
    import torch.nn.functional as F
    t = {k: torch.from_numpy(np.asarray(v, np.float64)) for k, v in weights.items()}
    x = torch.from_numpy(np.asarray(img, np.float64)).permute(0, 3, 1, 2)

    def same_pad(x, k, s, value):
        H, W = x.shape[-2:]
        oh, ow = -(-H // s), -(-W // s)
        ph, pw = max((oh - 1) * s + k - H, 0), max((ow - 1) * s + k - W, 0)
        return F.pad(x, (pw // 2, pw - pw // 2, ph // 2, ph - ph // 2), value=value)

    for i in range(cfg["n_conv_layers"]):
        k = cfg["kernel_size"]
        x = F.conv2d(same_pad(x, k, cfg["stride"], 0.0), t[f"tokenizer.conv.{i}.kernel"].permute(3, 2, 0, 1), stride=cfg["stride"])
        x = F.max_pool2d(same_pad(F.relu(x), cfg["pooling_kernel_size"], cfg["pooling_stride"], -math.inf), cfg["pooling_kernel_size"],
                         cfg["pooling_stride"])
    x = x.flatten(2).transpose(1, 2)
    if cfg["positional_embedding"] == "none":
        x = F.pad(x, (0, 0, 0, max(cfg["sequence_length"] - x.shape[1], 0)))
    else:
        x = x + t["positional_emb"]
    d, h = cfg["dim"], cfg["heads"]

    def ln(x, n):
        return F.layer_norm(x, (d,), t[n + ".gamma"], t[n + ".beta"], eps=1e-3)

    for n in range(cfg["depth"]):
        p = f"layers.{n}."
        q, kk, v = (ln(x, p + "attn_norm") @ t[p + "to_qkv.kernel"]).chunk(3, dim=-1)
        q, kk, v = (y.unflatten(-1, (h, d // h)).transpose(1, 2) for y in (q, kk, v))
        o = torch.softmax(q @ kk.transpose(-1, -2) * (d // h) ** -0.5, dim=-1) @ v
        x = x + o.transpose(1, 2).flatten(2) @ t[p + "to_out.kernel"] + t[p + "to_out.bias"]
        x = ln(x, p + "norm1")
        x = x + F.gelu(x @ t[p + "fc1.kernel"] + t[p + "fc1.bias"]) @ t[p + "fc2.kernel"] + t[p + "fc2.bias"]
    x = ln(x, "norm")
    a = torch.softmax(x @ t["attention_pool.kernel"] + t["attention_pool.bias"], dim=1)
    return ((a * x).sum(1) @ t["head.kernel"] + t["head.bias"]).numpy()


# ------------------------------------------------------------------------------------------------ the reference's cct.py
def _shim_layers():
    _arr = tf_shim._arr

    class Conv2D(tf_shim._Weighted):
        _order = ("kernel", "bias")

        def __init__(self, filters, kernel_size, strides=(1, 1), padding='valid', use_bias=True, name=None, **kwargs):
            super().__init__(name=name)
            self.filters, self.use_bias = int(filters), bool(use_bias)
            self.k = kernel_size if isinstance(kernel_size, int) else kernel_size[0]
            self.s = strides if isinstance(strides, int) else strides[0]
            self.padding = padding.upper()
            self.kernel = self.bias = None

        def call(self, inputs):
            x = _arr(inputs)
            k, cin = self.k, x.shape[-1]
            if self.kernel is None:                                       # glorot_uniform over the receptive field / zeros
                lim = math.sqrt(6.0 / (k * k * (cin + self.filters)))
                self.kernel = tf_shim.Variable(tf_shim._RNG[0].uniform(-lim, lim, size=(k, k, cin, self.filters)))
                if self.use_bias:
                    self.bias = tf_shim.Variable(np.zeros(self.filters))
            p = tf_shim._extract_patches(x, [1, k, k, 1], [1, self.s, self.s, 1], [1, 1, 1, 1], self.padding)
            y = p @ self.kernel.view(np.ndarray).reshape(k * k * cin, self.filters)
            return y + self.bias.view(np.ndarray) if self.use_bias else y

    class MaxPool2D(tf_shim.Layer):
        def __init__(self, pool_size=(2, 2), strides=None, padding='valid', name=None, **kwargs):
            super().__init__(name=name)
            self.k = pool_size if isinstance(pool_size, int) else pool_size[0]
            s = strides if strides is not None else self.k
            self.s = s if isinstance(s, int) else s[0]
            if padding.upper() != "SAME":
                raise NotImplementedError("MaxPool2D: only padding='SAME' is used by cct.py")

        def call(self, inputs):
            return maxpool_same(_arr(inputs), self.k, self.s)

    class ReLU(tf_shim.Layer):
        def call(self, inputs):
            return np.maximum(_arr(inputs), 0)

    return Conv2D, MaxPool2D, ReLU


def _truncated_normal(shape, mean=0.0, stddev=1.0, dtype=None, **_):
    a = tf_shim._RNG[0].standard_normal(tuple(shape))
    while (np.abs(a) > 2).any():
        a[np.abs(a) > 2] = tf_shim._RNG[0].standard_normal(int((np.abs(a) > 2).sum()))
    return (mean + stddev * a).astype(dtype or tf_shim.get_dtype())


@contextlib.contextmanager
def installed(reference_dir):
    """tf_shim.installed(reference_dir) plus what cct.py needs beyond the other modules; `import cct` inside the block is the
    reference's own file, removed from sys.modules again on exit."""
    saved = sys.modules.pop("cct", None)
    with tf_shim.installed(reference_dir) as tf:
        Conv2D, MaxPool2D, ReLU = _shim_layers()
        layers = sys.modules["tensorflow.keras.layers"]
        layers.Conv2D, layers.MaxPool2D, layers.ReLU = Conv2D, MaxPool2D, ReLU
        arr = tf_shim._arr
        extra = dict(
            sin=lambda x: np.sin(arr(x)), cos=lambda x: np.cos(arr(x)), floor=lambda x: np.floor(arr(x)),
            divide=lambda x, y: np.divide(arr(x), y), rank=lambda x: np.asarray(np.ndim(x), np.int32),
            pad=lambda tensor, paddings, mode="CONSTANT", constant_values=0, **_: np.pad(arr(tensor), paddings, constant_values=constant_values),
            tile=lambda input, multiples, **_: np.tile(arr(input), multiples),
            squeeze=lambda input, axis=None, **_: np.squeeze(arr(input), axis=axis))
        for k, f in extra.items():
            setattr(tf, k, tf_shim._returns_tensor(f))
        # the elements answer .numpy() (cct.py:259): a list of 0-d tensors
        tf.linspace = lambda start, stop, num, **_: [np.asarray(v).view(tf_shim.Tensor) for v in np.linspace(start, stop, num)]
        tf.random.truncated_normal = tf_shim._returns_tensor(_truncated_normal)
        try:
            yield tf
        finally:
            sys.modules.pop("cct", None)
            if saved is not None:
                sys.modules["cct"] = saved


def load_weights(model, w):
    """The oracle's weights into a reference CCT by attribute path (cct.py:188-202,244-267)."""
    convs = model.tokenizer.conv_layers.layers                       # [Conv2D, ReLU, MaxPool2D] per conv layer
    i = 0
    while f"tokenizer.conv.{i}.kernel" in w:
        convs[3 * i].set_weights([w[f"tokenizer.conv.{i}.kernel"]])
        i += 1
    c = model.classifier
    if c.positional_emb is not None:
        c.positional_emb.assign(w["positional_emb"])
    for n, blk in enumerate(c.blocks.layers):
        p = f"layers.{n}."
        blk.pre_norm.set_weights([w[p + "attn_norm.gamma"], w[p + "attn_norm.beta"]])
        blk.self_attn.to_qkv.set_weights([w[p + "to_qkv.kernel"]])
        blk.self_attn.proj.layers[0].set_weights([w[p + "to_out.kernel"], w[p + "to_out.bias"]])
        blk.norm1.set_weights([w[p + "norm1.gamma"], w[p + "norm1.beta"]])
        blk.linear1.set_weights([w[p + "fc1.kernel"], w[p + "fc1.bias"]])
        blk.linear2.set_weights([w[p + "fc2.kernel"], w[p + "fc2.bias"]])
    c.norm.set_weights([w["norm.gamma"], w["norm.beta"]])
    c.attention_pool.set_weights([w["attention_pool.kernel"], w["attention_pool.bias"]])
    c.fc.set_weights([w["head.kernel"], w["head.bias"]])


def reference_logits(cfg, w, img, dtype=np.float64, reference_dir=None, img_call=None):
    """Build the reference's CCT for `cfg` over the shim in `dtype`, run it once on a config-size image so that Keras builds its
    variables, load `w`, and return `model(img_call or img, training=False)`."""
    import importlib
    tf_shim.set_dtype(dtype)
    try:
        with installed(reference_dir):
            model = importlib.import_module("cct").CCT(**ctor_kwargs(cfg))
            model(np.asarray(img, dtype), training=False)
            load_weights(model, {k: np.asarray(v, dtype) for k, v in w.items()})
            x = img if img_call is None else img_call
            return np.asarray(model(np.asarray(x, dtype), training=False)).view(np.ndarray).copy()
    finally:
        tf_shim.set_dtype(np.float32)


# ------------------------------------------------------------------------------------------------ cases
# small cases (fixtures with float32 and float64 reference logits) and the two configurations tools/cct_bench.py measures
SMALL = {
    "cct_small_sine": dict(img_size=32, embedding_dim=64, n_conv_layers=2, kernel_size=3, stride=1, num_layers=2, num_heads=2,
                           mlp_ratio=2, num_classes=10),
    "cct_small_learnable": dict(img_size=(24, 40), embedding_dim=128, n_conv_layers=1, kernel_size=7, stride=2, num_layers=2,
                                num_heads=2, mlp_ratio=1, num_classes=7, positional_embedding='learnable'),
    "cct_small_none": dict(img_size=20, embedding_dim=48, n_conv_layers=1, kernel_size=3, stride=1, pooling_kernel_size=3,
                           pooling_stride=2, num_layers=1, num_heads=3, mlp_ratio=1.5, num_classes=5, positional_embedding='none'),
}
BENCH = {
    "cct_14_7x2": factory_kwargs("cct_14", img_size=224, kernel_size=7, n_conv_layers=2),    # ImageNet: 196 tokens, dim 384
    "cct_7_3x1": factory_kwargs("cct_7", img_size=32, kernel_size=3, n_conv_layers=1, num_classes=10),   # CIFAR: 256 tokens, dim 256
}
WEIGHT_SEED, IMAGE_SEED, BATCH = 11, 12, 2

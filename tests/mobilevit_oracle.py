"""Test oracle of MobileViT (reference mobile_vit.py), kept beside the tests that use it.

  * make_config / weight_specs / init_weights / stress_weights: configs and seeded weights in the engine's names (SURVEY.md
    App. B: the reference's attribute paths), the reference's initial distributions;
  * forward: the float64 numpy restatement of MobileViT.call (mobile_vit.py:260-271) with inference BatchNormalization;
  * forward_torch: an independent PyTorch restatement (conv2d with the asymmetric SAME padding spelled out, grouped depthwise
    convolutions, F.batch_norm, F.silu, F.layer_norm);
  * installed(): levit_oracle's stand-in plus what mobile_vit.py calls beyond it (Conv2D with groups, at any stride,
    tf.keras.activations.swish, and tf.transpose with a perm shorter than the rank), so that the reference's mobile_vit.py runs
    unmodified; reference_logits loads the oracle's weights by attribute path.

One quirk of the reference is resolved here rather than reproduced: mobile_vit.py:101 transposes the 5-D k [b, p, h, n, d] with the
4-entry perm [0, 1, 3, 2], which TensorFlow refuses (perm must have the tensor's rank).  The stand-in applies such a perm to the
trailing axes, which is the evident intent (k^T per head, as vit.py's attention does), and the engine computes that.

The TensorFlow semantics restated here (third-party, public API documentation): Conv2D with groups = g splits the input channels
into g groups and filter f reads group f // (filters / g); padding 'SAME' pads max((out - 1) * stride + k - in, 0) in total with
the smaller half first; swish(x) = x * sigmoid(x); BatchNormalization at inference normalises with moving_mean / moving_variance
(epsilon added to the variance); LayerNormalization uses the biased variance, epsilon 1e-3 by default.
"""
from __future__ import annotations

import collections
import contextlib
import math
import sys

import numpy as np

import levit_oracle
from oracle import spec_numpy, tf_shim
from vit_tensorflow_b200.models import MOBILEVIT_CTOR_KEYS

MOBILEVIT_DEFAULTS = dict(expansion=4, kernel_size=3, patch_size=(2, 2), depths=(2, 4, 3))   # mobile_vit.py:210-219
BN_EPS, LN_EPS = 1e-5, 1e-3
BN_LEAVES = levit_oracle.BN_LEAVES
HEADS, DH = 4, 8                                                                             # mobile_vit.py:182


def make_config(**kw) -> dict:
    cfg = dict(MOBILEVIT_DEFAULTS)
    cfg.update(kw)
    cfg["kind"] = "mobilevit"
    return cfg


def ctor_kwargs(cfg) -> dict:
    return {k: cfg[k] for k in MOBILEVIT_CTOR_KEYS if k in cfg}


def mlp_dims(cfg):
    return tuple(int(cfg["dims"][s] * m) for s, m in enumerate((2, 4, 4)))                  # mobile_vit.py:241,246,251


def blocks(cfg):
    """The seven MV2 blocks as mobile_vit.py:233-252 wires them, restated here from `channels` and `expansion` alone: (attribute path,
    width of the input the block reads, hidden, output width, stride, expand convolution present, residual).  MV2Block(dim_in,
    dim_out, stride) (:131-137) takes hidden = int(dim_in * expansion) and adds its input iff stride == 1 and dim_in == dim_out;
    Keras infers the input width from the previous block's output, which for the fourth stem block is channels[3], not its
    dim_in = channels[2]."""
    c, e = cfg["channels"], cfg["expansion"]
    wiring = [("stem.0", c[0], c[1], 1), ("stem.1", c[1], c[2], 2), ("stem.2", c[2], c[3], 1), ("stem.3", c[2], c[3], 1),
              ("trunk.0.0", c[3], c[4], 2), ("trunk.1.0", c[5], c[6], 2), ("trunk.2.0", c[7], c[8], 2)]
    out, width = [], c[0]                                       # conv1's output feeds the stem
    for path, dim_in, dim_out, stride in wiring:
        if path.startswith("trunk."):
            width = c[3 + 2 * int(path[6])]                     # the stem's output, then MobileViTBlock(channels[5 | 7])
        out.append((path, width, int(dim_in * e), dim_out, stride, e != 1, stride == 1 and dim_in == dim_out))
        width = dim_out
    return out


def mv2_prefix(path):
    return path + ".conv."


def weight_specs(cfg):
    s = collections.OrderedDict()
    ch, k = cfg["channels"], cfg["kernel_size"]

    def bn(n, d):
        for leaf in BN_LEAVES:
            s[f"{n}.{leaf}"] = ((d,), leaf)

    def cbn(n, kk, cin, cout):
        s[f"{n}.layers.0.kernel"] = ((kk, kk, cin, cout), "glorot")
        bn(f"{n}.layers.1", cout)

    cbn("conv1", 3, 3, ch[0])
    for path, cin, hid, cout, _, expand, _ in blocks(cfg):
        p = mv2_prefix(path)
        if expand:
            s[p + "0.kernel"] = ((1, 1, cin, hid), "glorot"); bn(p + "1", hid)
            s[p + "3.kernel"] = ((3, 3, 1, hid), "glorot"); bn(p + "4", hid)
            s[p + "6.kernel"] = ((1, 1, hid, cout), "glorot"); bn(p + "7", cout)
        else:
            s[p + "0.kernel"] = ((3, 3, 1, hid), "glorot"); bn(p + "1", hid)
            s[p + "3.kernel"] = ((1, 1, hid, cout), "glorot"); bn(p + "4", cout)
    for st in range(3):
        p, d, c, cin, mlp = f"trunk.{st}.1.", cfg["dims"][st], ch[5 + 2 * st], ch[4 + 2 * st], mlp_dims(cfg)[st]
        cbn(p + "conv1", k, cin, c)
        cbn(p + "conv2", 1, c, d)
        for L in range(cfg["depths"][st]):
            b = f"{p}transformer.layers.{L}."
            s[b + "0.norm.gamma"], s[b + "0.norm.beta"] = ((d,), "gamma"), ((d,), "beta")
            s[b + "0.fn.to_qkv.kernel"] = ((d, 3 * HEADS * DH), "glorot")
            s[b + "0.fn.to_out.0.kernel"], s[b + "0.fn.to_out.0.bias"] = ((HEADS * DH, d), "glorot"), ((d,), "zeros")
            s[b + "1.norm.gamma"], s[b + "1.norm.beta"] = ((d,), "gamma"), ((d,), "beta")
            s[b + "1.fn.net.0.kernel"], s[b + "1.fn.net.0.bias"] = ((d, mlp), "glorot"), ((mlp,), "zeros")
            s[b + "1.fn.net.3.kernel"], s[b + "1.fn.net.3.bias"] = ((mlp, d), "glorot"), ((d,), "zeros")
        cbn(p + "conv3", 1, d, c)
        cbn(p + "conv4", k, c + cin, c)
    cbn("to_logits.0", 1, ch[9], ch[-1])
    s["to_logits.2.kernel"] = ((ch[-1], cfg["num_classes"]), "glorot")
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
        else:
            raise AssertionError(init)
        out[name] = np.ascontiguousarray(a, dtype=np.float32)
    return out


def stress_weights(cfg, seed=1):
    """init_weights with what the Keras defaults hide: non-zero biases, betas and moving means (N(0, 0.3)), gammas around 1 and
    moving variances in [0.3, 3] -- BatchNorms far from the identity."""
    rng = np.random.default_rng(seed)
    out = init_weights(cfg, seed)
    for name, (shape, init) in weight_specs(cfg).items():
        if init == "gamma":
            a = 1.0 + 0.25 * rng.standard_normal(shape)
        elif init in ("zeros", "beta", "moving_mean"):
            a = 0.3 * rng.standard_normal(shape)
        elif init == "moving_variance":
            a = rng.uniform(0.3, 3.0, size=shape)
        else:
            continue
        out[name] = a.astype(np.float32)
    return out


def make_image(cfg, batch, seed=0, h=None, w=None):
    rng = np.random.default_rng(seed)
    ih, iw = cfg["image_size"]
    return rng.standard_normal((batch, h or ih, w or iw, 3), dtype=np.float32)


# ------------------------------------------------------------------------------------------------ float64 spec
def silu(x):
    return x / (1.0 + np.exp(-x))


def _bn(x, w, n):
    return (x - w[n + ".moving_mean"]) / np.sqrt(w[n + ".moving_variance"] + BN_EPS) * w[n + ".gamma"] + w[n + ".beta"]


def _conv(x, kern, stride):
    """Conv2D SAME without bias, kernel [k, k, cin, cout]."""
    return spec_numpy.extract_patches_same(x, kern.shape[0], stride) @ kern.reshape(-1, kern.shape[-1])


def _dwconv(x, kern, stride):
    """Depthwise Conv2D SAME (groups = channels), kernel [3, 3, 1, C]."""
    p = spec_numpy.extract_patches_same(x, 3, stride)
    b, oh, ow, _ = p.shape
    return (p.reshape(b, oh, ow, 9, -1) * kern.reshape(9, -1)).sum(-2)


def _cbn(x, w, n, stride=1):
    return silu(_bn(_conv(x, w[n + ".layers.0.kernel"], stride), w, n + ".layers.1"))


def _ln(x, w, n):
    mu = x.mean(-1, keepdims=True)
    var = ((x - mu) ** 2).mean(-1, keepdims=True)
    return (x - mu) / np.sqrt(var + LN_EPS) * w[n + ".gamma"] + w[n + ".beta"]


def mv2(x, w, path, stride, expand, residual):
    p = mv2_prefix(path)
    y = x
    if expand:
        y = silu(_bn(_conv(y, w[p + "0.kernel"], 1), w, p + "1"))
        y = silu(_bn(_dwconv(y, w[p + "3.kernel"], stride), w, p + "4"))
        y = _bn(_conv(y, w[p + "6.kernel"], 1), w, p + "7")
    else:
        y = silu(_bn(_dwconv(y, w[p + "0.kernel"], stride), w, p + "1"))
        y = _bn(_conv(y, w[p + "3.kernel"], 1), w, p + "4")
    return y + x if residual else y


def attention(x, w, n):
    """Attention.call (mobile_vit.py:95-107) on x [b, p, n, d]."""
    qkv = x @ w[n + "to_qkv.kernel"]
    b, P, N, _ = x.shape
    q, k, v = (t.reshape(b, P, N, HEADS, DH).transpose(0, 1, 3, 2, 4) for t in np.split(qkv, 3, axis=-1))
    dots = q @ k.transpose(0, 1, 2, 4, 3) * DH ** -0.5
    a = np.exp(dots - dots.max(-1, keepdims=True))
    a = a / a.sum(-1, keepdims=True)
    o = (a @ v).transpose(0, 1, 3, 2, 4).reshape(b, P, N, HEADS * DH)
    return o @ w[n + "to_out.0.kernel"] + w[n + "to_out.0.bias"]


def mobilevit_block(x, w, cfg, st):
    p, (ph, pw) = f"trunk.{st}.1.", cfg["patch_size"]
    y = x
    x = _cbn(_cbn(x, w, p + "conv1"), w, p + "conv2")
    b, H, W, d = x.shape
    h, wd = H // ph, W // pw
    t = x.reshape(b, h, ph, wd, pw, d).transpose(0, 2, 4, 1, 3, 5).reshape(b, ph * pw, h * wd, d)   # 'b (h ph) (w pw) d -> b (ph pw) (h w) d'
    for L in range(cfg["depths"][st]):
        n = f"{p}transformer.layers.{L}."
        t = attention(_ln(t, w, n + "0.norm"), w, n + "0.fn.") + t
        hdn = silu(_ln(t, w, n + "1.norm") @ w[n + "1.fn.net.0.kernel"] + w[n + "1.fn.net.0.bias"])
        t = hdn @ w[n + "1.fn.net.3.kernel"] + w[n + "1.fn.net.3.bias"] + t
    x = t.reshape(b, ph, pw, h, wd, d).transpose(0, 3, 1, 4, 2, 5).reshape(b, H, W, d)
    x = _cbn(x, w, p + "conv3")
    return _cbn(np.concatenate([x, y], -1), w, p + "conv4")


def forward(img, weights, cfg, dtype=np.float64):
    """MobileViT.call(img, training=False): logits [b, num_classes]."""
    w = {k: np.asarray(v, dtype=dtype) for k, v in weights.items()}
    x = _cbn(np.asarray(img, dtype=dtype), w, "conv1", 2)
    mv2s = blocks(cfg)
    for path, _, _, _, stride, expand, residual in mv2s[:4]:
        x = mv2(x, w, path, stride, expand, residual)
    for st in range(3):
        path, _, _, _, stride, expand, residual = mv2s[4 + st]
        x = mobilevit_block(mv2(x, w, path, stride, expand, residual), w, cfg, st)
    z = _cbn(x, w, "to_logits.0").mean(axis=(1, 2))
    return z @ w["to_logits.2.kernel"]


def forward_torch(img, weights, cfg):
    """The same model restated in PyTorch (float64): F.conv2d with the SAME padding spelled out (groups for the depthwise
    convolutions), F.batch_norm in inference mode, F.silu, F.layer_norm, softmax attention on explicit reshapes."""
    import torch
    import torch.nn.functional as F
    t = {k: torch.from_numpy(np.asarray(v, np.float64)) for k, v in weights.items()}
    x = torch.from_numpy(np.asarray(img, np.float64)).permute(0, 3, 1, 2)

    def conv(x, n, stride=1, groups=1):
        kern = t[n]
        k = kern.shape[0]
        H, W = x.shape[-2:]
        ph, pw = max((-(-H // stride) - 1) * stride + k - H, 0), max((-(-W // stride) - 1) * stride + k - W, 0)
        x = F.pad(x, (pw // 2, pw - pw // 2, ph // 2, ph - ph // 2))
        return F.conv2d(x, kern.permute(3, 2, 0, 1), None, stride=stride, groups=groups)

    def bn(x, n):
        return F.batch_norm(x, t[n + ".moving_mean"], t[n + ".moving_variance"], t[n + ".gamma"], t[n + ".beta"], False, 0.0, BN_EPS)

    def cbn(x, n, stride=1):
        return F.silu(bn(conv(x, n + ".layers.0.kernel", stride), n + ".layers.1"))

    x = cbn(x, "conv1", 2)
    mv2s = blocks(cfg)

    def mv2_t(x, path, stride, expand, residual):
        p = mv2_prefix(path)
        if expand:
            y = F.silu(bn(conv(x, p + "0.kernel"), p + "1"))
            y = F.silu(bn(conv(y, p + "3.kernel", stride, y.shape[1]), p + "4"))
            y = bn(conv(y, p + "6.kernel"), p + "7")
        else:
            y = F.silu(bn(conv(x, p + "0.kernel", stride, x.shape[1]), p + "1"))
            y = bn(conv(y, p + "3.kernel"), p + "4")
        return y + x if residual else y

    for path, _, _, _, stride, expand, residual in mv2s[:4]:
        x = mv2_t(x, path, stride, expand, residual)
    ph, pw = cfg["patch_size"]
    for st in range(3):
        path, _, _, _, stride, expand, residual = mv2s[4 + st]
        x = mv2_t(x, path, stride, expand, residual)
        p = f"trunk.{st}.1."
        y = x
        x = cbn(cbn(x, p + "conv1"), p + "conv2")
        b, d, H, W = x.shape
        h, wd = H // ph, W // pw
        s = x.reshape(b, d, h, ph, wd, pw).permute(0, 3, 5, 2, 4, 1).reshape(b, ph * pw, h * wd, d)
        for L in range(cfg["depths"][st]):
            n = f"{p}transformer.layers.{L}."
            a = F.layer_norm(s, (d,), t[n + "0.norm.gamma"], t[n + "0.norm.beta"], LN_EPS)
            q, k, v = (z.unflatten(-1, (HEADS, DH)).transpose(2, 3) for z in (a @ t[n + "0.fn.to_qkv.kernel"]).chunk(3, dim=-1))
            o = torch.softmax(q @ k.transpose(-1, -2) * DH ** -0.5, dim=-1) @ v
            s = o.transpose(2, 3).flatten(-2) @ t[n + "0.fn.to_out.0.kernel"] + t[n + "0.fn.to_out.0.bias"] + s
            a = F.layer_norm(s, (d,), t[n + "1.norm.gamma"], t[n + "1.norm.beta"], LN_EPS)
            s = F.silu(a @ t[n + "1.fn.net.0.kernel"] + t[n + "1.fn.net.0.bias"]) @ t[n + "1.fn.net.3.kernel"] + t[n + "1.fn.net.3.bias"] + s
        x = s.reshape(b, ph, pw, h, wd, d).permute(0, 5, 3, 1, 4, 2).reshape(b, d, H, W)
        x = cbn(x, p + "conv3")
        x = cbn(torch.cat([x, y], dim=1), p + "conv4")
    z = cbn(x, "to_logits.0").mean(dim=(2, 3))
    return (z @ t["to_logits.2.kernel"]).numpy()


# ------------------------------------------------------------------------------------------------ the reference's mobile_vit.py
def _grouped_conv2d(base):
    """cct_oracle's Conv2D stand-in with Keras' `groups`: the kernel is [k, k, cin / groups, filters] and filter f reads input group
    f // (filters / groups)."""
    _arr = tf_shim._arr

    class Conv2D(base):
        def __init__(self, filters, kernel_size, strides=(1, 1), padding='valid', use_bias=True, groups=1, name=None, **kwargs):
            super().__init__(filters, kernel_size, strides=strides, padding=padding, use_bias=use_bias, name=name, **kwargs)
            self.groups = int(groups)

        def call(self, inputs):
            if self.groups == 1:
                return super().call(inputs)
            x = _arr(inputs)
            k, cin, g = self.k, x.shape[-1], self.groups
            if cin % g or self.filters % g:
                raise ValueError(f"Conv2D: {cin} input channels and {self.filters} filters are not divisible by groups={g}")
            cg, fg = cin // g, self.filters // g
            if self.kernel is None:
                lim = math.sqrt(6.0 / (k * k * (cg + self.filters)))
                self.kernel = tf_shim.Variable(tf_shim._RNG[0].uniform(-lim, lim, size=(k, k, cg, self.filters)))
                if self.use_bias:
                    self.bias = tf_shim.Variable(np.zeros(self.filters))
            p = tf_shim._extract_patches(x, [1, k, k, 1], [1, self.s, self.s, 1], [1, 1, 1, 1], self.padding)
            b, oh, ow, _ = p.shape
            p = p.reshape(b, oh, ow, k * k, g, cg)
            kern = self.kernel.view(np.ndarray).reshape(k * k, cg, g, fg)
            y = np.einsum("bhwtgc,tcgf->bhwgf", p, kern).reshape(b, oh, ow, self.filters)
            return y + self.bias.view(np.ndarray) if self.use_bias else y

    return Conv2D


@contextlib.contextmanager
def installed(reference_dir):
    """levit_oracle.installed(reference_dir) plus what mobile_vit.py needs beyond it; `import mobile_vit` inside the block is the
    reference's own file, removed from sys.modules again on exit."""
    saved = sys.modules.pop("mobile_vit", None)
    with levit_oracle.installed(reference_dir) as tf:
        layers = sys.modules["tensorflow.keras.layers"]
        layers.Conv2D = _grouped_conv2d(layers.Conv2D)
        tf.keras.activations = tf_shim._module("tensorflow.keras.activations",
                                               swish=tf_shim._returns_tensor(lambda x: silu(tf_shim._arr(x))))
        plain_transpose = tf.transpose

        def transpose(a, perm=None, **kw):                  # a short perm permutes the trailing axes (see the module docstring)
            x = tf_shim._arr(a)
            if perm is not None and len(perm) < x.ndim:
                lead = x.ndim - len(perm)
                perm = list(range(lead)) + [lead + p for p in perm]
            return plain_transpose(x, perm, **kw)
        tf.transpose = transpose
        try:
            yield tf
        finally:
            sys.modules.pop("mobile_vit", None)
            if saved is not None:
                sys.modules["mobile_vit"] = saved


def load_weights(model, w, cfg):
    """The oracle's weights into a reference MobileViT by attribute path (mobile_vit.py:230-258)."""
    def cbn(layer, n):
        layer.layers.layers[0].set_weights([w[n + ".layers.0.kernel"]])
        layer.layers.layers[1].set_weights([w[f"{n}.layers.1.{leaf}"] for leaf in BN_LEAVES])

    def mv2_load(block, path, expand):
        seq, p = block.conv.layers, mv2_prefix(path)
        for j in ((0, 3, 6) if expand else (0, 3)):
            seq[j].set_weights([w[f"{p}{j}.kernel"]])
            seq[j + 1].set_weights([w[f"{p}{j + 1}.{leaf}"] for leaf in BN_LEAVES])

    cbn(model.conv1, "conv1")
    mv2s = blocks(cfg)
    for i, blk in enumerate(model.stem.layers):
        mv2_load(blk, mv2s[i][0], mv2s[i][5])
    for st, (conv, attn) in enumerate(model.trunk):
        mv2_load(conv, mv2s[4 + st][0], mv2s[4 + st][5])
        p = f"trunk.{st}.1."
        for n in ("conv1", "conv2", "conv3", "conv4"):
            cbn(getattr(attn, n), p + n)
        for L, (a, f) in enumerate(attn.transformer.layers):
            b = f"{p}transformer.layers.{L}."
            a.norm.set_weights([w[b + "0.norm.gamma"], w[b + "0.norm.beta"]])
            a.fn.to_qkv.set_weights([w[b + "0.fn.to_qkv.kernel"]])
            a.fn.to_out.layers[0].set_weights([w[b + "0.fn.to_out.0.kernel"], w[b + "0.fn.to_out.0.bias"]])
            f.norm.set_weights([w[b + "1.norm.gamma"], w[b + "1.norm.beta"]])
            f.fn.net.layers[0].set_weights([w[b + "1.fn.net.0.kernel"], w[b + "1.fn.net.0.bias"]])
            f.fn.net.layers[3].set_weights([w[b + "1.fn.net.3.kernel"], w[b + "1.fn.net.3.bias"]])
    cbn(model.to_logits.layers[0], "to_logits.0")
    model.to_logits.layers[2].set_weights([w["to_logits.2.kernel"]])


@contextlib.contextmanager
def reference_module(reference_dir, dtype=np.float64):
    """The reference's mobile_vit module over the stand-in in `dtype`."""
    import importlib
    tf_shim.set_dtype(dtype)
    try:
        with installed(reference_dir):
            yield importlib.import_module("mobile_vit")
    finally:
        tf_shim.set_dtype(np.float32)


def reference_logits(mod, cfg, w, img, dtype=np.float64):
    """Build the reference's MobileViT for `cfg`, call it once on `img` so that Keras builds every variable, load `w` and return
    `model(img, training=False)`."""
    model = mod.MobileViT(**ctor_kwargs(cfg))
    model(np.asarray(img, dtype), training=False)
    load_weights(model, {k: np.asarray(v, dtype) for k, v in w.items()}, cfg)
    return np.asarray(model(np.asarray(img, dtype), training=False)).view(np.ndarray).copy()


# ------------------------------------------------------------------------------------------------ cases
XS = dict(dims=(96, 120, 144), channels=(16, 32, 48, 48, 64, 64, 80, 80, 96, 96, 384))                # the reference's usage block
XXS = dict(dims=(64, 80, 96), channels=(16, 16, 24, 24, 48, 48, 64, 64, 80, 80, 320), expansion=2)
S = dict(dims=(144, 192, 240), channels=(16, 32, 64, 64, 96, 96, 128, 128, 160, 160, 640))
# small cases (fixtures with float64 reference logits): a square and a rectangular image, patch (2, 2) and (2, 4), kernel_size 3
# and 5, expansion 4, 2 and 1, channels[2] != channels[3] with expansion != 1, widths off a multiple of 64
SMALL = {
    "mobilevit_sq": dict(image_size=(64, 64), num_classes=10, dims=(24, 40, 48), channels=(8, 16, 24, 24, 32, 32, 40, 40, 48, 48, 96),
                         depths=(1, 2, 1)),
    "mobilevit_rect_p24": dict(image_size=(64, 128), num_classes=7, dims=(32, 24, 40), channels=(8, 12, 20, 28, 36, 24, 44, 36, 52, 40, 72),
                               expansion=2, patch_size=(2, 4), depths=(2, 1, 1)),
    "mobilevit_k5_e1": dict(image_size=(128, 64), num_classes=5, dims=(16, 24, 32), channels=(16, 16, 24, 24, 24, 40, 40, 56, 56, 72, 80),
                            expansion=1, kernel_size=5, depths=(1, 1, 2)),
    "mobilevit_xxs_64": dict(image_size=(64, 64), num_classes=12, **XXS, depths=(1, 1, 1)),
}
BENCH = {"mobilevit_xs": dict(image_size=(256, 256), num_classes=1000, **XS),
         "mobilevit_xxs": dict(image_size=(256, 256), num_classes=1000, **XXS),
         "mobilevit_s": dict(image_size=(256, 256), num_classes=1000, **S)}
WEIGHT_SEED, IMAGE_SEED, BATCH = 31, 32, 2

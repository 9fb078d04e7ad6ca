"""Test oracle of RegionViT (reference regionvit.py), kept beside the tests that use it.

  * make_config / weight_specs / init_weights / stress_weights: configs and seeded weights in the engine's names (SURVEY.md
    App. B: the reference's attribute paths), the reference's initial distributions;
  * forward: the float64 numpy restatement of RegionViT.call (regionvit.py:249-263);
  * forward_bf16_storage: forward() with what the bf16 engine stores rounded to bfloat16;
  * r2l_attention: the engine's regional-to-local attention on its own (vb_op_r2l_attention);
  * installed(): crossformer_oracle's stand-in plus tf.pad and an Embedding that raises on an index outside its table (as
    TensorFlow's CPU kernel does, where numpy would wrap a negative one), so that the reference's regionvit.py runs unmodified;
    load_weights sets the oracle's weights by attribute path.

The TensorFlow semantics restated here (third-party, public API documentation): Conv2D 'SAME' gives ceil(in / stride) positions and
pads max((out - 1) * stride + k - in, 0) in total, the smaller half on the top and left; a Conv2D with groups == filters == input
channels is depthwise, kernel [k, k, 1, C]; LayerNormalization's epsilon is 1e-3; Embedding initialises uniform(-0.05, 0.05).
"""
from __future__ import annotations

import collections
import contextlib
import math
import sys

import numpy as np

import crossformer_oracle
from oracle import spec_numpy, tf_shim
from vit_tensorflow_b200.models import REGIONVIT_CTOR_KEYS, regionvit_size_error

REGIONVIT_DEFAULTS = dict(dim=(64, 128, 256, 512), depth=(2, 2, 8, 2), window_size=7, num_classes=1000, tokenize_local_3_conv=False,
                          local_patch_size=4, use_peg=False, attn_dropout=0.0, ff_dropout=0.0)   # regionvit.py:185-195
LN_EPS = 1e-3                                             # Keras LayerNormalization
HEADS, DIM_HEAD = 4, 32                                   # R2LTransformer / Attention defaults (regionvit.py:119, :239)


def make_config(image_size=224, image_h=None, image_w=None, **kw) -> dict:
    """A RegionViT config: the reference's constructor kwargs (defaults filled in) plus the image size the tests call it with."""
    cfg = dict(REGIONVIT_DEFAULTS)
    cfg.update(kw)
    cfg["kind"] = "regionvit"
    cfg["image_h"], cfg["image_w"] = image_h or image_size, image_w or image_h or image_size
    return cfg


def ctor_kwargs(cfg) -> dict:
    return {k: cfg[k] for k in REGIONVIT_CTOR_KEYS if k in cfg}


def _cast4(v):
    return tuple(v) if isinstance(v, tuple) else (v,) * 4


def dims(cfg):
    return _cast4(cfg["dim"])


def depths(cfg):
    return _cast4(cfg["depth"])


def weight_specs(cfg):
    s = collections.OrderedDict()
    d0, ws, p = dims(cfg)[0], cfg["window_size"], cfg["local_patch_size"] * cfg["window_size"]

    def conv(n, k, cin, cout):
        s[n + ".kernel"], s[n + ".bias"] = ((k, k, cin, cout), "glorot"), ((cout,), "zeros")

    def ln(n, d):
        s[n + ".gamma"], s[n + ".beta"] = ((d,), "ones"), ((d,), "zeros")

    if cfg["tokenize_local_3_conv"]:
        conv("local_encoder.0", 3, 3, d0)
        ln("local_encoder.1", d0)
        conv("local_encoder.3", 3, d0, d0)
        ln("local_encoder.4", d0)
        conv("local_encoder.6", 3, d0, d0)
    else:
        conv("local_encoder", 8, 3, d0)
    conv("region_encoder.1", 1, 3 * p * p, d0)
    for st, (d, depth) in enumerate(zip(dims(cfg), depths(cfg))):
        pre = f"region_layers.{st}."
        if st:
            conv(pre + "0.conv", 3, dims(cfg)[st - 1], d)
            if cfg["use_peg"]:
                s[pre + "1.proj.kernel"], s[pre + "1.proj.bias"] = ((3, 3, 1, d), "glorot_dw"), ((d,), "zeros")
        s[pre + "2.local_rel_pos_bias.embeddings"] = (((2 * ws - 1) ** 2, HEADS), "embedding")
        for L in range(depth):
            b = f"{pre}2.layers.{L}."
            ln(b + "0.norm", d)
            s[b + "0.to_qkv.kernel"] = ((d, 3 * HEADS * DIM_HEAD), "glorot")
            s[b + "0.to_out.kernel"], s[b + "0.to_out.bias"] = ((HEADS * DIM_HEAD, d), "glorot"), ((d,), "zeros")
            ln(b + "1.net.0", d)
            s[b + "1.net.1.kernel"], s[b + "1.net.1.bias"] = ((d, 4 * d), "glorot"), ((4 * d,), "zeros")
            s[b + "1.net.4.kernel"], s[b + "1.net.4.bias"] = ((4 * d, d), "glorot"), ((d,), "zeros")
    last = dims(cfg)[-1]
    ln("to_logits.1", last)
    s["to_logits.2.kernel"], s["to_logits.2.bias"] = ((last, cfg["num_classes"]), "glorot"), ((cfg["num_classes"],), "zeros")
    return s


def init_weights(cfg, seed=0):
    rng = np.random.default_rng(seed)
    out = collections.OrderedDict()
    for name, (shape, init) in weight_specs(cfg).items():
        if init in ("glorot", "glorot_dw"):
            rf = int(np.prod(shape[:-2]))
            lim = math.sqrt(6.0 / (rf * (shape[-2] + shape[-1])))
            a = rng.uniform(-lim, lim, size=shape)
        elif init == "zeros":
            a = np.zeros(shape)
        elif init == "ones":
            a = np.ones(shape)
        elif init == "embedding":
            a = rng.uniform(-0.05, 0.05, size=shape)
        else:
            raise AssertionError(init)
        out[name] = np.ascontiguousarray(a, dtype=np.float32)
    return out


def stress_weights(cfg, seed=1):
    """init_weights with what the defaults hide: non-zero biases (0.2 N), LayerNorm gamma = 1 + 0.2 N with every fifth channel
    negated, beta = 0.2 N, and a window table of N(0, 1) (twenty times the initial spread, so that a wrong offset shows)."""
    rng = np.random.default_rng(seed)
    out = init_weights(cfg, seed)
    for name, (shape, init) in weight_specs(cfg).items():
        if init == "ones":
            a = 1.0 + 0.2 * rng.standard_normal(shape)
            a.reshape(-1)[::5] *= -1.0
        elif init == "zeros":
            a = 0.2 * rng.standard_normal(shape)
        elif init == "embedding":
            a = rng.standard_normal(shape)
        else:
            continue
        out[name] = a.astype(np.float32)
    return out


def make_image(cfg, batch, seed=0, h=None, w=None):
    rng = np.random.default_rng(seed)
    return rng.standard_normal((batch, h or cfg["image_h"], w or cfg["image_w"], 3), dtype=np.float32)


def size_error(cfg, h, w):
    """None when the reference runs an h x w image; otherwise what the engine says (its asserts' messages first)."""
    p, lp = cfg["local_patch_size"] * cfg["window_size"], cfg["local_patch_size"]
    if h % p or w % p:
        return "height and width must be divisible by region patch size"
    if h % lp or w % lp:
        return "height and width must be divisible by local patch size"
    return regionvit_size_error(h, w, lp, cfg["window_size"])


# ------------------------------------------------------------------------------------------------ float64 spec
def layer_norm(x, g, b, eps=LN_EPS):
    mu = x.mean(-1, keepdims=True)
    return (x - mu) / np.sqrt(x.var(-1, keepdims=True) + eps) * np.reshape(g, -1) + np.reshape(b, -1)


def _store(x):                                            # forward_bf16_storage rounds what the engine stores here
    return x


def _matmul(x, k):                                        # forward_bf16_storage rounds the operands and the result
    return x @ k


def conv_same(x, k, bias, stride):
    """Conv2D(k x k, stride, SAME) with bias: im2col over the zero-padded map, taps (row, column, channel)."""
    b, H, W, C = x.shape
    kk = k.shape[0]
    oh, ow = -(-H // stride), -(-W // stride)
    ph, pw = max((oh - 1) * stride + kk - H, 0), max((ow - 1) * stride + kk - W, 0)
    xp = np.pad(x, ((0, 0), (ph // 2, ph - ph // 2), (pw // 2, pw - pw // 2), (0, 0)))
    cols = np.concatenate([xp[:, ky:ky + (oh - 1) * stride + 1:stride, kx:kx + (ow - 1) * stride + 1:stride]
                           for ky in range(kk) for kx in range(kk)], -1)
    return _store(_matmul(cols, k.reshape(kk * kk * C, -1)) + bias)


def depthwise_same(x, k, bias):
    """The PEG's depthwise Conv2D(3, SAME, stride 1), kernel [3, 3, 1, C]."""
    b, H, W, C = x.shape
    xp = np.pad(x, ((0, 0), (1, 1), (1, 1), (0, 0)))
    return sum(xp[:, ky:ky + H, kx:kx + W] * k[ky, kx, 0] for ky in range(3) for kx in range(3)) + bias


def window_bias(table, ws, wh, ww):
    """rel_pos_bias of R2LTransformer.call (regionvit.py:143-155) for a wh x ww window: [heads, 1 + n, 1 + n], zero on row and
    column 0, table row (dr + ws - 1) + (dc + ws - 1) (2 ws - 1) for the local tokens (row-major in the window)."""
    r, c = np.meshgrid(np.arange(wh), np.arange(ww), indexing="ij")
    r, c = r.reshape(-1), c.reshape(-1)
    idx = (r[:, None] - r[None, :] + ws - 1) + (c[:, None] - c[None, :] + ws - 1) * (2 * ws - 1)
    if idx.min() < 0 or idx.max() >= table.shape[0]:
        raise IndexError(f"the {wh} x {ww} window reaches past the ({2 * ws - 1})^2 relative-position table")
    out = np.zeros((table.shape[1], wh * ww + 1, wh * ww + 1))
    out[:, 1:, 1:] = np.transpose(table[idx], (2, 0, 1))
    return out


def softmax_attention(qkv, heads, dh, bias=None):
    """softmax(q k^T dh^-0.5 + bias) v per head over the rows of qkv [n_seq, n, 3 heads dh] -> [n_seq, n, heads dh]."""
    inner = heads * dh
    q, k, v = (qkv[..., i * inner:(i + 1) * inner].reshape(qkv.shape[0], -1, heads, dh).transpose(0, 2, 1, 3) for i in range(3))
    sim = q @ np.swapaxes(k, -1, -2) * dh ** -0.5
    if bias is not None:
        sim = sim + bias
    a = np.exp(sim - sim.max(-1, keepdims=True))
    o = (a / a.sum(-1, keepdims=True)) @ v
    return o.transpose(0, 2, 1, 3).reshape(qkv.shape[0], -1, inner)


def to_windows(local, rh, rw):
    """'b (h p1) (w p2) d -> (b h w) (p1 p2) d' (regionvit.py:164)."""
    b, lh, lw, d = local.shape
    wh, ww = lh // rh, lw // rw
    return local.reshape(b, rh, wh, rw, ww, d).transpose(0, 1, 3, 2, 4, 5).reshape(b * rh * rw, wh * ww, d)


def from_windows(t, b, lh, lw, rh, rw):
    d = t.shape[-1]
    return t.reshape(b, rh, rw, lh // rh, lw // rw, d).transpose(0, 1, 3, 2, 4, 5).reshape(b, lh, lw, d)


def r2l_attention(qkv_local, qkv_region, heads, dh, table, ws):
    """The R2L attention alone: qkv_local [b, lh, lw, >= 3 heads dh], qkv_region [b, rh, rw, ...] -> (out_local [b, lh, lw, heads dh],
    out_region [b, rh, rw, heads dh]); table [(2 ws - 1)^2, heads] (the Embedding's layout)."""
    b, lh, lw, _ = qkv_local.shape
    _, rh, rw, _ = qkv_region.shape
    n3 = 3 * heads * dh
    t = np.concatenate([qkv_region[..., :n3].reshape(b * rh * rw, 1, n3), to_windows(qkv_local[..., :n3], rh, rw)], 1)
    o = softmax_attention(t, heads, dh, window_bias(table, ws, lh // rh, lw // rw))
    return from_windows(o[:, 1:], b, lh, lw, rh, rw), o[:, 0].reshape(b, rh, rw, -1)


def attention(x, w, a, bias=None):
    """Attention.call (regionvit.py:93-116) over sequences x [n_seq, n, d]."""
    qkv = _store(_matmul(layer_norm(x, w[a + "0.norm.gamma"], w[a + "0.norm.beta"]), w[a + "0.to_qkv.kernel"]))
    o = _store(softmax_attention(qkv, HEADS, DIM_HEAD, bias))
    return _matmul(o, w[a + "0.to_out.kernel"]) + w[a + "0.to_out.bias"]


def mlp(x, w, a):
    y = _matmul(layer_norm(x, w[a + "1.net.0.gamma"], w[a + "1.net.0.beta"]), w[a + "1.net.1.kernel"]) + w[a + "1.net.1.bias"]
    return _matmul(_store(spec_numpy.gelu(y)), w[a + "1.net.4.kernel"]) + w[a + "1.net.4.bias"]


def forward(img, weights, cfg, dtype=np.float64):
    """RegionViT.call(img) -> logits [b, num_classes] (no BatchNorm; ff_dropout 0)."""
    w = {k: np.asarray(v, dtype=dtype) for k, v in weights.items()}
    x = np.asarray(img, dtype=dtype)
    b, H, W, c = x.shape
    ws, p = cfg["window_size"], cfg["local_patch_size"] * cfg["window_size"]
    if cfg["tokenize_local_3_conv"]:                      # regionvit.py:211-218
        y = conv_same(x, w["local_encoder.0.kernel"], w["local_encoder.0.bias"], 2)
        y = _store(spec_numpy.gelu(layer_norm(y, w["local_encoder.1.gamma"], w["local_encoder.1.beta"])))
        y = conv_same(y, w["local_encoder.3.kernel"], w["local_encoder.3.bias"], 2)
        y = _store(spec_numpy.gelu(layer_norm(y, w["local_encoder.4.gamma"], w["local_encoder.4.beta"])))
        local = conv_same(y, w["local_encoder.6.kernel"], w["local_encoder.6.bias"], 1)
    else:
        local = conv_same(x, w["local_encoder.kernel"], w["local_encoder.bias"], 4)
    r = x.reshape(b, H // p, p, W // p, p, c).transpose(0, 1, 3, 5, 2, 4).reshape(b, H // p, W // p, c * p * p)   # (c p1 p2)
    region = _store(_matmul(r, w["region_encoder.1.kernel"].reshape(c * p * p, -1)) + w["region_encoder.1.bias"])
    for st, depth in enumerate(depths(cfg)):
        pre = f"region_layers.{st}."
        if st:                                            # regionvit.py:258: one Downsample for both maps
            local = conv_same(local, w[pre + "0.conv.kernel"], w[pre + "0.conv.bias"], 2)
            region = conv_same(region, w[pre + "0.conv.kernel"], w[pre + "0.conv.bias"], 2)
            if cfg["use_peg"]:
                local = _store(depthwise_same(local, w[pre + "1.proj.kernel"], w[pre + "1.proj.bias"]) + local)
        _, lh, lw, d = local.shape
        _, rh, rw, _ = region.shape
        bias = window_bias(w[pre + "2.local_rel_pos_bias.embeddings"], ws, lh // rh, lw // rw)
        R = region.reshape(b, rh * rw, d)
        Lw = to_windows(local, rh, rw)
        for L in range(depth):
            a = f"{pre}2.layers.{L}."
            R = _store(attention(R, w, a) + R)                                       # :159
            T = np.concatenate([R.reshape(b * rh * rw, 1, d), Lw], 1)
            T = _store(attention(T, w, a, bias) + T)                                 # :169
            T = _store(mlp(T, w, a) + T)                                             # :172
            R, Lw = T[:, 0].reshape(b, rh * rw, d), T[:, 1:]
        local, region = from_windows(Lw, b, lh, lw, rh, rw), R.reshape(b, rh, rw, d)
    z = layer_norm(region.mean(axis=(1, 2)), w["to_logits.1.gamma"], w["to_logits.1.beta"])   # :243-247
    return spec_numpy.dense(z, w, "to_logits.2")


def bf16_round(x):
    return crossformer_oracle.bf16_round(x)


def forward_bf16_storage(img, weights, cfg):
    """forward() with what the bf16 engine stores rounded to bfloat16 -- the operands and results of every convolution and Dense,
    q|k|v, the attention output, the GELU activations and the residual stream after every sub-block -- and everything else in
    float64: a lower estimate of what storing activations and weights in bf16 alone costs."""
    global _matmul, _store
    exact, store = _matmul, _store
    _matmul, _store = (lambda x, k: bf16_round(bf16_round(x) @ bf16_round(k))), bf16_round
    try:
        return forward(img, weights, cfg)
    finally:
        _matmul, _store = exact, store


# ------------------------------------------------------------------------------------------------ the reference's regionvit.py
class _StrictEmbedding(tf_shim.Embedding):
    """The stand-in's Embedding, raising on an index outside the table as TensorFlow's CPU lookup does (numpy would wrap a
    negative index and read another row)."""

    def call(self, inputs):
        idx = np.asarray(inputs)
        if idx.size and (idx.min() < 0 or idx.max() >= self.input_dim):
            raise IndexError(f"Embedding: indices in [{idx.min()}, {idx.max()}] are outside [0, {self.input_dim})")
        return super().call(inputs)


@contextlib.contextmanager
def installed(reference_dir):
    """crossformer_oracle.installed(reference_dir) (with its int32 convert_to_tensor, and levit_oracle's meshgrid / stack) plus
    tf.pad and the strict Embedding; `import regionvit` inside the block is the reference's own file, removed from sys.modules
    again on exit."""
    saved = sys.modules.pop("regionvit", None)
    with crossformer_oracle.installed(reference_dir) as tf:
        layers = sys.modules["tensorflow.keras.layers"]
        previous = layers.Embedding
        layers.Embedding = _StrictEmbedding
        tf.pad = tf_shim._returns_tensor(
            lambda tensor, paddings, mode="CONSTANT", constant_values=0, **_: np.pad(tf_shim._arr(tensor), np.asarray(paddings),
                                                                                      constant_values=constant_values))
        try:
            yield tf
        finally:
            layers.Embedding = previous
            del tf.pad
            sys.modules.pop("regionvit", None)
            if saved is not None:
                sys.modules["regionvit"] = saved


def load_weights(model, w):
    """The oracle's weights into a reference RegionViT by attribute path (regionvit.py:210-247)."""
    def conv(layer, n, bias=True):
        layer.set_weights([w[n + ".kernel"], w[n + ".bias"]] if bias else [w[n + ".kernel"]])

    def ln(layer, n):
        layer.set_weights([w[n + ".gamma"], w[n + ".beta"]])

    if hasattr(model.local_encoder, "layers"):
        seq = model.local_encoder.layers
        for i in (0, 3, 6):
            conv(seq[i], f"local_encoder.{i}")
        for i in (1, 4):
            ln(seq[i], f"local_encoder.{i}")
    else:
        conv(model.local_encoder, "local_encoder")
    conv(model.region_encoder.layers[1], "region_encoder.1")
    for st, (down, peg, tr) in enumerate(model.region_layers):
        pre = f"region_layers.{st}."
        if hasattr(down, "conv"):
            conv(down.conv, pre + "0.conv")
        if hasattr(peg, "proj"):
            conv(peg.proj, pre + "1.proj")
        tr.local_rel_pos_bias.embeddings.assign(w[pre + "2.local_rel_pos_bias.embeddings"])
        for L, (attn, ff) in enumerate(tr.layers):
            a = f"{pre}2.layers.{L}."
            ln(attn.norm, a + "0.norm")
            conv(attn.to_qkv, a + "0.to_qkv", False)
            conv(attn.to_out, a + "0.to_out")
            net = ff.net.layers
            ln(net[0], a + "1.net.0")
            conv(net[1], a + "1.net.1")
            conv(net[4], a + "1.net.4")
    ln(model.to_logits.layers[1], "to_logits.1")
    conv(model.to_logits.layers[2], "to_logits.2")


@contextlib.contextmanager
def reference_module(reference_dir, dtype=np.float64):
    """The reference's regionvit module over the stand-in in `dtype`."""
    import importlib
    tf_shim.set_dtype(dtype)
    try:
        with installed(reference_dir):
            yield importlib.import_module("regionvit")
    finally:
        tf_shim.set_dtype(np.float32)


def reference_model(mod, cfg, w, img, dtype=np.float64):
    model = mod.RegionViT(**ctor_kwargs(cfg))
    model(np.asarray(img, dtype))
    load_weights(model, {k: np.asarray(v, dtype) for k, v in w.items()})
    return model


def reference_logits(mod, cfg, w, img, dtype=np.float64):
    """Build the reference's RegionViT for `cfg`, call it once on `img` so that Keras builds every variable, load `w` and return
    `model(img)` (its default training=True: there is no BatchNorm and ff_dropout is 0)."""
    model = reference_model(mod, cfg, w, img, dtype)
    out = model(np.asarray(img, dtype))
    return np.asarray(out).view(np.ndarray).copy()


# ------------------------------------------------------------------------------------------------ cases
# small cases (fixtures with float32 and float64 reference logits) and the two configurations tools/regionvit_bench.py measures
SMALL = {
    # the README model's widths at 56 x 56 with one layer per stage: local maps 14 -> 7 -> 4 -> 2, windows 7, 7, 4, 2
    "regionvit_readme_small": dict(image_size=56, dim=(64, 128, 256, 512), depth=(1, 1, 1, 1), num_classes=10),
    # the 3-conv tokenizer with the PEG, widths 48 / 96 / 144 / 200 (none a multiple of 64), 56 x 56
    "regionvit_3conv_peg": dict(image_size=56, dim=(48, 96, 144, 200), depth=(1, 1, 2, 1), tokenize_local_3_conv=True, use_peg=True,
                                num_classes=7),
    # window_size 14 at 112 x 112: windows of 14 x 14 local tokens plus the regional one (197 tokens), then 14, 7, 4
    "regionvit_ws14": dict(image_size=112, dim=32, depth=(1, 1, 0, 1), window_size=14, num_classes=5),
    # a rectangular 28 x 56 image: local maps 7 x 14 -> 4 x 7 -> 2 x 4 -> 1 x 2 over region maps 1 x 2 -> 1 x 1: 4 x 7 windows
    "regionvit_rect": dict(image_size=28, image_h=28, image_w=56, dim=(32, 64, 64, 96), depth=1, num_classes=6),
    # int dim and depth: the same width at every stage, no doubling
    "regionvit_int": dict(image_size=56, dim=96, depth=1, num_classes=4),
}
BENCH = {
    "regionvit_readme": dict(image_size=224, dim=(64, 128, 256, 512), depth=(2, 2, 8, 2), num_classes=1000),
    "regionvit_s": dict(image_size=224, dim=(96, 192, 384, 768), depth=(2, 2, 14, 2), tokenize_local_3_conv=True, num_classes=1000),
}
WEIGHT_SEED, IMAGE_SEED, BATCH = 71, 72, 2

"""Test oracle of CrossFormer (reference crossformer.py), kept beside the tests that use it.

  * make_config / weight_specs / init_weights / stress_weights: configs and seeded weights in the engine's names (SURVEY.md
    App. B: the reference's attribute paths), the reference's initial distributions;
  * forward: the float64 numpy restatement of CrossFormer.call (crossformer.py:263-269);
  * forward_torch: an independent PyTorch restatement (F.conv2d with explicit asymmetric SAME padding per kernel size, windows by
    reshape / permute);
  * forward_bf16_storage: forward() with what the bf16 engine stores rounded to bfloat16;
  * window_table: the (2 w - 1)^2 table of one DynamicPositionBias that the reference's rel_pos_indices read;
  * installed(): cvt_oracle's stand-in plus what crossformer.py calls beyond it (a convert_to_tensor that keeps Python ints
    integer, as TensorFlow's does: the reference indexes with its result, crossformer.py:131,163), so that the reference's
    crossformer.py runs unmodified; load_weights sets the oracle's weights by attribute path.

The TensorFlow semantics restated here (third-party, public API documentation): 'SAME' gives ceil(in / stride) positions and pads
max((out - 1) * stride + k - in, 0) in total, the smaller half, on the top and left; LayerNormalization's epsilon is 1e-3.
"""
from __future__ import annotations

import collections
import contextlib
import math
import random
import sys

import numpy as np

import cvt_oracle
from oracle import spec_numpy, tf_shim
from vit_tensorflow_b200.models import CROSSFORMER_CTOR_KEYS, crossformer_size_error

CROSSFORMER_DEFAULTS = dict(dim=(64, 128, 256, 512), depth=(2, 2, 8, 2), global_window_size=(8, 4, 2, 1), local_window_size=7,
                            cross_embed_kernel_sizes=((4, 8, 16, 32), (2, 4), (2, 4), (2, 4)), cross_embed_strides=(4, 2, 2, 2),
                            num_classes=1000, attn_dropout=0.0, ff_dropout=0.0)   # crossformer.py:206-216
DIM_HEAD, MLP_MULT = 32, 4                                # crossformer.py:105,90
LN_EPS, DPB_LN_EPS = 1e-5, 1e-3                           # the module's LayerNorm (:74); Keras LayerNormalization (:57)


def _tuple4(v):
    return v if isinstance(v, tuple) else (v,) * 4        # cast_tuple, crossformer.py:11-12


def make_config(image_size=224, image_w=None, **kw) -> dict:
    """A CrossFormer config: the reference's constructor kwargs (defaults filled in) plus the image size the tests call it with."""
    cfg = dict(CROSSFORMER_DEFAULTS)
    cfg.update(kw)
    cfg["kind"] = "crossformer"
    cfg["image_h"], cfg["image_w"] = image_size, image_w or image_size
    return cfg


def ctor_kwargs(cfg) -> dict:
    return {k: cfg[k] for k in CROSSFORMER_CTOR_KEYS if k in cfg}


def stages(cfg):
    keys = ("dim", "depth", "global_window_size", "local_window_size", "cross_embed_kernel_sizes", "cross_embed_strides")
    vals = [_tuple4(cfg[k]) for k in keys]
    return [dict(dim=d, depth=n, global_wsz=g, local_wsz=lw, kernels=tuple(sorted(k)), stride=s) for d, n, g, lw, k, s in zip(*vals)]


def dim_scales(dim, n):                                   # crossformer.py:38-39
    s = [int(dim / (2 ** i)) for i in range(1, n)]
    return s + [dim - sum(s)]


def weight_specs(cfg):
    s = collections.OrderedDict()
    cin = 3
    for st, c in enumerate(stages(cfg)):
        p, d = f"crossformer_layers.{st}.", c["dim"]
        inner, d4 = DIM_HEAD * (d // DIM_HEAD), d // 4
        for i, (k, ds) in enumerate(zip(c["kernels"], dim_scales(d, len(c["kernels"])))):
            s[f"{p}0.convs.{i}.kernel"], s[f"{p}0.convs.{i}.bias"] = ((k, k, cin, ds), "glorot"), ((ds,), "zeros")
        for L in range(c["depth"]):
            b = f"{p}1.layers.{L}."
            for a in ("0.", "2."):
                s[b + a + "norm.g"], s[b + a + "norm.b"] = ((1, 1, 1, d), "ones"), ((1, 1, 1, d), "zeros")
                s[b + a + "to_qkv.kernel"] = ((1, 1, d, 3 * inner), "glorot")
                s[b + a + "to_out.kernel"], s[b + a + "to_out.bias"] = ((1, 1, inner, d), "glorot"), ((d,), "zeros")
                q = b + a + "dpb.dpb_layers."
                for li in (0, 3, 6, 9):
                    s[f"{q}{li}.kernel"] = ((2 if li == 0 else d4, 1 if li == 9 else d4), "glorot")
                    s[f"{q}{li}.bias"] = ((1 if li == 9 else d4,), "zeros")
                for li in (1, 4, 7):
                    s[f"{q}{li}.gamma"], s[f"{q}{li}.beta"] = ((d4,), "ones"), ((d4,), "zeros")
            for m in ("1.", "3."):
                s[b + m + "net.0.g"], s[b + m + "net.0.b"] = ((1, 1, 1, d), "ones"), ((1, 1, 1, d), "zeros")
                s[b + m + "net.1.kernel"], s[b + m + "net.1.bias"] = ((1, 1, d, MLP_MULT * d), "glorot"), ((MLP_MULT * d,), "zeros")
                s[b + m + "net.4.kernel"], s[b + m + "net.4.bias"] = ((1, 1, MLP_MULT * d, d), "glorot"), ((d,), "zeros")
        cin = d
    s["to_logits.1.kernel"], s["to_logits.1.bias"] = ((cin, cfg["num_classes"]), "glorot"), ((cfg["num_classes"],), "zeros")
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
        else:
            raise AssertionError(init)
        out[name] = np.ascontiguousarray(a, dtype=np.float32)
    return out


def stress_weights(cfg, seed=1):
    """init_weights with what the defaults hide: non-zero biases, LayerNorm g / gamma = 1 + 0.2 N and b / beta = 0.2 N."""
    rng = np.random.default_rng(seed)
    out = init_weights(cfg, seed)
    for name, (shape, init) in weight_specs(cfg).items():
        if init == "ones":
            a = 1.0 + 0.2 * rng.standard_normal(shape)
        elif init == "zeros":
            a = 0.2 * rng.standard_normal(shape)
        else:
            continue
        out[name] = a.astype(np.float32)
    return out


def make_image(cfg, batch, seed=0, h=None, w=None):
    rng = np.random.default_rng(seed)
    return rng.standard_normal((batch, h or cfg["image_h"], w or cfg["image_w"], 3), dtype=np.float32)


def size_error(cfg, h, w):
    return crossformer_size_error(stages(cfg), h, w)


# ------------------------------------------------------------------------------------------------ float64 spec
def layer_norm(x, g, b, eps):
    mu = x.mean(-1, keepdims=True)
    return (x - mu) / np.sqrt(x.var(-1, keepdims=True) + eps) * np.reshape(g, -1) + np.reshape(b, -1)


def _store(x):                                            # forward_bf16_storage rounds what the engine stores here
    return x


def _matmul(x, k):                                        # forward_bf16_storage rounds the operands and the result
    return x @ k


def conv_same(x, k, bias, stride):
    """Conv2D(SAME, strides=stride) with bias: x [b, H, W, C], k [k, k, C, O]."""
    b, H, W, C = x.shape
    kk = k.shape[0]
    oh, ow = -(-H // stride), -(-W // stride)
    ph, pw = max((oh - 1) * stride + kk - H, 0), max((ow - 1) * stride + kk - W, 0)
    xp = np.pad(x, ((0, 0), (ph // 2, ph - ph // 2), (pw // 2, pw - pw // 2), (0, 0)))
    cols = np.stack([xp[:, ky:ky + (oh - 1) * stride + 1:stride, kx:kx + (ow - 1) * stride + 1:stride] for ky in range(kk) for kx in range(kk)], 3)
    return _matmul(cols.reshape(b, oh, ow, kk * kk * C), k.reshape(kk * kk * C, -1)) + bias


def cross_embed(x, w, p, c):
    """CrossEmbedLayer.call (crossformer.py:45-48): the sorted kernel sizes' SAME convolutions, concatenated."""
    return _store(np.concatenate([conv_same(x, w[f"{p}convs.{i}.kernel"], w[f"{p}convs.{i}.bias"], c["stride"])
                                  for i in range(len(c["kernels"]))], -1))


def conv1x1(x, w, n, bias=True):
    k = w[n + ".kernel"]
    y = _matmul(x, k.reshape(k.shape[-2], k.shape[-1]))
    return _store(y + w[n + ".bias"] if bias else y)


def dpb_biases(w, n, wsz):
    """DynamicPositionBias on the offsets range(-wsz, wsz + 1)^2, (row, column) order (crossformer.py:158-162)."""
    pos = np.arange(-wsz, wsz + 1, dtype=np.float64)
    x = np.stack(np.meshgrid(pos, pos, indexing="ij"), -1).reshape(-1, 2)
    for li in (0, 3, 6):
        x = x @ w[f"{n}{li}.kernel"] + w[f"{n}{li}.bias"]
        mu = x.mean(-1, keepdims=True)
        x = np.maximum((x - mu) / np.sqrt(x.var(-1, keepdims=True) + DPB_LN_EPS) * w[f"{n}{li + 1}.gamma"] + w[f"{n}{li + 1}.beta"], 0.0)
    return (x @ w[f"{n}9.kernel"] + w[f"{n}9.bias"])[:, 0]


def rel_pos_indices(wsz):
    """crossformer.py:126-131, as written: offsets shifted by wsz - 1 with a row pitch of 2 wsz - 1."""
    pos = np.arange(wsz)
    grid = np.stack(np.meshgrid(pos, pos, indexing="ij")).reshape(2, -1).T
    rel = grid[:, None] - grid[None, :] + wsz - 1
    return (rel * np.array([2 * wsz - 1, 1])).sum(-1)


def window_table(w, n, wsz):
    """The first (2 wsz - 1)^2 DPB outputs: the entries rel_pos_indices reach (the engine's PosBias::wsz table)."""
    return dpb_biases(w, n, wsz)[:(2 * wsz - 1) ** 2]


def windows(t, wsz, long):
    """[b, H, W, c] -> [(b h w), wsz^2, c]: 'b (h s1) (w s2) d -> (b h w) s1 s2 d' (short) / 'b (l1 h) (l2 w) d -> (b h w) l1 l2 d'."""
    b, H, W, c = t.shape
    if long:
        return t.reshape(b, wsz, H // wsz, wsz, W // wsz, c).transpose(0, 2, 4, 1, 3, 5).reshape(-1, wsz * wsz, c)
    return t.reshape(b, H // wsz, wsz, W // wsz, wsz, c).transpose(0, 1, 3, 2, 4, 5).reshape(-1, wsz * wsz, c)


def unwindows(t, b, H, W, wsz, long):
    c = t.shape[-1]
    if long:
        return t.reshape(b, H // wsz, W // wsz, wsz, wsz, c).transpose(0, 3, 1, 4, 2, 5).reshape(b, H, W, c)
    return t.reshape(b, H // wsz, W // wsz, wsz, wsz, c).transpose(0, 1, 3, 2, 4, 5).reshape(b, H, W, c)


def window_attention(qkv, heads, bias, wsz, long, b, H, W):
    """softmax(q k^T * 32^-0.5 + bias) v within each window; qkv [b, H, W, 3 * heads * 32] -> [b, H, W, heads * 32]."""
    inner = heads * DIM_HEAD
    t = windows(qkv, wsz, long)
    q, k, v = (t[..., i * inner:(i + 1) * inner].reshape(t.shape[0], -1, heads, DIM_HEAD).transpose(0, 2, 1, 3) for i in range(3))
    sim = q * DIM_HEAD ** -0.5 @ np.swapaxes(k, -1, -2) + bias
    a = np.exp(sim - sim.max(-1, keepdims=True))
    o = (a / a.sum(-1, keepdims=True)) @ v
    return unwindows(o.transpose(0, 2, 1, 3).reshape(t.shape[0], -1, inner), b, H, W, wsz, long)


def attention(x, w, a, wsz, long):
    """Attention.call (crossformer.py:133-180)."""
    b, H, W, d = x.shape
    heads = d // DIM_HEAD
    qkv = conv1x1(layer_norm(x, w[a + "norm.g"], w[a + "norm.b"], LN_EPS), w, a + "to_qkv", False)
    bias = dpb_biases(w, a + "dpb.dpb_layers.", wsz)[rel_pos_indices(wsz)]
    return conv1x1(window_attention(qkv, heads, bias, wsz, long, b, H, W), w, a + "to_out")


def mlp(x, w, m):
    return conv1x1(spec_numpy.gelu(conv1x1(layer_norm(x, w[m + "net.0.g"], w[m + "net.0.b"], LN_EPS), w, m + "net.1")), w, m + "net.4")


def forward(img, weights, cfg, dtype=np.float64):
    """CrossFormer.call(img) -> logits [b, num_classes] (no BatchNorm; dropout 0)."""
    w = {k: np.asarray(v, dtype=dtype) for k, v in weights.items()}
    x = np.asarray(img, dtype=dtype)
    for st, c in enumerate(stages(cfg)):
        p = f"crossformer_layers.{st}."
        x = cross_embed(x, w, p + "0.", c)
        for L in range(c["depth"]):
            b = f"{p}1.layers.{L}."
            x = _store(attention(x, w, b + "0.", c["local_wsz"], False) + x)
            x = _store(mlp(x, w, b + "1.") + x)
            x = _store(attention(x, w, b + "2.", c["global_wsz"], True) + x)
            x = _store(mlp(x, w, b + "3.") + x)
    return spec_numpy.dense(x.mean(axis=(1, 2)), w, "to_logits.1")


def forward_torch(img, weights, cfg):
    """The same model restated in PyTorch (float64, NCHW)."""
    import torch
    import torch.nn.functional as F
    t = {k: torch.from_numpy(np.asarray(v, np.float64)) for k, v in weights.items()}
    x = torch.from_numpy(np.asarray(img, np.float64)).permute(0, 3, 1, 2)

    def ln(x, n):
        return F.layer_norm(x.permute(0, 2, 3, 1), (x.shape[1],), t[n + ".g"].reshape(-1), t[n + ".b"].reshape(-1), LN_EPS).permute(0, 3, 1, 2)

    def conv(x, n, bias=True, stride=1, pad=(0, 0, 0, 0)):
        return F.conv2d(F.pad(x, pad), t[n + ".kernel"].permute(3, 2, 0, 1), t[n + ".bias"] if bias else None, stride=stride)

    def same_pad(size, k, s):
        total = max((-(-size // s) - 1) * s + k - size, 0)
        return total // 2, total - total // 2

    def dpb(n, wsz):
        pos = torch.arange(-wsz, wsz + 1, dtype=torch.float64)
        z = torch.stack(torch.meshgrid(pos, pos, indexing="ij"), -1).reshape(-1, 2)
        for li in (0, 3, 6):
            z = F.linear(z, t[f"{n}{li}.kernel"].T, t[f"{n}{li}.bias"])
            z = F.relu(F.layer_norm(z, (z.shape[-1],), t[f"{n}{li + 1}.gamma"], t[f"{n}{li + 1}.beta"], DPB_LN_EPS))
        return F.linear(z, t[f"{n}9.kernel"].T, t[f"{n}9.bias"])[:, 0]

    def attn(x, a, wsz, long):
        b, d, H, W = x.shape
        heads, inner = d // DIM_HEAD, DIM_HEAD * (d // DIM_HEAD)
        qkv = conv(ln(x, a + "norm"), a + "to_qkv", False)                        # [b, 3 inner, H, W]
        h, w = H // wsz, W // wsz
        if long:                                                                  # channel, l1, h, l2, w
            z = qkv.reshape(b, 3 * inner, wsz, h, wsz, w).permute(0, 3, 5, 2, 4, 1)
        else:                                                                     # channel, h, s1, w, s2
            z = qkv.reshape(b, 3 * inner, h, wsz, w, wsz).permute(0, 2, 4, 3, 5, 1)
        z = z.reshape(b * h * w, wsz * wsz, 3, heads, DIM_HEAD).permute(2, 0, 3, 1, 4)
        r = torch.arange(wsz)
        ry, rx = torch.meshgrid(r, r, indexing="ij")
        dy = ry.reshape(-1)[:, None] - ry.reshape(-1)[None, :] + wsz - 1
        dx = rx.reshape(-1)[:, None] - rx.reshape(-1)[None, :] + wsz - 1
        bias = dpb(a + "dpb.dpb_layers.", wsz)[dy * (2 * wsz - 1) + dx]
        sim = z[0] @ z[1].transpose(-1, -2) * DIM_HEAD ** -0.5 + bias
        o = torch.softmax(sim, -1) @ z[2]                                         # [bhw, heads, n, 32]
        o = o.permute(0, 2, 1, 3).reshape(b, h, w, wsz, wsz, inner)
        o = o.permute(0, 5, 3, 1, 4, 2) if long else o.permute(0, 5, 1, 3, 2, 4)
        return conv(o.reshape(b, inner, H, W), a + "to_out")

    def ff(x, m):
        return conv(F.gelu(conv(ln(x, m + "net.0"), m + "net.1")), m + "net.4")

    for st, c in enumerate(stages(cfg)):
        p = f"crossformer_layers.{st}."
        outs = []
        for i, k in enumerate(c["kernels"]):
            (pt, pb), (pl, pr) = same_pad(x.shape[2], k, c["stride"]), same_pad(x.shape[3], k, c["stride"])
            outs.append(conv(x, f"{p}0.convs.{i}", stride=c["stride"], pad=(pl, pr, pt, pb)))
        x = torch.cat(outs, 1)
        for L in range(c["depth"]):
            b = f"{p}1.layers.{L}."
            x = attn(x, b + "0.", c["local_wsz"], False) + x
            x = ff(x, b + "1.") + x
            x = attn(x, b + "2.", c["global_wsz"], True) + x
            x = ff(x, b + "3.") + x
    return (x.mean(dim=(2, 3)) @ t["to_logits.1.kernel"] + t["to_logits.1.bias"]).numpy()


def bf16_round(x):
    return cvt_oracle.bf16_round(x)


def forward_bf16_storage(img, weights, cfg):
    """forward() with what the bf16 engine stores rounded to bfloat16 -- the operands and results of every convolution (the cross-
    scale embedding and the 1x1s), the residual stream after every sub-block -- and everything else in float64: a lower estimate
    of what storing activations and weights in bf16 alone costs."""
    global _matmul, _store
    exact, store = _matmul, _store
    _matmul, _store = (lambda x, k: bf16_round(bf16_round(x) @ bf16_round(k))), bf16_round
    try:
        return forward(img, weights, cfg)
    finally:
        _matmul, _store = exact, store


# ------------------------------------------------------------------------------------------------ the reference's crossformer.py
@contextlib.contextmanager
def installed(reference_dir):
    """cvt_oracle.installed(reference_dir) plus a convert_to_tensor that infers int32 from Python ints, as TensorFlow does (the
    stand-in's yields floats, and crossformer.py:163 indexes with the result); `import crossformer` inside the block is the
    reference's own file, removed from sys.modules again on exit."""
    saved = sys.modules.pop("crossformer", None)
    with cvt_oracle.installed(reference_dir) as tf:
        previous = tf.convert_to_tensor

        def convert_to_tensor(value, dtype=None, **_):
            a = np.asarray(value.view(np.ndarray) if isinstance(value, np.ndarray) else value)
            if dtype is None and a.dtype.kind in "iub":
                return a.astype(np.int32)
            return a.astype(dtype or tf_shim.get_dtype())
        tf.convert_to_tensor = tf_shim._returns_tensor(convert_to_tensor)
        try:
            yield tf
        finally:
            tf.convert_to_tensor = previous
            sys.modules.pop("crossformer", None)
            if saved is not None:
                sys.modules["crossformer"] = saved


def load_weights(model, w):
    """The oracle's weights into a reference CrossFormer by attribute path (crossformer.py:244-261)."""
    def conv(layer, n, bias=True):
        layer.set_weights([w[n + ".kernel"], w[n + ".bias"]] if bias else [w[n + ".kernel"]])

    def ln(norm, n):
        norm.g.assign(w[n + ".g"])
        norm.b.assign(w[n + ".b"])

    for st, (cel, tr) in enumerate(model.crossformer_layers):
        p = f"crossformer_layers.{st}."
        for i, c in enumerate(cel.convs):
            conv(c, f"{p}0.convs.{i}")
        for L, layer in enumerate(tr.layers):
            b = f"{p}1.layers.{L}."
            for j, mod in enumerate(layer):
                n = f"{b}{j}."
                if j in (0, 2):
                    ln(mod.norm, n + "norm")
                    conv(mod.to_qkv, n + "to_qkv", False)
                    conv(mod.to_out, n + "to_out")
                    dl = mod.dpb.dpb_layers.layers
                    for li in (0, 3, 6, 9):
                        conv(dl[li], f"{n}dpb.dpb_layers.{li}")
                    for li in (1, 4, 7):
                        dl[li].set_weights([w[f"{n}dpb.dpb_layers.{li}.gamma"], w[f"{n}dpb.dpb_layers.{li}.beta"]])
                else:
                    net = mod.net.layers
                    ln(net[0], n + "net.0")
                    conv(net[1], n + "net.1")
                    conv(net[4], n + "net.4")
    model.to_logits.layers[1].set_weights([w["to_logits.1.kernel"], w["to_logits.1.bias"]])


@contextlib.contextmanager
def reference_module(reference_dir, dtype=np.float64):
    """The reference's crossformer module over the stand-in in `dtype`."""
    import importlib
    tf_shim.set_dtype(dtype)
    try:
        with installed(reference_dir):
            yield importlib.import_module("crossformer")
    finally:
        tf_shim.set_dtype(np.float32)


def reference_model(mod, cfg, w, img, dtype=np.float64):
    model = mod.CrossFormer(**ctor_kwargs(cfg))
    model(np.asarray(img, dtype))
    load_weights(model, {k: np.asarray(v, dtype) for k, v in w.items()})
    return model


def reference_logits(mod, cfg, w, img, dtype=np.float64):
    """Build the reference's CrossFormer for `cfg`, call it once on `img` so that Keras builds every variable, load `w` and return
    `model(img)` (its default training=True: there is no BatchNorm and the dropout rate is 0)."""
    model = reference_model(mod, cfg, w, img, dtype)
    out = model(np.asarray(img, dtype))
    return np.asarray(out).view(np.ndarray).copy()


def random_config(seed):
    """A small random configuration: 1 to 4 kernel sizes of one parity at or above the stride, strides 1 to 4, windows of 1 to 9
    tokens a side, dims off 64 (3 heads at 96) and non-square images whose stage maps meet the shape rule."""
    r = random.Random(seed)
    while True:
        kw = dict(num_classes=r.randint(2, 9))
        stride = (r.choice([2, 3, 4]),) + tuple(r.choice([1, 2, 2, 3]) for _ in range(3))
        kernels = []
        for i, s in enumerate(stride):
            par = r.randint(0, 1)
            kernels.append(tuple(r.sample([k for k in range(s, s + 9) if k % 2 == par], r.randint(1, 4 if i == 0 else 2))))
        kw.update(dim=tuple(r.choice([32, 48, 64, 96]) for _ in range(4)), depth=tuple(r.randint(0, 1) for _ in range(4)),
                  global_window_size=tuple(r.choice([1, 1, 2, 3]) for _ in range(4)),
                  local_window_size=tuple(r.choice([1, 2, 3]) for _ in range(4)), cross_embed_kernel_sizes=tuple(kernels),
                  cross_embed_strides=stride)
        for _ in range(2000):
            h, w = r.randint(8, 72), r.randint(8, 72)
            cfg = make_config(image_size=h, image_w=w, **kw)
            if size_error(cfg, h, w) is None:
                return cfg


# ------------------------------------------------------------------------------------------------ cases
# small cases (fixtures with float32 and float64 reference logits) and the two configurations tools/crossformer_bench.py measures
SMALL = {
    # a four-kernel stage 1 at stride 4, maps 32 -> 16 -> 8 -> 4: short windows of 16, 4, 4 and 1 token(s), long of 4, 16, 1 and 4
    "crossformer_small": dict(image_size=128, dim=(64, 64, 128, 64), depth=(1, 1, 1, 1), global_window_size=(2, 4, 1, 2),
                              local_window_size=(4, 2, 2, 1), num_classes=10),
    # odd kernels (3, 5, 7) at stride 3 on a 62 x 80 image (asymmetric SAME padding: 2 before, 3 after), maps 21 x 27 -> 21 x 27 ->
    # 7 x 9 -> 7 x 9; width 96 (3 heads, padded to 128); windows of 9 and 1 token(s), short and long
    "crossformer_odd": dict(image_size=62, image_w=80, dim=(96, 64, 64, 32), depth=(1, 1, 1, 1), global_window_size=(3, 3, 1, 1),
                            local_window_size=(3, 3, 1, 1), cross_embed_kernel_sizes=((3, 5, 7), (1, 3), (3, 5), (1,)),
                            cross_embed_strides=(3, 1, 3, 1), num_classes=7),
    # maps 40 x 80 -> 20 x 40 -> 20 x 40 -> 10 x 20: windows of 25, 64, 16, 25, 4, 100 (two query tiles and key blocks), 25, 4 tokens
    "crossformer_wide": dict(image_size=80, image_w=160, dim=(32, 64, 64, 32), depth=(1, 1, 1, 1), global_window_size=(8, 5, 10, 2),
                             local_window_size=(5, 4, 2, 5), cross_embed_kernel_sizes=((2, 4), (2, 4), (1, 3), (2,)),
                             cross_embed_strides=(2, 2, 1, 2), num_classes=5),
    # maps 63 -> 21 -> 7 -> 7: windows of 49 and 81, 49 and 9, 49 and 1, 1 and 49 tokens
    "crossformer_p9": dict(image_size=189, dim=(32, 32, 64, 32), depth=(1, 1, 1, 1), global_window_size=(9, 3, 1, 7),
                           local_window_size=(7, 7, 7, 1), cross_embed_kernel_sizes=((3, 5), (3,), (3, 5), (1,)),
                           cross_embed_strides=(3, 3, 3, 1), num_classes=6),
}
BENCH = {
    "crossformer_readme": dict(image_size=224, num_classes=1000),               # the reference README's model = the defaults
    "crossformer_96": dict(image_size=224, num_classes=1000, dim=(96, 192, 384, 768), depth=(2, 2, 6, 2)),
}
WEIGHT_SEED, IMAGE_SEED, BATCH = 51, 52, 2

"""Test oracle of ScalableViT (reference scalable_vit.py), kept beside the tests that use it.

  * make_config / stages / weight_specs / init_weights / stress_weights: configs and seeded weights in the engine's names
    (SURVEY.md App. B: the reference's attribute paths), the reference's initial distributions;
  * forward: the float64 numpy restatement of ScalableViT.call (scalable_vit.py:308-319) in the order the blocks execute;
  * forward_torch: an independent PyTorch restatement (F.conv2d with the SAME padding spelled out, the VALID r x r convolution,
    the grouped PEG, F.layer_norm, F.gelu, F.unfold-free window reshapes);
  * installed(): cvt_oracle's stand-in, which already covers what scalable_vit.py calls (Conv2D with groups and VALID strides,
    tf.math.reduce_variance, tf.sqrt, tf.ones; the shim supplies einops.layers.tensorflow.Reduce), so the reference's
    scalable_vit.py runs unmodified; load_weights sets the oracle's weights by attribute path.

The block order: Transformer builds each block as [SSA, MLP, PEG or None, MLP, IWSA] (scalable_vit.py:222-231) and unpacks it as
`ssa, ff1, peg, iwsa, ff2` (:236), so the variable named iwsa is the second MLP and ff2 is the IWSA: every block runs SSA, MLP,
PEG (first block only), MLP, IWSA.  Weight names follow construction order (element 3 is the second MLP, element 4 the IWSA).

The TensorFlow semantics restated here (third-party, public API documentation): 'VALID' gives floor((in - k) / stride) + 1
positions and refuses a window larger than the input; 'SAME' gives ceil(in / stride) positions and pads max((out - 1) * stride +
k - in, 0) in total, the smaller half first; LayerNormalization uses the biased variance, epsilon 1e-3 by default.
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
from vit_tensorflow_b200.models import SCALABLE_VIT_CTOR_KEYS, SCALABLE_VIT_STAGE_KEYS

SVIT_DEFAULTS = dict(window_size=None, iwsa_dim_key=32, iwsa_dim_value=32, ssa_dim_key=32, ssa_dim_value=32, ff_expansion_factor=4,
                     channels=3, dropout=0.0)                                 # scalable_vit.py:251-264
LN_EPS, HEAD_LN_EPS = 1e-5, 1e-3                                              # :47, Keras LayerNormalization (:304)


def make_config(image_size=(64, 64), **kw) -> dict:
    """A ScalableViT config: the reference's constructor kwargs (defaults filled in) plus the image size the tests call it with."""
    cfg = dict(SVIT_DEFAULTS)
    cfg.update(kw)
    cfg["kind"] = "scalable_vit"
    cfg["image_size"] = tuple(image_size)
    return cfg


def ctor_kwargs(cfg) -> dict:
    return {k: cfg[k] for k in SCALABLE_VIT_CTOR_KEYS if k in cfg}


def stages(cfg):
    """Per-stage hyperparameters as scalable_vit.py:270-289 derives them (cast_tuple to len(depth)), plus dim and depth."""
    n = len(cfg["depth"])
    cast = {k: (cfg[k] if isinstance(cfg[k], tuple) else (cfg[k],) * n) for k in SCALABLE_VIT_STAGE_KEYS}
    return [dict(dim=cfg["dim"] * 2 ** i, depth=cfg["depth"][i], **{k: cast[k][i] for k in SCALABLE_VIT_STAGE_KEYS}) for i in range(n)]


def block_prefix(s, L):
    return f"scalable_layers.{s}.0.layers.{L}."


def weight_specs(cfg):
    sp = collections.OrderedDict()
    f = cfg["ff_expansion_factor"]

    def conv(n, k, cin, cout, bias=True):
        sp[n + ".kernel"] = ((k, k, cin, cout), "glorot")
        if bias:
            sp[n + ".bias"] = ((cout,), "zeros")

    def ln(n, d):
        sp[n + ".g"], sp[n + ".b"] = ((1, 1, 1, d), "g"), ((1, 1, 1, d), "b")

    conv("to_patches", 7, cfg["channels"], cfg["dim"])
    sts = stages(cfg)
    for s, st in enumerate(sts):
        d, h, r = st["dim"], st["heads"], st["reduction_factor"]
        for L in range(st["depth"]):
            b = block_prefix(s, L)
            ln(b + "0.norm", d)
            conv(b + "0.fn.to_q", 1, d, h * st["ssa_dim_key"], False)
            conv(b + "0.fn.to_k", r, d, h * st["ssa_dim_key"], False)
            conv(b + "0.fn.to_v", r, d, h * st["ssa_dim_value"], False)
            conv(b + "0.fn.to_out.0", 1, h * st["ssa_dim_value"], d)
            for j in (1, 3):
                ln(f"{b}{j}.norm", d)
                conv(f"{b}{j}.fn.net.0", 1, d, f * d)
                conv(f"{b}{j}.fn.net.3", 1, f * d, d)
                if j == 1 and L == 0:
                    conv(b + "2.proj", 3, 1, d)
            hv = h * st["iwsa_dim_value"]
            ln(b + "4.norm", d)
            conv(b + "4.fn.local_interactive_module", 3, hv, hv)
            conv(b + "4.fn.to_q", 1, d, h * st["iwsa_dim_key"], False)
            conv(b + "4.fn.to_k", 1, d, h * st["iwsa_dim_key"], False)
            conv(b + "4.fn.to_v", 1, d, hv, False)
            conv(b + "4.fn.to_out.0", 1, hv, d)
        ln(f"scalable_layers.{s}.0.norm", st["dim"])
        if s < len(sts) - 1:
            conv(f"scalable_layers.{s}.1.conv", 3, st["dim"], 2 * st["dim"])
    dl = sts[-1]["dim"]
    sp["mlp_head.1.gamma"], sp["mlp_head.1.beta"] = ((dl,), "gamma"), ((dl,), "beta")
    sp["mlp_head.2.kernel"], sp["mlp_head.2.bias"] = ((dl, cfg["num_classes"]), "glorot"), ((cfg["num_classes"],), "zeros")
    return sp


def init_weights(cfg, seed=0):
    """Keras' initialisers: glorot-uniform over the receptive field (a depthwise kernel [3, 3, 1, d] has fan_in 9, fan_out 9 d), zero
    biases; the model's LayerNorm g 1 / b 0 (:50-51) and LayerNormalization gamma 1 / beta 0."""
    rng = np.random.default_rng(seed)
    out = collections.OrderedDict()
    for name, (shape, init) in weight_specs(cfg).items():
        if init == "glorot":
            rf = int(np.prod(shape[:-2]))
            lim = math.sqrt(6.0 / (rf * (shape[-2] + shape[-1])))
            a = rng.uniform(-lim, lim, size=shape)
        elif init in ("zeros", "b", "beta"):
            a = np.zeros(shape)
        elif init in ("g", "gamma"):
            a = np.ones(shape)
        else:
            raise AssertionError(init)
        out[name] = np.ascontiguousarray(a, dtype=np.float32)
    return out


def stress_weights(cfg, seed=1):
    """init_weights with what the Keras defaults hide: non-zero biases and betas (N(0, 0.3)), gammas around 1 (1 + N(0, 0.25))."""
    rng = np.random.default_rng(seed)
    out = init_weights(cfg, seed)
    for name, (shape, init) in weight_specs(cfg).items():
        if init in ("g", "gamma"):
            a = 1.0 + 0.25 * rng.standard_normal(shape)
        elif init in ("zeros", "b", "beta"):
            a = 0.3 * rng.standard_normal(shape)
        else:
            continue
        out[name] = a.astype(np.float32)
    return out


def make_image(cfg, batch, seed=0, h=None, w=None):
    rng = np.random.default_rng(seed)
    ih, iw = cfg["image_size"]
    return rng.standard_normal((batch, h or ih, w or iw, cfg["channels"]), dtype=np.float32)


# ------------------------------------------------------------------------------------------------ float64 spec
def gelu(x):
    from scipy.special import erf
    return 0.5 * x * (1.0 + erf(x / math.sqrt(2.0)))


def _conv_same(x, w, n, stride=1):
    kern = w[n + ".kernel"]
    y = spec_numpy.extract_patches_same(x, kern.shape[0], stride) @ kern.reshape(-1, kern.shape[-1])
    return y + w[n + ".bias"] if n + ".bias" in w else y


def _conv_valid(x, kern, r):
    """Conv2D(kernel r, strides r, VALID), no bias: floor(h / r) x floor(w / r) positions."""
    b, h, wd, c = x.shape
    kh, kw = h // r, wd // r
    if kh == 0 or kw == 0:
        raise ValueError("VALID convolution larger than its input")
    p = x[:, :kh * r, :kw * r].reshape(b, kh, r, kw, r, c).transpose(0, 1, 3, 2, 4, 5).reshape(b, kh, kw, r * r * c)
    return p @ kern.reshape(-1, kern.shape[-1])


def _ln(x, w, n):
    mu = x.mean(-1, keepdims=True)
    var = ((x - mu) ** 2).mean(-1, keepdims=True)
    return (x - mu) / np.sqrt(var + LN_EPS) * w[n + ".g"].reshape(-1) + w[n + ".b"].reshape(-1)


def _softmax(s):
    e = np.exp(s - s.max(-1, keepdims=True))
    return e / e.sum(-1, keepdims=True)


def _heads(t, h):                                # 'b ... (h d) -> b h (...) d'
    b = t.shape[0]
    return t.reshape(b, -1, h, t.shape[-1] // h).transpose(0, 2, 1, 3)


def ssa(x, w, n, st):
    b, H, W, _ = x.shape
    h, r = st["heads"], st["reduction_factor"]
    q = _heads(x @ w[n + "to_q.kernel"].reshape(x.shape[-1], -1), h)
    k = _heads(_conv_valid(x, w[n + "to_k.kernel"], r), h)
    v = _heads(_conv_valid(x, w[n + "to_v.kernel"], r), h)
    o = _softmax(q @ k.transpose(0, 1, 3, 2) * st["ssa_dim_key"] ** -0.5) @ v
    o = o.transpose(0, 2, 1, 3).reshape(b, H, W, -1)
    return o @ w[n + "to_out.0.kernel"].reshape(o.shape[-1], -1) + w[n + "to_out.0.bias"]


def iwsa(x, w, n, st):
    b, H, W, d = x.shape
    h = st["heads"]
    wh, ww = st["window_size"] or H, st["window_size"] or W
    assert H % wh == 0 and W % ww == 0
    q, k, v = (x @ w[n + f"to_{t}.kernel"].reshape(d, -1) for t in "qkv")
    local = _conv_same(v, w, n + "local_interactive_module")

    def win(t):                                  # 'b (x w1) (y w2) (h d) -> (b x y) h (w1 w2) d'
        c = t.shape[-1]
        return (t.reshape(b, H // wh, wh, W // ww, ww, h, c // h).transpose(0, 1, 3, 5, 2, 4, 6)
                .reshape(-1, h, wh * ww, c // h))
    o = _softmax(win(q) @ win(k).transpose(0, 1, 3, 2) * st["iwsa_dim_key"] ** -0.5) @ win(v)
    dv = o.shape[-1]
    o = o.reshape(b, H // wh, W // ww, h, wh, ww, dv).transpose(0, 1, 4, 2, 5, 3, 6).reshape(b, H, W, h * dv)
    o = o + local
    return o @ w[n + "to_out.0.kernel"].reshape(h * dv, d) + w[n + "to_out.0.bias"]


def mlp(x, w, n):
    d = x.shape[-1]
    hdn = gelu(x @ w[n + "net.0.kernel"].reshape(d, -1) + w[n + "net.0.bias"])
    return hdn @ w[n + "net.3.kernel"].reshape(hdn.shape[-1], d) + w[n + "net.3.bias"]


def peg(x, w, n):
    kern = w[n + ".kernel"]
    p = spec_numpy.extract_patches_same(x, 3, 1)
    b, oh, ow, _ = p.shape
    return (p.reshape(b, oh, ow, 9, -1) * kern.reshape(9, -1)).sum(-2) + w[n + ".bias"] + x


def forward(img, weights, cfg, dtype=np.float64):
    """ScalableViT.call(img) with dropout 0: logits [b, num_classes], the blocks in the order they execute."""
    w = {k: np.asarray(v, dtype=dtype) for k, v in weights.items()}
    x = _conv_same(np.asarray(img, dtype=dtype), w, "to_patches", 4)
    sts = stages(cfg)
    for s, st in enumerate(sts):
        for L in range(st["depth"]):
            b = block_prefix(s, L)
            x = ssa(_ln(x, w, b + "0.norm"), w, b + "0.fn.", st) + x       # element 0 (`ssa`)
            x = mlp(_ln(x, w, b + "1.norm"), w, b + "1.fn.") + x           # element 1 (`ff1`)
            if L == 0:
                x = peg(x, w, b + "2.proj")                                # element 2 (`peg`)
            x = mlp(_ln(x, w, b + "3.norm"), w, b + "3.fn.") + x           # element 3 (unpacked as `iwsa`)
            x = iwsa(_ln(x, w, b + "4.norm"), w, b + "4.fn.", st) + x      # element 4 (unpacked as `ff2`)
        x = _ln(x, w, f"scalable_layers.{s}.0.norm")
        if s < len(sts) - 1:
            x = _conv_same(x, w, f"scalable_layers.{s}.1.conv", 2)
    z = x.mean(axis=(1, 2))
    mu = z.mean(-1, keepdims=True)
    z = (z - mu) / np.sqrt(((z - mu) ** 2).mean(-1, keepdims=True) + HEAD_LN_EPS) * w["mlp_head.1.gamma"] + w["mlp_head.1.beta"]
    return z @ w["mlp_head.2.kernel"] + w["mlp_head.2.bias"]


def forward_torch(img, weights, cfg, device="cpu"):
    """The same model restated in PyTorch (float64): NCHW F.conv2d with explicit SAME padding, the VALID convolution as F.conv2d
    with stride r, the PEG as a grouped F.conv2d, F.layer_norm over channels, F.gelu, softmax attention on explicit reshapes."""
    import torch
    import torch.nn.functional as F
    t = {k: torch.from_numpy(np.asarray(v, np.float64)).to(device) for k, v in weights.items()}
    x = torch.from_numpy(np.asarray(img, np.float64)).to(device).permute(0, 3, 1, 2)

    def conv(x, n, stride=1, pad=True, groups=1):
        kern = t[n + ".kernel"]
        k = kern.shape[0]
        if pad:
            H, W = x.shape[-2:]
            ph, pw = max((-(-H // stride) - 1) * stride + k - H, 0), max((-(-W // stride) - 1) * stride + k - W, 0)
            x = F.pad(x, (pw // 2, pw - pw // 2, ph // 2, ph - ph // 2))
        return F.conv2d(x, kern.permute(3, 2, 0, 1), t.get(n + ".bias"), stride=stride, groups=groups)

    def ln(x, n):
        d = x.shape[1]
        return F.layer_norm(x.permute(0, 2, 3, 1), (d,), t[n + ".g"].reshape(d), t[n + ".b"].reshape(d), LN_EPS).permute(0, 3, 1, 2)

    def attend(q, k, v, scale):                  # [n, h, tokens, d]
        return torch.softmax(q @ k.transpose(-1, -2) * scale, dim=-1) @ v

    x = conv(x, "to_patches", 4)
    sts = stages(cfg)
    for s, st in enumerate(sts):
        h = st["heads"]
        for L in range(st["depth"]):
            b = block_prefix(s, L)
            B, d, H, W = x.shape
            a = ln(x, b + "0.norm")
            q = conv(a, b + "0.fn.to_q", pad=False)
            k = conv(a, b + "0.fn.to_k", st["reduction_factor"], pad=False)
            v = conv(a, b + "0.fn.to_v", st["reduction_factor"], pad=False)
            sp = [z.reshape(B, h, -1, z.shape[-2] * z.shape[-1]).transpose(-1, -2) for z in (q, k, v)]
            o = attend(*sp, st["ssa_dim_key"] ** -0.5).transpose(-1, -2).reshape(B, -1, H, W)
            x = conv(o, b + "0.fn.to_out.0", pad=False) + x
            for j in (1, 3):
                if j == 3 and L == 0:
                    x = conv(x, b + "2.proj", groups=d) + x
                a = ln(x, f"{b}{j}.norm")
                x = conv(F.gelu(conv(a, f"{b}{j}.fn.net.0", pad=False)), f"{b}{j}.fn.net.3", pad=False) + x
            a = ln(x, b + "4.norm")
            wh, ww = st["window_size"] or H, st["window_size"] or W
            q, k, v = (conv(a, b + f"4.fn.to_{c}", pad=False) for c in "qkv")
            local = conv(v, b + "4.fn.local_interactive_module")

            def win(z):
                c = z.shape[1] // h
                return z.reshape(B, h, c, H // wh, wh, W // ww, ww).permute(0, 3, 5, 1, 4, 6, 2).reshape(-1, h, wh * ww, c)
            o = attend(win(q), win(k), win(v), st["iwsa_dim_key"] ** -0.5)
            c = o.shape[-1]
            o = o.reshape(B, H // wh, W // ww, h, wh, ww, c).permute(0, 3, 6, 1, 4, 2, 5).reshape(B, h * c, H, W)
            x = conv(o + local, b + "4.fn.to_out.0", pad=False) + x
        x = ln(x, f"scalable_layers.{s}.0.norm")
        if s < len(sts) - 1:
            x = conv(x, f"scalable_layers.{s}.1.conv", 2)
    z = x.mean(dim=(2, 3))
    z = F.layer_norm(z, (z.shape[-1],), t["mlp_head.1.gamma"], t["mlp_head.1.beta"], HEAD_LN_EPS)
    return (z @ t["mlp_head.2.kernel"] + t["mlp_head.2.bias"]).cpu().numpy()


# ------------------------------------------------------------------------------------------------ the reference's scalable_vit.py
@contextlib.contextmanager
def installed(reference_dir):
    """cvt_oracle.installed(reference_dir); `import scalable_vit` inside the block is the reference's own file, removed from
    sys.modules again on exit."""
    saved = sys.modules.pop("scalable_vit", None)
    with cvt_oracle.installed(reference_dir) as tf:
        try:
            yield tf
        finally:
            sys.modules.pop("scalable_vit", None)
            if saved is not None:
                sys.modules["scalable_vit"] = saved


def load_weights(model, w, cfg):
    """The oracle's weights into a reference ScalableViT by attribute path (scalable_vit.py:261-306)."""
    def ln(norm, n):
        norm.g.assign(w[n + ".g"])
        norm.b.assign(w[n + ".b"])

    def conv(layer, n):
        layer.set_weights([w[n + ".kernel"], w[n + ".bias"]] if n + ".bias" in w else [w[n + ".kernel"]])

    conv(model.to_patches, "to_patches")
    for s, (tr, down) in enumerate(model.scalable_layers):
        for L, (a, f1, pg, f3, iw) in enumerate(tr.layers):              # construction order
            b = block_prefix(s, L)
            ln(a.norm, b + "0.norm")
            for n in ("to_q", "to_k", "to_v"):
                conv(getattr(a.fn, n), f"{b}0.fn.{n}")
            conv(a.fn.to_out.layers[0], b + "0.fn.to_out.0")
            for j, f in ((1, f1), (3, f3)):
                ln(f.norm, f"{b}{j}.norm")
                conv(f.fn.net.layers[0], f"{b}{j}.fn.net.0")
                conv(f.fn.net.layers[3], f"{b}{j}.fn.net.3")
            if pg is not None:
                conv(pg.proj, b + "2.proj")
            ln(iw.norm, b + "4.norm")
            for n in ("local_interactive_module", "to_q", "to_k", "to_v"):
                conv(getattr(iw.fn, n), f"{b}4.fn.{n}")
            conv(iw.fn.to_out.layers[0], b + "4.fn.to_out.0")
        ln(tr.norm, f"scalable_layers.{s}.0.norm")
        if down is not None:
            conv(down.conv, f"scalable_layers.{s}.1.conv")
    model.mlp_head.layers[1].set_weights([w["mlp_head.1.gamma"], w["mlp_head.1.beta"]])
    model.mlp_head.layers[2].set_weights([w["mlp_head.2.kernel"], w["mlp_head.2.bias"]])


@contextlib.contextmanager
def reference_module(reference_dir, dtype=np.float64):
    """The reference's scalable_vit module over the stand-in in `dtype`."""
    import importlib
    tf_shim.set_dtype(dtype)
    try:
        with installed(reference_dir):
            yield importlib.import_module("scalable_vit")
    finally:
        tf_shim.set_dtype(np.float32)


def reference_logits(mod, cfg, w, img, dtype=np.float64):
    """Build the reference's ScalableViT for `cfg`, call it once on `img` so that Keras builds every variable, load `w` and return
    `model(img, training=False)`."""
    model = mod.ScalableViT(**ctor_kwargs(cfg))
    model(np.asarray(img, dtype), training=False)
    load_weights(model, {k: np.asarray(v, dtype) for k, v in w.items()}, cfg)
    return np.asarray(model(np.asarray(img, dtype), training=False)).view(np.ndarray).copy()


# ------------------------------------------------------------------------------------------------ cases
README = dict(num_classes=1000, dim=64, heads=(2, 4, 8, 16), depth=(2, 2, 20, 2), ssa_dim_key=(40, 40, 40, 32),
              reduction_factor=(8, 4, 2, 1), window_size=(64, 32, None, None))                      # the reference's usage block
# small cases (fixtures with float64 reference logits).  Between them: real and None windows; windows of more than 64 tokens (100,
# 120, 165: several query tiles and key blocks); a rectangular image with odd maps (SAME ceil in the stem and Downsample, VALID
# floor in the SSA); r = 1; dk != dv widened to 32 / 64; head widths 32, 64 and 72 (over 64: the materialised path); 1, 2 and 4
# stages; channel widths off a multiple of 64; a second block (no PEG).
SMALL = {
    "scalable_vit_s2_win10": dict(image_size=(80, 80), num_classes=10, dim=32, depth=(1, 2), heads=(2, 4), ssa_dim_key=(24, 40),
                          ssa_dim_value=(16, 32), reduction_factor=(4, 1), window_size=(10, None), iwsa_dim_key=16,
                          iwsa_dim_value=(32, 48)),
    "scalable_vit_rect_odd": dict(image_size=(60, 44), num_classes=7, dim=24, depth=(1, 1), heads=3, ssa_dim_key=16, ssa_dim_value=16,
                          reduction_factor=(2, 3), window_size=(None, 2), iwsa_dim_key=32, iwsa_dim_value=32),
    "scalable_vit_4stage": dict(image_size=(64, 64), num_classes=5, dim=16, depth=(1, 1, 1, 1), heads=(1, 2, 2, 4), ssa_dim_key=8,
                        ssa_dim_value=(8, 8, 8, 12), reduction_factor=(4, 2, 1, 1), window_size=(4, None, 2, None), iwsa_dim_key=(8, 16, 72, 8),
                        iwsa_dim_value=(8, 16, 40, 8), ff_expansion_factor=2),
    "scalable_vit_1stage": dict(image_size=(48, 40), num_classes=6, dim=64, depth=(2,), heads=2, ssa_dim_key=32, ssa_dim_value=32,
                        reduction_factor=3, window_size=None, iwsa_dim_key=64, iwsa_dim_value=48, ff_expansion_factor=2),
}
BENCH = {"scalable_vit_readme": dict(image_size=(256, 256), **README),
         "scalable_vit_win8": dict(image_size=(256, 256), **{**README, "window_size": (8, 8, None, None)})}
WEIGHT_SEED, IMAGE_SEED, BATCH = 41, 42, 2


def random_config(seed):
    """A small random config (1 to 4 stages, any of the per-stage hyperparameters as a tuple or a scalar) and an image size it runs
    at: every stage map at least its reduction_factor and divisible by its window."""
    rnd = random.Random(seed)
    n = rnd.randint(1, 4)
    h0, w0 = rnd.choice([4, 6, 8]) * 2 ** (n - 1), rnd.choice([4, 6, 8]) * 2 ** (n - 1)
    maps = [(h0 >> i, w0 >> i) for i in range(n)]

    def per_stage(choices):
        v = tuple(rnd.choice(choices) for _ in range(n))
        return v if rnd.random() < 0.7 else v[0]
    r = tuple(rnd.choice([d for d in (1, 2, 3, 4) if d <= min(maps[i])]) for i in range(n))
    win = tuple(rnd.choice([None] + [d for d in (2, 4) if maps[i][0] % d == 0 and maps[i][1] % d == 0]) for i in range(n))
    cfg = make_config(image_size=(4 * h0 - rnd.randint(0, 3), 4 * w0 - rnd.randint(0, 3)), num_classes=rnd.randint(2, 6),
                      dim=rnd.choice([8, 12, 16]), depth=tuple(rnd.randint(0, 2) for _ in range(n)), heads=per_stage([1, 2, 3]),
                      ssa_dim_key=per_stage([4, 8, 12]), ssa_dim_value=per_stage([4, 8]), reduction_factor=r,
                      window_size=win if rnd.random() < 0.8 else None, iwsa_dim_key=per_stage([4, 8]),
                      iwsa_dim_value=per_stage([4, 8, 12]), ff_expansion_factor=rnd.choice([1, 2, 4]))
    return cfg

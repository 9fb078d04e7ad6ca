"""Test oracle of Twins-SVT (reference twins_svt.py), kept beside the tests that use it.

  * make_config / weight_specs / init_weights / stress_weights: configs and seeded weights in the engine's names (SURVEY.md
    App. B: the reference's attribute paths), the reference's initial distributions;
  * forward: the float64 numpy restatement of TwinsSVT.call (twins_svt.py:266-268);
  * forward_torch: an independent PyTorch restatement (F.pixel_unshuffle for the c-slowest patch vectors, F.unfold / F.fold for
    the windows, F.conv2d for the VALID k|v convolution and the grouped SAME PEG with explicit asymmetric padding);
  * installed(): cvt_oracle's stand-in, which already covers what twins_svt.py calls (Conv2D with groups and VALID strides,
    tf.math.reduce_variance, tf.sqrt, tf.ones, GlobalAvgPool2D), so the reference's twins_svt.py runs unmodified; load_weights
    sets the oracle's weights by attribute path.

The TensorFlow semantics restated here (third-party, public API documentation): 'VALID' gives floor((in - k) / stride) + 1
positions; 'SAME' at stride 1 pads k - 1 in total, the smaller half, (k - 1) // 2, on the top and left.
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
from vit_tensorflow_b200.models import TWINS_CTOR_KEYS, TWINS_STAGE_KEYS

TWINS_DEFAULTS = dict(s1_emb_dim=64, s1_patch_size=4, s1_local_patch_size=7, s1_global_k=7, s1_depth=1, s2_emb_dim=128, s2_patch_size=2,
                      s2_local_patch_size=7, s2_global_k=7, s2_depth=1, s3_emb_dim=256, s3_patch_size=2, s3_local_patch_size=7,
                      s3_global_k=7, s3_depth=5, s4_emb_dim=512, s4_patch_size=2, s4_local_patch_size=7, s4_global_k=7, s4_depth=4,
                      peg_kernel_size=3, dropout=0.0)   # twins_svt.py:217-239
HEADS, DIM_HEAD, MLP_MULT = 8, 64, 4                    # never passed to Transformer (twins_svt.py:254-258)
INNER = HEADS * DIM_HEAD
LN_EPS = cvt_oracle.LN_EPS


def make_config(image_size=224, image_w=None, **kw) -> dict:
    """A Twins-SVT config: the reference's constructor kwargs (defaults filled in) plus the image size the tests call it with."""
    cfg = dict(TWINS_DEFAULTS)
    cfg.update(kw)
    cfg["kind"] = "twins_svt"
    cfg["image_h"], cfg["image_w"] = image_size, image_w or image_size
    return cfg


def ctor_kwargs(cfg) -> dict:
    return {k: cfg[k] for k in TWINS_CTOR_KEYS if k in cfg}


def stages(cfg):
    return [{k: cfg[f"s{i}_{k}"] for k in TWINS_STAGE_KEYS} for i in (1, 2, 3, 4)]


def layer_prefixes(cfg, st):
    """The layer prefixes of stage st: the depth-1 Transformer before the PEG, then the depth-s one after it."""
    p = f"svt_layers.{st}."
    return [f"{p}1.layers.0."] + [f"{p}3.layers.{L}." for L in range(stages(cfg)[st]["depth"])]


def weight_specs(cfg):
    s = collections.OrderedDict()
    cin = 3
    for st, c in enumerate(stages(cfg)):
        p, d, ps, kg, k = f"svt_layers.{st}.", c["emb_dim"], c["patch_size"], c["global_k"], cfg["peg_kernel_size"]

        def ln(n):
            s[n + ".g"], s[n + ".b"] = ((1, 1, 1, d), "ones"), ((1, 1, 1, d), "zeros")

        def mlp(m):
            ln(m + ".fn.norm")
            s[m + ".fn.fn.net.0.kernel"], s[m + ".fn.fn.net.0.bias"] = ((1, 1, d, MLP_MULT * d), "glorot"), ((MLP_MULT * d,), "zeros")
            s[m + ".fn.fn.net.3.kernel"], s[m + ".fn.fn.net.3.bias"] = ((1, 1, MLP_MULT * d, d), "glorot"), ((d,), "zeros")

        s[p + "0.proj.kernel"], s[p + "0.proj.bias"] = ((1, 1, cin * ps * ps, d), "glorot"), ((d,), "zeros")
        for i, b in enumerate(layer_prefixes(cfg, st)):
            if st < 3:
                ln(b + "0.fn.norm")
                s[b + "0.fn.fn.to_q.kernel"] = ((1, 1, d, INNER), "glorot")
                s[b + "0.fn.fn.to_kv.kernel"] = ((1, 1, d, 2 * INNER), "glorot")
                s[b + "0.fn.fn.to_out.0.kernel"], s[b + "0.fn.fn.to_out.0.bias"] = ((1, 1, INNER, d), "glorot"), ((d,), "zeros")
                mlp(b + "1")
            ln(b + "2.fn.norm")
            s[b + "2.fn.fn.to_q.kernel"] = ((1, 1, d, INNER), "glorot")
            s[b + "2.fn.fn.to_kv.kernel"] = ((kg, kg, d, 2 * INNER), "glorot")
            s[b + "2.fn.fn.to_out.0.kernel"], s[b + "2.fn.fn.to_out.0.bias"] = ((1, 1, INNER, d), "glorot"), ((d,), "zeros")
            mlp(b + "3")
            if i == 0:
                s[p + "2.proj.fn.kernel"], s[p + "2.proj.fn.bias"] = ((k, k, 1, d), "glorot"), ((d,), "zeros")
        cin = d
    s["svt_layers.4.1.kernel"], s["svt_layers.4.1.bias"] = ((cin, cfg["num_classes"]), "glorot"), ((cfg["num_classes"],), "zeros")
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
    """init_weights with what the defaults hide: non-zero biases, LayerNorm g = 1 + 0.2 N and b = 0.2 N."""
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
    from vit_tensorflow_b200.models import twins_size_error
    return twins_size_error(stages(cfg), h, w)


# ------------------------------------------------------------------------------------------------ float64 spec
layer_norm = cvt_oracle.layer_norm


def conv1x1(x, w, n, bias=True):
    k = w[n + ".kernel"]
    y = x @ k.reshape(k.shape[-2], k.shape[-1])
    return y + w[n + ".bias"] if bias else y


def softmax_attention(q, k, v):
    """q [..., n, d], k / v [..., m, d]: softmax(q k^T / 8) v."""
    dots = q @ np.swapaxes(k, -1, -2) * DIM_HEAD ** -0.5
    a = np.exp(dots - dots.max(-1, keepdims=True))
    return (a / a.sum(-1, keepdims=True)) @ v


def local_attention(y, w, a, p):
    """LocalAttention.call (twins_svt.py:135-156) on the normalised map y [b, H, W, dim]."""
    b, H, W, _ = y.shape
    q, kv = conv1x1(y, w, a + "to_q", False), conv1x1(y, w, a + "to_kv", False)

    def windows(t):                                   # b (x p1) (y p2) (h d) -> (b x y) h (p1 p2) d
        return t.reshape(b, H // p, p, W // p, p, HEADS, DIM_HEAD).transpose(0, 1, 3, 5, 2, 4, 6).reshape(-1, HEADS, p * p, DIM_HEAD)

    o = softmax_attention(windows(q), windows(kv[..., :INNER]), windows(kv[..., INNER:]))
    o = o.reshape(b, H // p, W // p, HEADS, p, p, DIM_HEAD).transpose(0, 1, 4, 2, 5, 3, 6).reshape(b, H, W, INNER)
    return conv1x1(o, w, a + "to_out.0")


def global_attention(y, w, a, k):
    """GlobalAttention.call (twins_svt.py:175-190): to_kv is Conv2D(k, stride k, VALID), floor(H / k) x floor(W / k) keys."""
    b, H, W, C = y.shape
    q = conv1x1(y, w, a + "to_q", False)
    kh, kw = (H - k) // k + 1, (W - k) // k + 1
    patches = y[:, :kh * k, :kw * k].reshape(b, kh, k, kw, k, C).transpose(0, 1, 3, 2, 4, 5).reshape(b, kh * kw, k * k * C)
    kv = _store(_store(patches) @ _store(w[a + "to_kv.kernel"].reshape(k * k * C, 2 * INNER)))

    def heads(t):
        return t.reshape(b, -1, HEADS, DIM_HEAD).transpose(0, 2, 1, 3)

    o = softmax_attention(heads(q.reshape(b, H * W, INNER)), heads(kv[..., :INNER]), heads(kv[..., INNER:]))
    return conv1x1(o.transpose(0, 2, 1, 3).reshape(b, H, W, INNER), w, a + "to_out.0")


def mlp(y, w, a):
    return conv1x1(spec_numpy.gelu(conv1x1(y, w, a + "net.0")), w, a + "net.3")


def patch_embedding(x, w, n, p):
    """PatchEmbedding.call (twins_svt.py:101-106): 'b (h p1) (w p2) c -> b h w (c p1 p2)', then the 1x1 Conv2D."""
    b, H, W, C = x.shape
    x = x.reshape(b, H // p, p, W // p, p, C).transpose(0, 1, 3, 5, 2, 4).reshape(b, H // p, W // p, C * p * p)
    return conv1x1(x, w, n)


def _store(x):                                       # forward_bf16_storage rounds what the engine stores here
    return x


def layer(x, w, b, c, local):
    if local:
        x = _store(local_attention(layer_norm(x, w[b + "0.fn.norm.g"], w[b + "0.fn.norm.b"]), w, b + "0.fn.fn.", c["local_patch_size"]) + x)
        x = _store(mlp(layer_norm(x, w[b + "1.fn.norm.g"], w[b + "1.fn.norm.b"]), w, b + "1.fn.fn.") + x)
    x = _store(global_attention(layer_norm(x, w[b + "2.fn.norm.g"], w[b + "2.fn.norm.b"]), w, b + "2.fn.fn.", c["global_k"]) + x)
    return _store(mlp(layer_norm(x, w[b + "3.fn.norm.g"], w[b + "3.fn.norm.b"]), w, b + "3.fn.fn.") + x)


def forward(img, weights, cfg, dtype=np.float64):
    """TwinsSVT.call(img) -> logits [b, num_classes] (no dropout, no BatchNorm: training does not matter at dropout 0)."""
    w = {k: np.asarray(v, dtype=dtype) for k, v in weights.items()}
    x = np.asarray(img, dtype=dtype)
    for st, c in enumerate(stages(cfg)):
        p = f"svt_layers.{st}."
        x = patch_embedding(x, w, p + "0.proj", c["patch_size"])
        pre, *post = layer_prefixes(cfg, st)
        x = layer(x, w, pre, c, st < 3)
        x = _store(x + cvt_oracle.dwconv_same(x, w[p + "2.proj.fn.kernel"], 1) + w[p + "2.proj.fn.bias"])   # PEG :108-115
        for b in post:
            x = layer(x, w, b, c, st < 3)
    return spec_numpy.dense(x.mean(axis=(1, 2)), w, "svt_layers.4.1")


def forward_torch(img, weights, cfg):
    """The same model restated in PyTorch (float64, NCHW)."""
    import torch
    import torch.nn.functional as F
    t = {k: torch.from_numpy(np.asarray(v, np.float64)) for k, v in weights.items()}
    x = torch.from_numpy(np.asarray(img, np.float64)).permute(0, 3, 1, 2)

    def ln(x, n):
        return F.layer_norm(x.permute(0, 2, 3, 1), (x.shape[1],), t[n + ".g"].reshape(-1), t[n + ".b"].reshape(-1), LN_EPS).permute(0, 3, 1, 2)

    def conv(x, n, bias=True, **kw):
        return F.conv2d(x, t[n + ".kernel"].permute(3, 2, 0, 1), t[n + ".bias"] if bias else None, **kw)

    def attend(q, k, v):                                           # [..., n, 64]
        return F.scaled_dot_product_attention(q, k, v)

    def local(y, a, p):
        b, _, H, W = y.shape
        q, kv = conv(y, a + "to_q", False), conv(y, a + "to_kv", False)
        L = (H // p) * (W // p)

        def win(z):                                                # [b, 512, H, W] -> [b, L, heads, p^2, 64]
            return F.unfold(z, p, stride=p).view(b, HEADS, DIM_HEAD, p * p, L).permute(0, 4, 1, 3, 2)

        o = attend(win(q), win(kv[:, :INNER]), win(kv[:, INNER:]))
        o = F.fold(o.permute(0, 2, 4, 3, 1).reshape(b, INNER * p * p, L), (H, W), p, stride=p)
        return conv(o, a + "to_out.0")

    def glob(y, a, k):
        b, _, H, W = y.shape
        q, kv = conv(y, a + "to_q", False), conv(y, a + "to_kv", False, stride=k)

        def heads(z):                                              # [b, 512, h, w] -> [b, heads, h*w, 64]
            return z.flatten(2).view(b, HEADS, DIM_HEAD, -1).transpose(-1, -2)

        o = attend(heads(q), heads(kv[:, :INNER]), heads(kv[:, INNER:]))
        return conv(o.transpose(-1, -2).reshape(b, INNER, H, W), a + "to_out.0")

    def ff(y, a):
        return conv(F.gelu(conv(y, a + "net.0")), a + "net.3")

    def lay(x, b, c, has_local):
        if has_local:
            x = local(ln(x, b + "0.fn.norm"), b + "0.fn.fn.", c["local_patch_size"]) + x
            x = ff(ln(x, b + "1.fn.norm"), b + "1.fn.fn.") + x
        x = glob(ln(x, b + "2.fn.norm"), b + "2.fn.fn.", c["global_k"]) + x
        return ff(ln(x, b + "3.fn.norm"), b + "3.fn.fn.") + x

    k = cfg["peg_kernel_size"]
    for st, c in enumerate(stages(cfg)):
        p = f"svt_layers.{st}."
        x = conv(F.pixel_unshuffle(x, c["patch_size"]), p + "0.proj")      # channel index c * p^2 + p1 * p + p2
        pre, *post = layer_prefixes(cfg, st)
        x = lay(x, pre, c, st < 3)
        lo = (k - 1) // 2
        x = x + F.conv2d(F.pad(x, (lo, k - 1 - lo, lo, k - 1 - lo)), t[p + "2.proj.fn.kernel"].permute(3, 2, 0, 1), t[p + "2.proj.fn.bias"],
                         groups=x.shape[1])
        for b in post:
            x = lay(x, b, c, st < 3)
    return (x.mean(dim=(2, 3)) @ t["svt_layers.4.1.kernel"] + t["svt_layers.4.1.bias"]).numpy()


def bf16_round(x):
    return cvt_oracle.bf16_round(x)


def forward_bf16_storage(img, weights, cfg):
    """forward() with what the bf16 engine stores rounded to bfloat16 -- the operands and results of every 1x1 convolution and of
    the global to_kv, the residual stream after every sub-block and the PEG -- and everything else in float64: a lower estimate of
    what storing activations and weights in bf16 alone costs."""
    global conv1x1, _store
    exact, store = conv1x1, _store

    def rounded(x, w, n, bias=True):
        k = w[n + ".kernel"]
        y = bf16_round(x) @ bf16_round(k.reshape(k.shape[-2], k.shape[-1]))
        return bf16_round(y + w[n + ".bias"] if bias else y)
    conv1x1, _store = rounded, bf16_round
    try:
        return forward(img, weights, cfg)
    finally:
        conv1x1, _store = exact, store


# ------------------------------------------------------------------------------------------------ the reference's twins_svt.py
@contextlib.contextmanager
def installed(reference_dir):
    """cvt_oracle.installed(reference_dir); `import twins_svt` inside the block is the reference's own file, removed from
    sys.modules again on exit."""
    saved = sys.modules.pop("twins_svt", None)
    with cvt_oracle.installed(reference_dir) as tf:
        try:
            yield tf
        finally:
            sys.modules.pop("twins_svt", None)
            if saved is not None:
                sys.modules["twins_svt"] = saved


def load_weights(model, w):
    """The oracle's weights into a reference TwinsSVT by attribute path (twins_svt.py:244-264)."""
    seqs = model.svt_layers.layers

    def ln(norm, n):
        norm.g.assign(w[n + ".g"])
        norm.b.assign(w[n + ".b"])

    def conv(layer, n, bias=True):
        layer.set_weights([w[n + ".kernel"], w[n + ".bias"]] if bias else [w[n + ".kernel"]])

    def mlp(res, n):
        ln(res.fn.norm, n + ".fn.norm")
        conv(res.fn.fn.net.layers[0], n + ".fn.fn.net.0")
        conv(res.fn.fn.net.layers[3], n + ".fn.fn.net.3")

    def attn(res, n):
        ln(res.fn.norm, n + ".fn.norm")
        conv(res.fn.fn.to_q, n + ".fn.fn.to_q", False)
        conv(res.fn.fn.to_kv, n + ".fn.fn.to_kv", False)
        conv(res.fn.fn.to_out.layers[0], n + ".fn.fn.to_out.0")

    for st in range(4):
        p = f"svt_layers.{st}."
        pe, tr1, peg, tr2 = seqs[st].layers
        conv(pe.proj, p + "0.proj")
        conv(peg.proj.fn, p + "2.proj.fn")
        for t, tr in ((1, tr1), (3, tr2)):
            for L, (la, f1, ga, f2) in enumerate(tr.layers):
                b = f"{p}{t}.layers.{L}."
                if st < 3:
                    attn(la, b + "0")
                    mlp(f1, b + "1")
                attn(ga, b + "2")
                mlp(f2, b + "3")
    seqs[4].layers[1].set_weights([w["svt_layers.4.1.kernel"], w["svt_layers.4.1.bias"]])


@contextlib.contextmanager
def reference_module(reference_dir, dtype=np.float64):
    """The reference's twins_svt module over the stand-in in `dtype`."""
    import importlib
    tf_shim.set_dtype(dtype)
    try:
        with installed(reference_dir):
            yield importlib.import_module("twins_svt")
    finally:
        tf_shim.set_dtype(np.float32)


def reference_logits(mod, cfg, w, img, dtype=np.float64):
    """Build the reference's TwinsSVT for `cfg`, call it once on `img` so that Keras builds every variable, load `w` and return
    `model(img)` (its default training=True: there is no BatchNorm and the dropout rate is 0)."""
    model = mod.TwinsSVT(**ctor_kwargs(cfg))
    model(np.asarray(img, dtype))
    load_weights(model, {k: np.asarray(v, dtype) for k, v in w.items()})
    out = model(np.asarray(img, dtype))
    return np.asarray(out).view(np.ndarray).copy()


def random_config(seed):
    """A small random configuration: windows with p^2 below, at and above 64, global_k unrelated to the window with
    floor-truncated key maps, even PEG kernels, widths off 64 and non-square images.  Built from stage 1 down, so that every
    map is divisible by the next patch_size and its own local_patch_size."""
    r = random.Random(seed)
    kw = dict(num_classes=r.randint(2, 9), peg_kernel_size=(1, 2, 3, 4, 5)[seed % 5], dropout=0.0)
    pl = (2, 3, 4, 8, 9)[seed % 5]
    h, w = pl * r.choice([1, 2]), pl * r.choice([1, 2])
    ps1 = r.choice([1, 2, 3])
    image = (h * ps1, w * ps1)
    for i in (1, 2, 3, 4):
        if i > 1:
            g = math.gcd(h, w)
            ps = r.choice([d for d in (1, 2) if g % d == 0])
            h, w = h // ps, w // ps
            g = math.gcd(h, w)
            pl = r.choice([d for d in (1, 2, 3, 4) if g % d == 0]) if i < 4 else 7
        else:
            ps = ps1
        kw.update({f"s{i}_emb_dim": r.choice([8, 16, 40, 64, 72]), f"s{i}_patch_size": ps, f"s{i}_local_patch_size": pl,
                   f"s{i}_global_k": r.randint(1, min(h, w, 5)), f"s{i}_depth": r.randint(0, 1)})
    return make_config(image_size=image[0], image_w=image[1], **kw)


# ------------------------------------------------------------------------------------------------ cases
def _small(**kw):
    base = dict(num_classes=10, s1_emb_dim=64, s1_patch_size=2, s1_local_patch_size=4, s1_global_k=4, s1_depth=1,
                s2_emb_dim=64, s2_patch_size=2, s2_local_patch_size=8, s2_global_k=3, s2_depth=1,
                s3_emb_dim=128, s3_patch_size=2, s3_local_patch_size=2, s3_global_k=2, s3_depth=1,
                s4_emb_dim=128, s4_patch_size=1, s4_local_patch_size=7, s4_global_k=4, s4_depth=1, peg_kernel_size=3)
    base.update(kw)
    return base


# small cases (fixtures with float32 and float64 reference logits) and the two configurations tools/twins_bench.py measures
SMALL = {
    # maps 16 -> 8 -> 4 -> 4: windows of 16, 64 and 4 tokens; global keys 4 x 4, 2 x 2 (floor), 2 x 2 and 1 (softmax = 1)
    "twins_small": dict(image_size=32, **_small()),
    # a 36 x 72 image: 9 x 9 windows (81 tokens: two query tiles and key blocks), even PEG kernel, widths 40 / 72
    "twins_p9_wide": dict(image_size=36, image_w=72, **_small(s1_emb_dim=40, s1_local_patch_size=9, s1_global_k=5, s2_emb_dim=72,
                                                              s2_patch_size=1, s2_local_patch_size=6, s2_global_k=4, s3_local_patch_size=3,
                                                              s4_emb_dim=40, s4_patch_size=3, s4_global_k=3, peg_kernel_size=2)),
    # 7 x 7 windows as in the README model, PEG kernel 4, the stage-4 map equal to global_k
    "twins_p7": dict(image_size=56, **_small(s1_patch_size=4, s1_local_patch_size=7, s1_global_k=7, s2_patch_size=1, s2_local_patch_size=7,
                                             s2_global_k=5, s3_patch_size=2, s3_local_patch_size=7, s3_global_k=3, s3_depth=2,
                                             s4_patch_size=1, s4_global_k=7, peg_kernel_size=4)),
}
BENCH = {
    "twins_readme": dict(image_size=224, num_classes=1000),                   # the reference README's model = the defaults
    "twins_2_2_10_4": dict(image_size=224, num_classes=1000, s3_depth=9, s4_depth=3),
}
WEIGHT_SEED, IMAGE_SEED, BATCH = 41, 42, 2

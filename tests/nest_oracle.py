"""Test oracle of NesT (reference nest.py), kept beside the tests that use it.

  * make_config / weight_specs / init_weights / stress_weights: configs and seeded weights in the engine's names (SURVEY.md
    App. B: the reference's attribute paths), the reference's initial distributions;
  * forward: the float64 numpy restatement of NesT.call (nest.py:202-216);
  * forward_torch: an independent PyTorch restatement (F.conv2d with explicit SAME padding, F.max_pool2d over a -inf pad, blocks
    by reshape / permute, F.scaled_dot_product_attention);
  * forward_bf16_storage: forward() with what the bf16 engine stores rounded to bfloat16;
  * block_attention / aggregate_tail: the engine's two NesT operators on their own (vb_op_block_attention, vb_op_nest_aggregate);
  * installed(): crossformer_oracle's stand-in, under which the reference's nest.py runs unmodified (it adds nothing beyond it);
    load_weights sets the oracle's weights by attribute path.

The TensorFlow semantics restated here (third-party, public API documentation): Conv2D / MaxPool2D 'SAME' give ceil(in / stride)
positions and pad max((out - 1) * stride + k - in, 0) in total, the smaller half on the top and left; padded taps never win a max.
"""
from __future__ import annotations

import collections
import contextlib
import math
import random
import sys

import numpy as np

import cct_oracle
import crossformer_oracle
from oracle import spec_numpy, tf_shim
from vit_tensorflow_b200.models import NEST_CTOR_KEYS, nest_plan, nest_size_error

NEST_DEFAULTS = dict(mlp_mult=4, dropout=0.0)             # nest.py:159-160
LN_EPS = 1e-5                                             # the module's LayerNorm (nest.py:29)


def make_config(image_size=224, image_h=None, image_w=None, **kw) -> dict:
    """A NesT config: the reference's constructor kwargs (defaults filled in) plus the image size the tests call it with (image_h x
    image_w, image_size x image_size unless given)."""
    cfg = dict(NEST_DEFAULTS)
    cfg.update(kw)
    cfg["kind"] = "nest"
    cfg["image_size"] = image_size
    cfg["image_h"], cfg["image_w"] = image_h or image_size, image_w or image_h or image_size
    return cfg


def ctor_kwargs(cfg) -> dict:
    return {k: cfg[k] for k in NEST_CTOR_KEYS if k in cfg}


def plan(cfg):
    return nest_plan(cfg["image_size"], cfg["patch_size"], cfg["dim"], cfg["heads"], cfg["num_hierarchies"], cfg["block_repeats"])


def weight_specs(cfg):
    pl = plan(cfg)
    s = collections.OrderedDict()
    p, d0, dh, mult = cfg["patch_size"], cfg["dim"], cfg["dim"] // cfg["heads"], cfg["mlp_mult"]
    s["patch_embedding.1.kernel"], s["patch_embedding.1.bias"] = ((1, 1, p * p * 3, d0), "glorot"), ((d0,), "zeros")
    for i, lv in enumerate(pl["levels"]):
        pre, d = f"nest_layers.{i}.", lv["dim"]
        inner = dh * lv["heads"]
        s[pre + "0.pos_emb"] = ((pl["seq_len"],), "normal")
        for L in range(lv["depth"]):
            b = f"{pre}0.layers.{L}."
            s[b + "0.norm.g"], s[b + "0.norm.b"] = ((1, 1, 1, d), "ones"), ((1, 1, 1, d), "zeros")
            s[b + "0.fn.to_qkv.kernel"] = ((1, 1, d, 3 * inner), "glorot")
            s[b + "0.fn.to_out.0.kernel"], s[b + "0.fn.to_out.0.bias"] = ((1, 1, inner, d), "glorot"), ((d,), "zeros")
            s[b + "1.norm.g"], s[b + "1.norm.b"] = ((1, 1, 1, d), "ones"), ((1, 1, 1, d), "zeros")
            s[b + "1.fn.net.0.kernel"], s[b + "1.fn.net.0.bias"] = ((1, 1, d, d * mult), "glorot"), ((d * mult,), "zeros")
            s[b + "1.fn.net.3.kernel"], s[b + "1.fn.net.3.bias"] = ((1, 1, d * mult, d), "glorot"), ((d,), "zeros")
        if lv["aggregate"]:
            dn = 2 * d
            s[pre + "1.ag_layers.0.kernel"], s[pre + "1.ag_layers.0.bias"] = ((3, 3, d, dn), "glorot"), ((dn,), "zeros")
            s[pre + "1.ag_layers.1.g"], s[pre + "1.ag_layers.1.b"] = ((1, 1, 1, dn), "ones"), ((1, 1, 1, dn), "zeros")
    last = pl["last_dim"]
    s["mlp_head.0.g"], s["mlp_head.0.b"] = ((1, 1, 1, last), "ones"), ((1, 1, 1, last), "zeros")
    s["mlp_head.2.kernel"], s["mlp_head.2.bias"] = ((last, cfg["num_classes"]), "glorot"), ((cfg["num_classes"],), "zeros")
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
        elif init == "normal":                                # tf.random.normal([seq_len]), nest.py:129
            a = rng.standard_normal(shape)
        else:
            raise AssertionError(init)
        out[name] = np.ascontiguousarray(a, dtype=np.float32)
    return out


def stress_weights(cfg, seed=1):
    """init_weights with what the defaults hide: non-zero biases (0.2 N), LayerNorm g = 1 + 0.2 N with every fifth channel
    negated (the aggregation's LayerNorm comes before the max), b = 0.2 N, and N(0, 1) pos_emb."""
    rng = np.random.default_rng(seed)
    out = init_weights(cfg, seed)
    for name, (shape, init) in weight_specs(cfg).items():
        if init == "ones":
            a = 1.0 + 0.2 * rng.standard_normal(shape)
            a.reshape(-1)[::5] *= -1.0
        elif init == "zeros":
            a = 0.2 * rng.standard_normal(shape)
        elif init == "normal":
            a = rng.standard_normal(shape)
        else:
            continue
        out[name] = a.astype(np.float32)
    return out


def make_image(cfg, batch, seed=0, h=None, w=None):
    rng = np.random.default_rng(seed)
    return rng.standard_normal((batch, h or cfg["image_h"], w or cfg["image_w"], 3), dtype=np.float32)


def size_error(cfg, h, w):
    return nest_size_error(plan(cfg), h, w)


# ------------------------------------------------------------------------------------------------ float64 spec
def layer_norm(x, g, b, eps=LN_EPS):
    mu = x.mean(-1, keepdims=True)
    return (x - mu) / np.sqrt(x.var(-1, keepdims=True) + eps) * np.reshape(g, -1) + np.reshape(b, -1)


def _store(x):                                            # forward_bf16_storage rounds what the engine stores here
    return x


def _matmul(x, k):                                        # forward_bf16_storage rounds the operands and the result
    return x @ k


def conv1x1(x, w, n, bias=True):
    k = w[n + ".kernel"]
    y = _matmul(x, k.reshape(k.shape[-2], k.shape[-1]))
    return _store(y + w[n + ".bias"] if bias else y)


def conv3x3_same(x, k, bias):
    """Conv2D(3, SAME, stride 1) with bias: one pixel of zeros on every side."""
    b, H, W, C = x.shape
    xp = np.pad(x, ((0, 0), (1, 1), (1, 1), (0, 0)))
    cols = np.concatenate([xp[:, ky:ky + H, kx:kx + W] for ky in range(3) for kx in range(3)], -1)
    return _store(_matmul(cols, k.reshape(9 * C, -1)) + bias)


def to_blocks(t, bs):
    """'b (b1 h) (b2 w) c -> (b b1 b2) (h w) c' (nest.py:209, the Transformer's token order)."""
    b, H, W, c = t.shape
    return t.reshape(b, bs, H // bs, bs, W // bs, c).transpose(0, 1, 3, 2, 4, 5).reshape(b * bs * bs, (H // bs) * (W // bs), c)


def from_blocks(t, b, H, W, bs):
    c = t.shape[-1]
    return t.reshape(b, bs, bs, H // bs, W // bs, c).transpose(0, 1, 3, 2, 4, 5).reshape(b, H, W, c)


def softmax_attention(qkv, heads, dh):
    """softmax(q k^T * dh^-0.5) v per head over the rows of qkv [n_blocks, n, 3 * heads * dh] -> [n_blocks, n, heads * dh]."""
    inner = heads * dh
    q, k, v = (qkv[..., i * inner:(i + 1) * inner].reshape(qkv.shape[0], -1, heads, dh).transpose(0, 2, 1, 3) for i in range(3))
    sim = q @ np.swapaxes(k, -1, -2) * dh ** -0.5
    a = np.exp(sim - sim.max(-1, keepdims=True))
    o = (a / a.sum(-1, keepdims=True)) @ v
    return o.transpose(0, 2, 1, 3).reshape(qkv.shape[0], -1, inner)


def block_attention(qkv, heads, dh, bh, bw):
    """NesT's attention within bh x bw blocks of a pixel-major map: qkv [b, H, W, >= 3 heads dh] -> [b, H, W, heads dh]."""
    b, H, W, _ = qkv.shape
    t = qkv[..., :3 * heads * dh].reshape(b, H // bh, bh, W // bw, bw, -1).transpose(0, 1, 3, 2, 4, 5).reshape(-1, bh * bw, 3 * heads * dh)
    o = softmax_attention(t, heads, dh)
    return o.reshape(b, H // bh, W // bw, bh, bw, -1).transpose(0, 1, 3, 2, 4, 5).reshape(b, H, W, -1)


def aggregate_tail(x, g, b, pos=None, bh=1, bw=1):
    """LayerNorm (eps 1e-5) -> MaxPool2D(3, 2, SAME) -> + pos[(r % bh) * bw + c % bw] (the next level's position add)."""
    y = cct_oracle.maxpool_same(layer_norm(x, g, b), 3, 2)
    if pos is not None:
        y = y + np.tile(np.reshape(pos, (bh, bw)), (y.shape[1] // bh, y.shape[2] // bw))[None, :, :, None]
    return y


def attention(x, w, a, heads, dh):
    """PreNorm(Attention).call (nest.py:50-51, 93-109) over one block of tokens: x [n_blocks, h, w, d]."""
    nb, h, wd, d = x.shape
    qkv = conv1x1(layer_norm(x, w[a + "0.norm.g"], w[a + "0.norm.b"]), w, a + "0.fn.to_qkv", False)
    o = softmax_attention(qkv.reshape(nb, h * wd, -1), heads, dh).reshape(nb, h, wd, -1)
    return conv1x1(_store(o), w, a + "0.fn.to_out.0")


def mlp(x, w, a):
    y = conv1x1(layer_norm(x, w[a + "1.norm.g"], w[a + "1.norm.b"]), w, a + "1.fn.net.0")
    return conv1x1(_store(spec_numpy.gelu(y)), w, a + "1.fn.net.3")


def forward(img, weights, cfg, dtype=np.float64):
    """NesT.call(img) -> logits [b, num_classes] (no BatchNorm; dropout 0)."""
    pl = plan(cfg)
    w = {k: np.asarray(v, dtype=dtype) for k, v in weights.items()}
    x = np.asarray(img, dtype=dtype)
    b, H, W, c = x.shape
    p, dh = cfg["patch_size"], cfg["dim"] // cfg["heads"]
    x = x.reshape(b, H // p, p, W // p, p, c).transpose(0, 1, 3, 2, 4, 5).reshape(b, H // p, W // p, p * p * c)   # (p1 p2 c)
    x = conv1x1(x, w, "patch_embedding.1")
    n = len(pl["levels"])
    for i, lv in enumerate(pl["levels"]):
        pre, bs = f"nest_layers.{i}.", 2 ** (n - 1 - i)
        mh, mw = x.shape[1], x.shape[2]
        bh, bw = mh // bs, mw // bs
        t = to_blocks(x, bs).reshape(-1, bh, bw, x.shape[-1])
        t = _store(t + w[pre + "0.pos_emb"][:bh * bw].reshape(1, bh, bw, 1))           # nest.py:140-142
        for L in range(lv["depth"]):
            a = f"{pre}0.layers.{L}."
            t = _store(attention(t, w, a, lv["heads"], dh) + t)
            t = _store(mlp(t, w, a) + t)
        x = from_blocks(t.reshape(t.shape[0], bh * bw, -1), b, mh, mw, bs)
        if lv["aggregate"]:
            y = conv3x3_same(x, w[pre + "1.ag_layers.0.kernel"], w[pre + "1.ag_layers.0.bias"])
            x = cct_oracle.maxpool_same(layer_norm(y, w[pre + "1.ag_layers.1.g"], w[pre + "1.ag_layers.1.b"]), 3, 2)
    y = layer_norm(x, w["mlp_head.0.g"], w["mlp_head.0.b"])                             # nest.py:196-200
    return spec_numpy.dense(y.mean(axis=(1, 2)), w, "mlp_head.2")


def forward_torch(img, weights, cfg):
    """The same model restated in PyTorch (float64, NCHW)."""
    import torch
    import torch.nn.functional as F
    pl = plan(cfg)
    t = {k: torch.from_numpy(np.asarray(v, np.float64)) for k, v in weights.items()}
    x = torch.from_numpy(np.asarray(img, np.float64)).permute(0, 3, 1, 2)
    p, dh = cfg["patch_size"], cfg["dim"] // cfg["heads"]

    def ln(x, n):
        return F.layer_norm(x.permute(0, 2, 3, 1), (x.shape[1],), t[n + ".g"].reshape(-1), t[n + ".b"].reshape(-1), LN_EPS).permute(0, 3, 1, 2)

    def conv(x, n, bias=True, padding=0):
        return F.conv2d(x, t[n + ".kernel"].permute(3, 2, 0, 1), t[n + ".bias"] if bias else None, padding=padding)

    # the patch embedding as one p x p stride-p convolution whose kernel rows are the (p1, p2, c) patch vector
    k0 = t["patch_embedding.1.kernel"].reshape(p, p, 3, -1).permute(3, 2, 0, 1)
    x = F.conv2d(x, k0, t["patch_embedding.1.bias"], stride=p)
    n = len(pl["levels"])
    for i, lv in enumerate(pl["levels"]):
        pre, bs = f"nest_layers.{i}.", 2 ** (n - 1 - i)
        b, d, H, W = x.shape
        bh, bw = H // bs, W // bs
        x = x + t[pre + "0.pos_emb"][:bh * bw].reshape(bh, bw).repeat(bs, bs)
        heads = lv["heads"]
        for L in range(lv["depth"]):
            a = f"{pre}0.layers.{L}."
            qkv = conv(ln(x, a + "0.norm"), a + "0.fn.to_qkv", False)                     # [b, 3 inner, H, W]
            z = qkv.reshape(b, 3, heads, dh, bs, bh, bs, bw).permute(1, 0, 4, 6, 2, 5, 7, 3).reshape(3, b * bs * bs, heads, bh * bw, dh)
            o = F.scaled_dot_product_attention(z[0], z[1], z[2])                             # scale dh^-0.5
            o = o.reshape(b, bs, bs, heads, bh, bw, dh).permute(0, 3, 6, 1, 4, 2, 5).reshape(b, heads * dh, H, W)
            x = conv(o, a + "0.fn.to_out.0") + x
            x = conv(F.gelu(conv(ln(x, a + "1.norm"), a + "1.fn.net.0")), a + "1.fn.net.3") + x
        if lv["aggregate"]:
            y = ln(conv(x, pre + "1.ag_layers.0", padding=1), pre + "1.ag_layers.1")
            oh, ow = -(-H // 2), -(-W // 2)
            ph, pw = max((oh - 1) * 2 + 3 - H, 0), max((ow - 1) * 2 + 3 - W, 0)
            y = F.pad(y, (pw // 2, pw - pw // 2, ph // 2, ph - ph // 2), value=-math.inf)
            x = F.max_pool2d(y, 3, 2)
    y = ln(x, "mlp_head.0")
    return (y.mean(dim=(2, 3)) @ t["mlp_head.2.kernel"] + t["mlp_head.2.bias"]).numpy()


def bf16_round(x):
    return crossformer_oracle.bf16_round(x)


def forward_bf16_storage(img, weights, cfg):
    """forward() with what the bf16 engine stores rounded to bfloat16 -- the operands and results of every convolution (the patch
    embedding, the 1x1s, the aggregation's 3 x 3), the attention output, the residual stream after every sub-block and the position
    add -- and everything else in float64: a lower estimate of what storing activations and weights in bf16 alone costs."""
    global _matmul, _store
    exact, store = _matmul, _store
    _matmul, _store = (lambda x, k: bf16_round(bf16_round(x) @ bf16_round(k))), bf16_round
    try:
        return forward(img, weights, cfg)
    finally:
        _matmul, _store = exact, store


# ------------------------------------------------------------------------------------------------ the reference's nest.py
@contextlib.contextmanager
def installed(reference_dir):
    """crossformer_oracle.installed(reference_dir): nest.py needs nothing beyond it (its MaxPool2D, 3 x 3 SAME Conv2D, module
    LayerNorm, einsum attention and einops Rearrange / Reduce are all there).  `import nest` inside the block is the reference's
    own file, removed from sys.modules again on exit."""
    saved = sys.modules.pop("nest", None)
    with crossformer_oracle.installed(reference_dir) as tf:
        try:
            yield tf
        finally:
            sys.modules.pop("nest", None)
            if saved is not None:
                sys.modules["nest"] = saved


def load_weights(model, w):
    """The oracle's weights into a reference NesT by attribute path (nest.py:178-200)."""
    def conv(layer, n, bias=True):
        layer.set_weights([w[n + ".kernel"], w[n + ".bias"]] if bias else [w[n + ".kernel"]])

    def ln(norm, n):
        norm.g.assign(w[n + ".g"])
        norm.b.assign(w[n + ".b"])

    conv(model.patch_embedding.layers[1], "patch_embedding.1")
    for i, (tr, ag) in enumerate(model.nest_layers):
        pre = f"nest_layers.{i}."
        tr.pos_emb.assign(w[pre + "0.pos_emb"])
        for L, (attn, ff) in enumerate(tr.layers):
            a = f"{pre}0.layers.{L}."
            ln(attn.norm, a + "0.norm")
            conv(attn.fn.to_qkv, a + "0.fn.to_qkv", False)
            conv(attn.fn.to_out.layers[0], a + "0.fn.to_out.0")
            ln(ff.norm, a + "1.norm")
            net = ff.fn.net.layers
            conv(net[0], a + "1.fn.net.0")
            conv(net[3], a + "1.fn.net.3")
        if hasattr(ag, "ag_layers"):
            conv(ag.ag_layers.layers[0], pre + "1.ag_layers.0")
            ln(ag.ag_layers.layers[1], pre + "1.ag_layers.1")
    ln(model.mlp_head.layers[0], "mlp_head.0")
    conv(model.mlp_head.layers[2], "mlp_head.2")


@contextlib.contextmanager
def reference_module(reference_dir, dtype=np.float64):
    """The reference's nest module over the stand-in in `dtype`."""
    import importlib
    tf_shim.set_dtype(dtype)
    try:
        with installed(reference_dir):
            yield importlib.import_module("nest")
    finally:
        tf_shim.set_dtype(np.float32)


def reference_model(mod, cfg, w, img, dtype=np.float64):
    model = mod.NesT(**ctor_kwargs(cfg))
    model(np.asarray(img, dtype))
    load_weights(model, {k: np.asarray(v, dtype) for k, v in w.items()})
    return model


def reference_logits(mod, cfg, w, img, dtype=np.float64):
    """Build the reference's NesT for `cfg`, call it once on `img` so that Keras builds every variable, load `w` and return
    `model(img)` (its default training=True: there is no BatchNorm and the dropout rate is 0)."""
    model = reference_model(mod, cfg, w, img, dtype)
    out = model(np.asarray(img, dtype))
    return np.asarray(out).view(np.ndarray).copy()


def random_config(seed):
    """A small random configuration: 1 to 4 hierarchies, head widths 8 to 64 (dim // heads, inner below dim when heads does not
    divide it), block_repeats as an int or a tuple one short, exact or one long, patch sizes 1 to 4, mlp_mult 1 to 4, and square or
    non-square images whose maps meet the shape rules."""
    r = random.Random(seed)
    while True:
        H = r.randint(1, 4)
        heads = r.randint(1, 3)
        dim = heads * r.choice([8, 16, 24, 32]) + r.choice([0, 0, 1])
        n = r.choice([H - 1, H, H, H + 1]) if H > 1 else r.choice([1, 2])
        br = r.randint(0, 2) if r.random() < 0.3 else tuple(r.randint(0, 2) for _ in range(max(n, 1)))
        p = r.randint(1, 4)
        side = r.randint(1, 4) * 2 ** (H - 1)
        kw = dict(image_size=side * p, patch_size=p, num_classes=r.randint(2, 9), dim=dim, heads=heads, num_hierarchies=H,
                  block_repeats=br, mlp_mult=r.randint(1, 4))
        for _ in range(200):
            h, w = r.randint(1, 2 * side) * p, r.randint(1, 2 * side) * p
            cfg = make_config(image_h=h, image_w=w, **kw)
            if size_error(cfg, h, w) is None:
                return cfg


# ------------------------------------------------------------------------------------------------ cases
# small cases (fixtures with float32 and float64 reference logits) and the two configurations tools/nest_bench.py measures
SMALL = {
    # one hierarchy: a single global block of 8 x 8 = 64 tokens, no Aggregate; heads of 32
    "nest_h1": dict(image_size=32, patch_size=4, dim=64, heads=2, num_hierarchies=1, block_repeats=2, num_classes=5),
    # two hierarchies, heads of 64, blocks of 10 x 10 = 100 tokens (two query tiles and key blocks), mlp_mult 2, maps 20 -> 10
    "nest_dh64": dict(image_size=80, patch_size=4, dim=64, heads=1, num_hierarchies=2, block_repeats=(1, 1), mlp_mult=2, num_classes=6),
    # three hierarchies, heads of 24 (the materialised-scores path), widths 48 / 96 / 192 (none a multiple of 64), blocks of 36
    "nest_dh24": dict(image_size=48, patch_size=2, dim=48, heads=2, num_hierarchies=3, block_repeats=(1, 1, 1), num_classes=7),
    # four hierarchies from an int block_repeats, heads of 32, blocks of 4 x 4, maps 32 -> 16 -> 8 -> 4, mlp_mult 2
    "nest_h4": dict(image_size=64, patch_size=2, dim=32, heads=1, num_hierarchies=4, block_repeats=1, mlp_mult=2, num_classes=4),
    # the README's widths and heads (96 / 192 / 384, heads of 32; seq_len 49) called on a 112 x 64 image: maps 28 x 16 -> 14 x 8 ->
    # 7 x 4, rectangular 7 x 4 blocks that use the first 28 pos_emb entries
    "nest_readme_small": dict(image_size=112, image_h=112, image_w=64, patch_size=4, dim=96, heads=3, num_hierarchies=3,
                              block_repeats=(1, 1, 2), num_classes=8),
    # a block_repeats tuple one short: two levels, both with an Aggregate, blocks relative to two levels; runs on a small image
    "nest_short": dict(image_size=64, image_h=32, image_w=32, patch_size=4, dim=32, heads=1, num_hierarchies=3, block_repeats=(1, 1),
                       num_classes=3),
}
BENCH = {
    "nest_readme": dict(image_size=224, patch_size=4, dim=96, heads=3, num_hierarchies=3, block_repeats=(2, 2, 8), num_classes=1000),
    "nest_b": dict(image_size=224, patch_size=4, dim=128, heads=4, num_hierarchies=3, block_repeats=(2, 2, 20), num_classes=1000),
}
WEIGHT_SEED, IMAGE_SEED, BATCH = 61, 62, 2

"""Test oracle of PiT (reference pit.py), kept beside the tests that use it.

  * make_config / stages / weight_specs / init_weights / stress_weights: configs and seeded weights in the engine's names (ViT's,
    SURVEY.md App. B, with layers.L counted across the stages) and the reference's initial distributions;
  * forward: the float64 numpy restatement of PiT.call (pit.py:207-219) as the reference runs it: no Pool is ever built
    (`ind < (len(depth) < 1)` is `ind < 0`, :194), so it is extract_patches(p, p // 2, VALID) + Dense, cls and positions, one ViT
    Transformer per (depth, heads) pair of zip(depth, cast_tuple(heads)), LayerNormalization + Dense on the cls row;
  * reference_module / reference_logits: the reference's own pit.py run unmodified over the numpy stand-in (oracle/tf_shim.py, whose
    extract_patches already has VALID), with the oracle's weights set by attribute path.

The TensorFlow semantics restated here (third-party, public API documentation): extract_patches with 'VALID' gives
floor((in - k) / stride) + 1 windows per side and orders each patch vector (row, column, channel), channel fastest;
LayerNormalization uses the biased variance, epsilon 1e-3.
"""
from __future__ import annotations

import collections
import contextlib
import math

import numpy as np
from scipy.special import erf

from vit_tensorflow_b200.models import PIT_CTOR_KEYS

PIT_DEFAULTS = dict(dim_head=64, dropout=0.0, emb_dropout=0.0)          # pit.py:167-169
LN_EPS = 1e-3


def make_config(**kw) -> dict:
    """A PiT config: the reference's constructor kwargs (defaults filled in)."""
    cfg = dict(PIT_DEFAULTS)
    cfg.update(kw)
    cfg["kind"] = "pit"
    return cfg


def ctor_kwargs(cfg) -> dict:
    return {k: cfg[k] for k in PIT_CTOR_KEYS if k in cfg}


def stages(cfg):
    """The (depth, heads) pairs the reference's zip leaves (pit.py:177,193): heads = cast_tuple(heads, len(depth)), then
    zip(depth, heads), which stops at the shorter of the two."""
    depth, heads = cfg["depth"], cfg["heads"]
    heads = heads if isinstance(heads, tuple) else (heads,) * len(depth)
    return tuple((depth[i], heads[i]) for i in range(min(len(depth), len(heads))))


def num_patches(cfg, h=None, w=None):
    """extract_patches' VALID count per side, floor((side - p) / (p // 2)) + 1, times the other side's."""
    p = cfg["patch_size"]
    side = lambda n: (n - p) // (p // 2) + 1
    return side(h or cfg["image_size"]) * side(w or cfg["image_size"])


def layer_plan(cfg):
    """[(L, stage, heads, project_out)] for every layer, in execution order."""
    out, L = [], 0
    for s, (depth, heads) in enumerate(stages(cfg)):
        for _ in range(depth):
            out.append((L, s, heads, not (heads == 1 and cfg["dim_head"] == cfg["dim"])))   # pit.py:59
            L += 1
    return out


def weight_specs(cfg):
    """name -> (shape, initialiser) in the engine's order."""
    d, dh, mlp = cfg["dim"], cfg["dim_head"], cfg["mlp_dim"]
    sp = collections.OrderedDict()
    sp["pos_embedding"] = ((1, num_patches(cfg) + 1, d), "normal")
    sp["cls_token"] = ((1, 1, d), "normal")
    sp["patch.kernel"], sp["patch.bias"] = ((cfg["patch_size"] ** 2 * 3, d), "glorot"), ((d,), "zeros")
    for L, _, heads, po in layer_plan(cfg):
        p = f"layers.{L}."
        sp[p + "attn_norm.gamma"], sp[p + "attn_norm.beta"] = ((d,), "gamma"), ((d,), "beta")
        sp[p + "to_qkv.kernel"] = ((d, 3 * heads * dh), "glorot")
        if po:
            sp[p + "to_out.kernel"], sp[p + "to_out.bias"] = ((heads * dh, d), "glorot"), ((d,), "zeros")
        sp[p + "ff_norm.gamma"], sp[p + "ff_norm.beta"] = ((d,), "gamma"), ((d,), "beta")
        sp[p + "fc1.kernel"], sp[p + "fc1.bias"] = ((d, mlp), "glorot"), ((mlp,), "zeros")
        sp[p + "fc2.kernel"], sp[p + "fc2.bias"] = ((mlp, d), "glorot"), ((d,), "zeros")
    sp["head_norm.gamma"], sp["head_norm.beta"] = ((d,), "gamma"), ((d,), "beta")
    sp["head.kernel"], sp["head.bias"] = ((d, cfg["num_classes"]), "glorot"), ((cfg["num_classes"],), "zeros")
    return sp


def init_weights(cfg, seed=0):
    """Keras' initialisers: glorot-uniform kernels, zero biases, LayerNormalization gamma 1 / beta 0; pos_embedding and cls_token
    tf.random.normal (pit.py:187-188)."""
    rng = np.random.default_rng(seed)
    out = collections.OrderedDict()
    for name, (shape, init) in weight_specs(cfg).items():
        if init == "glorot":
            lim = math.sqrt(6.0 / (shape[0] + shape[1]))
            a = rng.uniform(-lim, lim, size=shape)
        elif init == "normal":
            a = rng.standard_normal(shape)
        elif init in ("zeros", "beta"):
            a = np.zeros(shape)
        else:
            a = np.ones(shape)
        out[name] = np.ascontiguousarray(a, dtype=np.float32)
    return out


def stress_weights(cfg, seed=1):
    """init_weights with what the Keras defaults hide: non-zero biases and betas (N(0, 0.3)), gammas around 1 (1 + N(0, 0.25))."""
    rng = np.random.default_rng(seed)
    out = init_weights(cfg, seed)
    for name, (shape, init) in weight_specs(cfg).items():
        if init == "gamma":
            out[name] = (1.0 + 0.25 * rng.standard_normal(shape)).astype(np.float32)
        elif init in ("zeros", "beta"):
            out[name] = (0.3 * rng.standard_normal(shape)).astype(np.float32)
    return out


def make_image(cfg, batch, seed=0, h=None, w=None):
    rng = np.random.default_rng(seed)
    return rng.standard_normal((batch, h or cfg["image_size"], w or cfg["image_size"], 3), dtype=np.float32)


# ------------------------------------------------------------------------------------------------ float64 spec
def patches(img, p):
    """extract_patches(p, stride p // 2, VALID) -> [b, oh * ow, p * p * C], vectors (row, column, channel)."""
    s = p // 2
    b, H, W, C = img.shape
    oh, ow = (H - p) // s + 1, (W - p) // s + 1
    out = np.empty((b, oh, ow, p, p, C), img.dtype)
    for y in range(oh):
        for x in range(ow):
            out[:, y, x] = img[:, y * s:y * s + p, x * s:x * s + p]
    return out.reshape(b, oh * ow, p * p * C)


def _ln(x, g, b):
    mu = x.mean(-1, keepdims=True)
    return (x - mu) / np.sqrt(((x - mu) ** 2).mean(-1, keepdims=True) + LN_EPS) * g + b


def forward(img, w, cfg):
    """PiT.call in float64: img [b, H, W, 3] (any size with at most the table's patches) -> logits [b, num_classes]."""
    f = {k: np.asarray(v, np.float64) for k, v in w.items()}
    dh = cfg["dim_head"]
    x = patches(np.asarray(img, np.float64), cfg["patch_size"]) @ f["patch.kernel"] + f["patch.bias"]
    b, n, d = x.shape
    x = np.concatenate([np.broadcast_to(f["cls_token"], (b, 1, d)), x], 1) + f["pos_embedding"][:, :n + 1]
    n += 1
    for L, _, heads, po in layer_plan(cfg):
        p = f"layers.{L}."
        y = _ln(x, f[p + "attn_norm.gamma"], f[p + "attn_norm.beta"])
        q, k, v = (t.reshape(b, n, heads, dh).transpose(0, 2, 1, 3) for t in np.split(y @ f[p + "to_qkv.kernel"], 3, -1))
        s = q @ k.transpose(0, 1, 3, 2) * dh ** -0.5
        a = np.exp(s - s.max(-1, keepdims=True))
        o = ((a / a.sum(-1, keepdims=True)) @ v).transpose(0, 2, 1, 3).reshape(b, n, heads * dh)
        x = (o @ f[p + "to_out.kernel"] + f[p + "to_out.bias"] if po else o) + x
        y = _ln(x, f[p + "ff_norm.gamma"], f[p + "ff_norm.beta"]) @ f[p + "fc1.kernel"] + f[p + "fc1.bias"]
        x = (0.5 * y * (1.0 + erf(y / math.sqrt(2.0)))) @ f[p + "fc2.kernel"] + f[p + "fc2.bias"] + x
    z = _ln(x[:, 0], f["head_norm.gamma"], f["head_norm.beta"])
    return z @ f["head.kernel"] + f["head.bias"]


# ------------------------------------------------------------------------------------------------ the reference over the shim
def load_weights(model, w, cfg):
    """The oracle's weights into a reference PiT by attribute path (pit.py:179-205)."""
    model.patch_embedding.layers[1].set_weights([w["patch.kernel"], w["patch.bias"]])
    model.pos_embedding.assign(w["pos_embedding"])
    model.cls_token.assign(w["cls_token"])
    L = 0
    for tr in model.transformer_layers.layers:
        for attn, ff in tr.layers:
            p = f"layers.{L}."
            attn.norm.set_weights([w[p + "attn_norm.gamma"], w[p + "attn_norm.beta"]])
            attn.fn.to_qkv.set_weights([w[p + "to_qkv.kernel"]])
            if attn.fn.to_out.layers:
                attn.fn.to_out.layers[0].set_weights([w[p + "to_out.kernel"], w[p + "to_out.bias"]])
            else:
                assert p + "to_out.kernel" not in w
            ff.norm.set_weights([w[p + "ff_norm.gamma"], w[p + "ff_norm.beta"]])
            ff.fn.net.layers[0].set_weights([w[p + "fc1.kernel"], w[p + "fc1.bias"]])
            ff.fn.net.layers[3].set_weights([w[p + "fc2.kernel"], w[p + "fc2.bias"]])
            L += 1
    assert L == len(layer_plan(cfg))
    model.mlp_head.layers[0].set_weights([w["head_norm.gamma"], w["head_norm.beta"]])
    model.mlp_head.layers[1].set_weights([w["head.kernel"], w["head.bias"]])


@contextlib.contextmanager
def reference_module(reference_dir, dtype=np.float64):
    """The reference's unmodified pit module over the stand-in in `dtype`."""
    import importlib
    import sys
    from oracle import tf_shim
    saved = sys.modules.pop("pit", None)
    tf_shim.set_dtype(dtype)
    try:
        with tf_shim.installed(reference_dir):
            try:
                yield importlib.import_module("pit")
            finally:
                sys.modules.pop("pit", None)
    finally:
        tf_shim.set_dtype(np.float32)
        if saved is not None:
            sys.modules["pit"] = saved


def reference_logits(mod, cfg, w, img, dtype=np.float64):
    """Build the reference's PiT for `cfg`, call it once so that Keras builds every variable, load `w` and return
    `model(img, training=False)`."""
    model = mod.PiT(**ctor_kwargs(cfg))
    model(np.asarray(img, dtype), training=False)
    load_weights(model, {k: np.asarray(v, dtype) for k, v in w.items()}, cfg)
    return np.asarray(model(np.asarray(img, dtype), training=False)).view(np.ndarray).copy()


# ------------------------------------------------------------------------------------------------ cases
README = dict(image_size=224, patch_size=14, dim=256, num_classes=1000, depth=(3, 3, 3), heads=16, mlp_dim=2048)   # pit.py:222-232
# small cases (fixtures with float64 reference logits)
SMALL = {
    # even p: 32^2, p 8, stride 4 -> 7 x 7 = 49 patches; heads of 48 widened to 64; K = 192
    "pit_p8": dict(image_size=32, patch_size=8, num_classes=5, dim=64, depth=(1, 1), heads=2, dim_head=48, mlp_dim=128),
    # odd p with a non-exact tiling: 30^2, p 5, stride 2 -> 13 x 13 = 169 patches; dim_head 32 widened; K = 75 padded to 80
    "pit_p5_odd": dict(image_size=30, patch_size=5, num_classes=5, dim=64, depth=(2,), heads=4, dim_head=32, mlp_dim=128),
    # p 2, stride 1: 15 x 15 = 225 patches, n = 226 on the resident kernel; stage 0 has heads 1 and dim_head == dim: no to_out
    "pit_p2_stages": dict(image_size=16, patch_size=2, num_classes=5, dim=64, depth=(1, 1, 1), heads=(1, 2, 4), dim_head=64,
                          mlp_dim=128),
    # heads shorter than depth: zip keeps two stages of (1, 2) and (2, 4); heads of 16 widened; dim 48 (no LayerNorm folding)
    "pit_heads_short": dict(image_size=32, patch_size=4, num_classes=5, dim=48, depth=(1, 2, 3), heads=(2, 4), dim_head=16,
                            mlp_dim=96),
    # dim_head 80: the materialised-scores path; stage 1 has one head of 80 != dim, so it keeps to_out
    "pit_dh80": dict(image_size=24, patch_size=6, num_classes=5, dim=64, depth=(1, 1), heads=(2, 1), dim_head=80, mlp_dim=64),
    # 17 x 17 = 289 patches, n = 290: the streaming flash kernel
    "pit_stream": dict(image_size=36, patch_size=4, num_classes=5, dim=64, depth=(1, 1), heads=2, dim_head=64, mlp_dim=128),
    # dim_head 80 with heads (1, 4): inner 80 and 320, so in bf16 stage 0's LayerNorms are not folded into its GEMMs and stage 1's
    # are; stage 1 must fold with the row statistics of its own input, not of the embedding
    "pit_unfold_fold": dict(image_size=32, patch_size=8, num_classes=5, dim=64, depth=(1, 1), heads=(1, 4), dim_head=80, mlp_dim=64),
    # heads (4, 1, 4): folded, unfolded, folded
    "pit_fold_unfold_fold": dict(image_size=32, patch_size=8, num_classes=5, dim=64, depth=(1, 1, 1), heads=(4, 1, 4), dim_head=80,
                                 mlp_dim=64),
}
BENCH = {"pit_readme": README, "pit_readme_heads_4_8_16": dict(README, heads=(4, 8, 16))}
WEIGHTS = ("init_weights", "stress_weights")
WEIGHT_SEED, IMAGE_SEED, BATCH = 41, 42, 2


def fixture_name(name, gen):
    return f"{name}__{gen}__refshim.npz"

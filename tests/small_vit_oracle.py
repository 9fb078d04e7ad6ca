"""Float64 restatement of the small-dataset ViT (reference vit_for_small_dataset.py): shift (:15-47), SPT (:142-157), LSA (:88-121)
and ViT.call (:197-215), plus the reference's own module run over the numpy TensorFlow stand-in (oracle/tf_shim.py) with what
it needs beyond the other modules, and the weight sets of the fixtures."""
import contextlib
import sys

import numpy as np
from scipy.special import erf


def shift(x):
    """The four one-pixel shifts of NHWC images in the reference's order, zero fill: out[:, :, w] = x[:, :, w - 1],
    x[:, :, w + 1], then out[:, h] = x[:, h - 1], x[:, h + 1]."""
    out = [np.zeros_like(x) for _ in range(4)]
    out[0][:, :, 1:] = x[:, :, :-1]
    out[1][:, :, :-1] = x[:, :, 1:]
    out[2][:, 1:] = x[:, :-1]
    out[3][:, :-1] = x[:, 1:]
    return out


def spt_patches(img, p):
    """'b (h p1) (w p2) c -> b (h w) (p1 p2 c)' of [x, *shift(x)] concatenated on channels: [b, np, p^2 * 5 C]."""
    x = np.concatenate([img, *shift(img)], -1)
    b, H, W, c = x.shape
    return x.reshape(b, H // p, p, W // p, p, c).transpose(0, 1, 3, 2, 4, 5).reshape(b, (H // p) * (W // p), p * p * c)


def _ln(x, g, b, eps=1e-3):
    mu = x.mean(-1, keepdims=True)
    var = ((x - mu) ** 2).mean(-1, keepdims=True)
    return (x - mu) / np.sqrt(var + eps) * g + b


def lsa_scale(t):
    """exp(temperature), taken in float32 as TensorFlow does for the float32 Variable (:109)."""
    return float(np.exp(np.float32(t)))


def lsa(q, k, v, scale):
    """q, k, v [..., n, dh] -> softmax(q k^T * scale with the diagonal masked) v (:109-117)."""
    dots = q @ np.swapaxes(k, -1, -2) * scale
    n = dots.shape[-1]
    dots = np.where(np.eye(n, dtype=bool), -np.finfo(np.float64).max, dots)
    dots = dots - dots.max(-1, keepdims=True)
    a = np.exp(dots)
    return (a / a.sum(-1, keepdims=True)) @ v


def embed(w, img, p):
    """SPT + cls token + positions: [b, 1 + np, dim]."""
    f = lambda k: np.asarray(w[k], np.float64)
    x = _ln(spt_patches(np.asarray(img, np.float64), p), f("patch_norm.gamma"), f("patch_norm.beta")) @ f("patch.kernel") + f("patch.bias")
    b, n, d = x.shape
    x = np.concatenate([np.broadcast_to(f("cls_token"), (b, 1, d)), x], 1)
    return x + f("pos_embedding")[:, :n + 1]


def forward(w, img, cfg):
    """ViT.call in float64.  w: weight dict (the engine's names), img [b, H, W, 3], cfg: patch, heads, dim_head, depth, pool."""
    f = lambda k: np.asarray(w[k], np.float64)
    x = embed(w, img, cfg["patch"])
    b, n, _ = x.shape
    heads, dh = cfg["heads"], cfg["dim_head"]
    for L in range(cfg["depth"]):
        p = f"layers.{L}."
        y = _ln(x, f(p + "attn_norm.gamma"), f(p + "attn_norm.beta"))
        q, k, v = (t.reshape(b, n, heads, dh).transpose(0, 2, 1, 3) for t in np.split(y @ f(p + "to_qkv.kernel"), 3, -1))
        out = lsa(q, k, v, lsa_scale(w[p + "temperature"])).transpose(0, 2, 1, 3).reshape(b, n, heads * dh)
        x = out @ f(p + "to_out.kernel") + f(p + "to_out.bias") + x
        y = _ln(x, f(p + "ff_norm.gamma"), f(p + "ff_norm.beta"))
        h1 = y @ f(p + "fc1.kernel") + f(p + "fc1.bias")
        h1 = 0.5 * h1 * (1.0 + erf(h1 / np.sqrt(2.0)))
        x = h1 @ f(p + "fc2.kernel") + f(p + "fc2.bias") + x
    z = x.mean(1) if cfg["pool"] == "mean" else x[:, 0]
    z = _ln(z, f("head_norm.gamma"), f("head_norm.beta"))
    return z @ f("head.kernel") + f("head.bias")


def make_weights(cfg, kind, seed=0, num_classes=5):
    """kind 'init': Keras' initial values (glorot-uniform kernels, zero biases, LayerNorm ones / zeros, N(0, 1) positions and cls,
    temperature log(dim_head^-0.5)).  kind 'stress': every bias, beta and gamma random and nonzero, temperatures spread around
    their initial value, so that beta . W of SPT's cls row and the scale of every layer count."""
    rng = np.random.default_rng(seed)
    dim, heads, dh, mlp, p = cfg["dim"], cfg["heads"], cfg["dim_head"], cfg["mlp_dim"], cfg["patch"]
    H, W = cfg["image"]
    K, inner, n = p * p * 15, heads * dh, (H // p) * (W // p) + 1
    stress = kind == "stress"

    def dense(k, din, dout, bias=True):
        lim = np.sqrt(6.0 / (din + dout))
        w[k + ".kernel"] = rng.uniform(-lim, lim, (din, dout))
        if bias:
            w[k + ".bias"] = 0.2 * rng.standard_normal(dout) if stress else np.zeros(dout)

    def norm(k, d):
        w[k + ".gamma"] = 1 + 0.3 * rng.standard_normal(d) if stress else np.ones(d)
        w[k + ".beta"] = 0.3 * rng.standard_normal(d) if stress else np.zeros(d)

    w = {"pos_embedding": rng.standard_normal((1, n, dim)), "cls_token": rng.standard_normal((1, 1, dim))}
    norm("patch_norm", K)
    dense("patch", K, dim)
    for L in range(cfg["depth"]):
        pre = f"layers.{L}."
        norm(pre + "attn_norm", dim)
        dense(pre + "to_qkv", dim, 3 * inner, bias=False)
        dense(pre + "to_out", inner, dim)
        w[pre + "temperature"] = np.float32(np.log(np.float32(dh ** -0.5))) + (0.5 * rng.standard_normal() if stress else 0.0)
        norm(pre + "ff_norm", dim)
        dense(pre + "fc1", dim, mlp)
        dense(pre + "fc2", mlp, dim)
    norm("head_norm", dim)
    dense("head", dim, num_classes)
    return {k: np.asarray(v, np.float32) for k, v in w.items()}


# ------------------------------------------------------------------------------------------------ cases
SMALL = {
    # K = 240 padded to 256 in bf16; dh 64 native on the resident flash kernel
    "sq_p4_dh64": dict(image=(32, 32), patch=4, dim=64, depth=2, heads=2, dim_head=64, mlp_dim=128, pool="cls"),
    # rectangular, K = 960, dh 32 widened to 64, mean pool
    "rect_p8_dh32_mean": dict(image=(32, 48), patch=8, dim=64, depth=2, heads=4, dim_head=32, mlp_dim=64, pool="mean"),
    # dh 16 widened; dim 32: no LayerNorm folding anywhere in bf16
    "sq_p4_dh16": dict(image=(16, 16), patch=4, dim=32, depth=2, heads=2, dim_head=16, mlp_dim=64, pool="cls"),
    # dh 80: the materialised-scores path with the diagonal in its softmax
    "rect_p4_dh80_mean": dict(image=(16, 32), patch=4, dim=64, depth=2, heads=2, dim_head=80, mlp_dim=64, pool="mean"),
    # dh 48 widened, dim 96 (SPT unfolded in bf16), p = 8
    "sq_p8_dh48": dict(image=(32, 32), patch=8, dim=96, depth=2, heads=3, dim_head=48, mlp_dim=192, pool="cls"),
}
WEIGHTS = ("init", "stress")
BENCH = {
    # the reference README's model: 257 keys on the streaming flash kernel
    "readme": dict(image=(256, 256), patch=16, dim=1024, depth=6, heads=16, dim_head=64, mlp_dim=2048, pool="cls"),
    # a CIFAR-size model: 65 keys on the resident flash kernel
    "cifar": dict(image=(32, 32), patch=4, dim=192, depth=9, heads=12, dim_head=64, mlp_dim=384, pool="cls"),
}
BATCH = 2


def weights(cfg, kind="init", seed=0):
    return make_weights(cfg, kind, seed)


def images(cfg, b, seed=1):
    return np.random.default_rng(seed).standard_normal((b, *cfg["image"], 3)).astype(np.float32)


# ------------------------------------------------------------------------------------------------ the reference over the shim
@contextlib.contextmanager
def installed(reference_dir):
    """oracle/tf_shim.installed(reference_dir) plus what vit_for_small_dataset.py needs beyond the other modules: tf.roll, a bool
    tf.eye, tf.math.exp / log, and `.dtype.as_numpy_dtype` on tensors (:112).  `import vit_for_small_dataset` inside the block is
    the reference's own file, removed from sys.modules again on exit."""
    from oracle import tf_shim
    from ats_oracle import _DType
    saved = sys.modules.pop("vit_for_small_dataset", None)
    tensor = tf_shim.Tensor
    with tf_shim.installed(reference_dir) as tf:
        tf.roll = tf_shim._returns_tensor(lambda x, shift, axis, **_: np.roll(tf_shim._arr(x), shift, axis=axis))
        tf.eye = tf_shim._returns_tensor(lambda n, m=None, dtype=None, **_: np.eye(n, m, dtype=dtype or tf_shim.get_dtype()))
        tf.bool = np.bool_
        tf.math.exp = tf_shim._returns_tensor(lambda x, **_: np.exp(tf_shim._arr(x)))
        tf.math.log = tf_shim._returns_tensor(lambda x, **_: np.log(np.asarray(tf_shim._arr(x), tf_shim.get_dtype())))
        tensor.dtype = property(lambda self: _DType(np.ndarray.dtype.__get__(self)))
        try:
            yield tf
        finally:
            del tensor.dtype
            sys.modules.pop("vit_for_small_dataset", None)
            if saved is not None:
                sys.modules["vit_for_small_dataset"] = saved


def load_weights(model, w, dtype):
    """The oracle's weights into a reference vit_for_small_dataset.ViT by attribute path (:142-195)."""
    w = {k: np.asarray(v, dtype) for k, v in w.items()}
    tok = model.patch_embedding.to_patch_tokens.layers
    tok[1].set_weights([w["patch_norm.gamma"], w["patch_norm.beta"]])
    tok[2].set_weights([w["patch.kernel"], w["patch.bias"]])
    model.pos_embedding.assign(w["pos_embedding"])
    model.cls_token.assign(w["cls_token"])
    for L, (attn, ff) in enumerate(model.transformer.layers):
        p = f"layers.{L}."
        attn.norm.set_weights([w[p + "attn_norm.gamma"], w[p + "attn_norm.beta"]])
        attn.fn.to_qkv.set_weights([w[p + "to_qkv.kernel"]])
        attn.fn.to_out.layers[0].set_weights([w[p + "to_out.kernel"], w[p + "to_out.bias"]])
        attn.fn.temperature.assign(w[p + "temperature"])
        ff.norm.set_weights([w[p + "ff_norm.gamma"], w[p + "ff_norm.beta"]])
        ff.fn.net.layers[0].set_weights([w[p + "fc1.kernel"], w[p + "fc1.bias"]])
        ff.fn.net.layers[3].set_weights([w[p + "fc2.kernel"], w[p + "fc2.bias"]])
    model.mlp_head.layers[0].set_weights([w["head_norm.gamma"], w["head_norm.beta"]])
    model.mlp_head.layers[1].set_weights([w["head.kernel"], w["head.bias"]])


def reference_run(reference_dir, cases, dtype=np.float64):
    """{(name, kind): logits} of the reference's unmodified vit_for_small_dataset.ViT over the shim in `dtype`, called with
    training=False after one building call."""
    import importlib
    from oracle import tf_shim
    out = {}
    tf_shim.set_dtype(dtype)
    try:
        with installed(reference_dir):
            mod = importlib.import_module("vit_for_small_dataset")
            for name, cfg in cases.items():
                img = images(cfg, BATCH).astype(dtype)
                model = mod.ViT(image_size=cfg["image"], patch_size=cfg["patch"], num_classes=5, dim=cfg["dim"], depth=cfg["depth"],
                                heads=cfg["heads"], mlp_dim=cfg["mlp_dim"], pool=cfg["pool"], dim_head=cfg["dim_head"])
                model(img, training=False)
                for kind in WEIGHTS:
                    load_weights(model, weights(cfg, kind), dtype)
                    out[name, kind] = np.asarray(model(img, training=False)).view(np.ndarray).copy()
    finally:
        tf_shim.set_dtype(np.float32)
    return out

"""Float64 restatement of ATS-ViT's call (reference ats_vit.py:191-318) with the engine's defined noise (include/vitb200.h):
u = (word 0 of Philox4x32-10 >> 8) * 2^-24, key = the 64-bit seed, counter (j | k << 16, b, d_lo, d_hi), d counting the
sampling events since the seed was set.  The reference's own left-padded layout is restated as it is (masks, pads, gathers), so
the engine's compact layout is checked against it rather than against a copy of itself."""
import contextlib
import sys
import types

import numpy as np
from scipy.special import erf

M0, M1, W0, W1 = 0xD2511F53, 0xCD9E8D57, 0x9E3779B9, 0xBB67AE85
MASK32 = np.uint64(0xFFFFFFFF)


def philox4x32_10(ctr, key):
    """ctr: uint32-valued array [..., 4], key: (k0, k1) -> uint32 array [..., 4] (Random123's philox4x32 with 10 rounds)."""
    c = [np.asarray(ctr[..., i], np.uint64) for i in range(4)]
    k0, k1 = np.uint64(key[0]), np.uint64(key[1])
    for _ in range(10):
        p0 = np.uint64(M0) * c[0]
        p1 = np.uint64(M1) * c[2]
        hi0, lo0 = p0 >> np.uint64(32), p0 & MASK32
        hi1, lo1 = p1 >> np.uint64(32), p1 & MASK32
        c = [(hi1 ^ c[1] ^ k0) & MASK32, lo1, (hi0 ^ c[3] ^ k1) & MASK32, lo0]
        k0 = (k0 + np.uint64(W0)) & MASK32
        k1 = (k1 + np.uint64(W1)) & MASK32
    return np.stack(c, -1).astype(np.uint32)


def uniform(shape, seed, d):
    """The noise of one sampling event: u [b, K, n - 1] in [0, 1)."""
    b, K, n1 = shape
    bb, kk, jj = np.meshgrid(np.arange(b), np.arange(K), np.arange(n1), indexing="ij")
    ctr = np.stack([(jj | (kk << 16)).astype(np.uint64), bb.astype(np.uint64), np.full(bb.shape, d & 0xFFFFFFFF, np.uint64),
                    np.full(bb.shape, d >> 32, np.uint64)], -1)
    x = philox4x32_10(ctr, (seed & 0xFFFFFFFF, seed >> 32))[..., 0]
    return (x >> 8).astype(np.float64) * 2.0 ** -24


def _ln(x, g, b, eps=1e-3):
    mu = x.mean(-1, keepdims=True)
    var = ((x - mu) ** 2).mean(-1, keepdims=True)
    return (x - mu) / np.sqrt(var + eps) * g + b


def bf16_round(x):
    """Round to the nearest bfloat16 (ties to even), returned in float64."""
    a = np.asarray(x, np.float32)
    u = a.view(np.uint32).astype(np.uint64)
    u = ((u + 0x7FFF + ((u >> 16) & 1)) >> 16) << 16
    return u.astype(np.uint32).view(np.float32).astype(np.float64)


def forward(w, img, cfg, seed=0, d=0, forced=None, bf16_storage=False):
    """ATS ViT.call in float64.  w: weight dict (ViT names), img [b, H, W, 3], cfg: heads, dim_head, depth, max_tokens_per_depth,
    patch (ph, pw).  forced: {layer: draws [b, K]} (argmax + 1 positions) replacing that layer's Gumbel-max choices.
    bf16_storage: what the bf16 engine stores rounded to bfloat16 (every Dense's operands and result, q|k|v, the attention output,
    the residual stream after every sub-block), everything else in float64: a lower estimate of what bf16 storage alone costs.
    Returns dict(logits, token_ids (the reference's returned layout), sampled (layers that sampled), draws {layer: [b, K]},
    margin (smallest top-2 gap of a Gumbel-max draw), pert {layer: the perturbed pseudo-logits [b, K, n - 1]}, d (the counter
    after the call))."""
    f = lambda k: np.asarray(w[k], np.float64)
    st = bf16_round if bf16_storage else (lambda a: a)
    mm = (lambda a, k: bf16_round(bf16_round(a) @ bf16_round(k))) if bf16_storage else (lambda a, k: a @ k)
    x0 = np.asarray(img, np.float64)
    b, H, W, c = x0.shape
    ph, pw = cfg["patch"]
    x = x0.reshape(b, H // ph, ph, W // pw, pw, c).transpose(0, 1, 3, 2, 4, 5).reshape(b, (H // ph) * (W // pw), ph * pw * c)
    x = mm(x, f("patch.kernel")) + f("patch.bias")
    n = x.shape[1] + 1
    x = st(np.concatenate([np.broadcast_to(f("cls_token"), (b, 1, x.shape[2])), x], 1) + f("pos_embedding")[:, :n])
    heads, dh = cfg["heads"], cfg["dim_head"]
    mask = np.ones((b, n), bool)
    token_ids = np.broadcast_to(np.arange(n), (b, n)).copy()
    sampled, draws_out, pert_out, margin = [], {}, {}, np.inf
    for L, K in enumerate(cfg["max_tokens_per_depth"]):
        p = f"layers.{L}."
        n = x.shape[1]
        y = _ln(x, f(p + "attn_norm.gamma"), f(p + "attn_norm.beta"))
        qkv = mm(y, f(p + "to_qkv.kernel"))
        q, k, v = (st(t).reshape(b, n, heads, dh).transpose(0, 2, 1, 3) for t in np.split(qkv, 3, -1))
        dots = q @ k.transpose(0, 1, 3, 2) * dh ** -0.5
        dm = mask[:, None, :, None] & mask[:, None, None, :]
        dots = np.where(dm, dots, -np.finfo(np.float64).max)
        dots = dots - dots.max(-1, keepdims=True)
        attn = np.exp(dots)
        attn /= attn.sum(-1, keepdims=True)
        ids = None
        if n - 1 > K:                                                # ats_vit.py:213
            sampled.append(L)
            cls_attn = np.einsum("bhn,bhn->bn", attn[:, :, 0, 1:], np.linalg.norm(v[:, :, 1:], axis=-1))
            logits = np.log(cls_attn / (cls_attn.sum(-1, keepdims=True) + 1e-6) + 1e-6)
            logits = np.where(mask[:, 1:], logits, -np.finfo(np.float64).max / 2)
            u = uniform((b, K, n - 1), seed, d)
            d += 1
            pert = logits[:, None, :] + (-np.log(-np.log(u + 1e-6) + 1e-6))
            pert_out[L] = pert
            choice = pert.argmax(-1) + 1
            top2 = np.sort(pert, -1)[..., -2:]
            margin = min(margin, float((top2[..., 1] - top2[..., 0]).min()))
            if forced is not None and L in forced:
                choice = np.asarray(forced[L])
            draws_out[L] = choice
            kept = [np.unique(r) for r in choice]
            m = max(len(r) for r in kept)
            ids = np.zeros((b, m + 1), np.int64)
            for i, r in enumerate(kept):
                ids[i, 1 + m - len(r):] = r                          # pad_sequences: padding='pre'
            mask = ids != 0
            mask[:, 0] = True
            attn = np.take_along_axis(attn, ids[:, None, :, None], 2)
        out = st((attn @ v).transpose(0, 2, 1, 3).reshape(b, -1, heads * dh))
        out = mm(out, f(p + "to_out.kernel")) + f(p + "to_out.bias")
        if ids is not None:
            x = np.take_along_axis(x, ids[:, :, None], 1)
            token_ids = np.take_along_axis(token_ids, ids, 1)
        x = st(x + out)
        y = _ln(x, f(p + "ff_norm.gamma"), f(p + "ff_norm.beta"))
        h1 = mm(y, f(p + "fc1.kernel")) + f(p + "fc1.bias")
        h1 = 0.5 * h1 * (1.0 + erf(h1 / np.sqrt(2.0)))
        x = st(x + mm(h1, f(p + "fc2.kernel")) + f(p + "fc2.bias"))
    z = _ln(x[:, 0], f("head_norm.gamma"), f("head_norm.beta"))
    return dict(logits=z @ f("head.kernel") + f("head.bias"), token_ids=token_ids[:, 1:] - 1, sampled=sampled, draws=draws_out,
                pert=pert_out, margin=margin, d=d)


def small_weights(cfg, rng, num_classes=5):
    """Random float32 weights of an ATS-ViT config (ViT names), scaled so that activations stay O(1)."""
    dim, heads, dh, mlp = cfg["dim"], cfg["heads"], cfg["dim_head"], cfg["mlp_dim"]
    ph, pw = cfg["patch"]
    n = (cfg["image"][0] // ph) * (cfg["image"][1] // pw) + 1
    w = {"patch.kernel": rng.standard_normal((ph * pw * 3, dim)) * 0.2, "patch.bias": rng.standard_normal(dim) * 0.1,
         "pos_embedding": rng.standard_normal((1, n, dim)), "cls_token": rng.standard_normal((1, 1, dim)),
         "head_norm.gamma": 1 + 0.1 * rng.standard_normal(dim), "head_norm.beta": 0.1 * rng.standard_normal(dim),
         "head.kernel": rng.standard_normal((dim, num_classes)) * 0.2, "head.bias": rng.standard_normal(num_classes) * 0.1}
    for L in range(len(cfg["max_tokens_per_depth"])):
        p = f"layers.{L}."
        for nm in ("attn_norm", "ff_norm"):
            w[p + nm + ".gamma"] = 1 + 0.1 * rng.standard_normal(dim)
            w[p + nm + ".beta"] = 0.1 * rng.standard_normal(dim)
        w[p + "to_qkv.kernel"] = rng.standard_normal((dim, 3 * heads * dh)) * dim ** -0.5
        w[p + "to_out.kernel"] = rng.standard_normal((heads * dh, dim)) * (heads * dh) ** -0.5
        w[p + "to_out.bias"] = 0.1 * rng.standard_normal(dim)
        w[p + "fc1.kernel"] = rng.standard_normal((dim, mlp)) * dim ** -0.5
        w[p + "fc1.bias"] = 0.1 * rng.standard_normal(mlp)
        w[p + "fc2.kernel"] = rng.standard_normal((mlp, dim)) * mlp ** -0.5
        w[p + "fc2.bias"] = 0.1 * rng.standard_normal(dim)
    return {k: np.asarray(v, np.float32) for k, v in w.items()}


# ------------------------------------------------------------------------------------------------ cases
SMALL = {
    # dh 16 / 32 / 48 widened to 64 in bf16, 64 native, 80 on the materialised-scores path; rectangular; K above n - 1 first
    "dh16_rect": dict(image=(16, 24), patch=(4, 4), dim=64, heads=2, dim_head=16, mlp_dim=64, max_tokens_per_depth=(30, 12, 12, 5)),
    "dh32": dict(image=(32, 32), patch=(4, 4), dim=64, heads=2, dim_head=32, mlp_dim=128, max_tokens_per_depth=(40, 20, 9)),
    "dh48": dict(image=(32, 32), patch=(4, 4), dim=64, heads=3, dim_head=48, mlp_dim=64, max_tokens_per_depth=(63, 33, 20)),
    "dh64": dict(image=(48, 48), patch=(4, 4), dim=128, heads=2, dim_head=64, mlp_dim=128, max_tokens_per_depth=(200, 70, 17)),
    # layer 1 can sample (pitch 51 > 46) but the batch keeps at most 35 tokens after layer 0: skipped on the device
    "dh80": dict(image=(32, 32), patch=(4, 4), dim=64, heads=2, dim_head=80, mlp_dim=64, max_tokens_per_depth=(50, 45), wseed=1),
}
BENCH = {
    "readme": dict(image=(256, 256), patch=(16, 16), dim=1024, heads=16, dim_head=64, mlp_dim=2048,
                   max_tokens_per_depth=(256, 128, 64, 32, 16, 8)),
    "p16_384": dict(image=(384, 384), patch=(16, 16), dim=384, heads=6, dim_head=64, mlp_dim=768, max_tokens_per_depth=(400, 300, 100)),
}
BATCH, SEED = 3, 0


def weights(cfg, seed=0):
    return small_weights(cfg, np.random.default_rng(cfg.get("wseed", seed)))


def images(cfg, b, seed=1, size=None):
    h, w = size or cfg["image"]
    return np.random.default_rng(seed).standard_normal((b, h, w, 3)).astype(np.float32)


# ------------------------------------------------------------------------------------------------ the reference over the shim
class _DType:
    """What `.dtype` of a shim tensor returns inside installed(): the numpy dtype (np.dtype() and np.finfo accept the object
    through its `dtype` attribute) plus TensorFlow's `.as_numpy_dtype` (ats_vit.py:97, 204)."""

    def __init__(self, dt):
        self.dtype = np.dtype(dt)
        self.as_numpy_dtype = self.dtype.type

    def __getattr__(self, name):
        return getattr(self.dtype, name)

    def __eq__(self, other):
        return self.dtype == np.dtype(getattr(other, "dtype", other))

    def __hash__(self):
        return hash(self.dtype)


class _Shape(tuple):
    """TensorShape's num_elements() on a tuple (ats_vit.py:40)."""

    def num_elements(self):
        return int(np.prod(self))


@contextlib.contextmanager
def installed(reference_dir, seed=0):
    """oracle/tf_shim.installed(reference_dir) plus what ats_vit.py needs beyond the other modules: tf.unique / sort / unstack /
    norm / tile / pad / gather_nd / stack / ones / math.log, one-argument tf.where, keras' pad_sequences (int32, value 0, padding 'pre'),
    `.dtype.as_numpy_dtype` and `.shape.num_elements()` on tensors, and tf.random.uniform returning the engine's Philox noise for
    the call's shape with the draw counter counting the calls (yielded as `state['d']`).  `import ats_vit` inside the block is the
    reference's own file, removed from sys.modules again on exit."""
    from oracle import tf_shim
    saved = sys.modules.pop("ats_vit", None)
    state = {"d": 0}

    def uniform(shape, *_, **__):
        state.setdefault("shapes", []).append(tuple(int(s) for s in shape))
        u = globals()["uniform"](tuple(int(s) for s in shape), seed, state["d"])
        state["d"] += 1
        return u.astype(tf_shim.get_dtype())

    def unique(x, *_, **__):
        a = np.asarray(x)
        vals, first, inv = np.unique(a, return_index=True, return_inverse=True)
        order = np.argsort(first)                                    # tf.unique keeps the order of first occurrence
        rank = np.empty_like(order)
        rank[order] = np.arange(len(order))
        return a[np.sort(first)], rank[inv].astype(np.int32)

    def where(condition, x=None, y=None, **_):
        if x is None and y is None:
            return np.argwhere(np.asarray(condition)).astype(np.int64)
        return np.where(tf_shim._arr(condition), tf_shim._arr(x), tf_shim._arr(y))

    def pad_sequences(sequences, maxlen=None, dtype="int32", padding="pre", truncating="pre", value=0.0):
        seqs = [np.asarray(s) for s in sequences]
        m = maxlen or max(len(s) for s in seqs)
        out = np.full((len(seqs), m), value, dtype=dtype)
        for i, s in enumerate(seqs):
            s = s[-m:] if truncating == "pre" else s[:m]
            if padding == "pre":
                out[i, m - len(s):] = s
            else:
                out[i, :len(s)] = s
        return out

    extra = dict(
        unique=unique, sort=lambda x, axis=-1, **_: np.sort(np.asarray(x), axis=axis), unstack=lambda x, axis=0, **_: list(np.moveaxis(np.asarray(x), axis, 0)),
        norm=lambda x, ord="euclidean", axis=None, **_: np.linalg.norm(tf_shim._arr(x), axis=axis),
        tile=lambda x, multiples, **_: np.tile(np.asarray(x), tuple(multiples)),
        pad=lambda t, paddings, mode="CONSTANT", constant_values=0, **_: np.pad(np.asarray(t), np.asarray(paddings), constant_values=constant_values),
        gather_nd=lambda params, indices, **_: np.asarray(params)[tuple(np.moveaxis(np.asarray(indices), -1, 0))],
        stack=lambda values, axis=0, **_: np.stack([np.asarray(v) for v in values], axis=axis),
        ones=lambda shape, dtype=None, **_: np.ones(tuple(shape), dtype=dtype or tf_shim.get_dtype()), where=where)
    tensor = tf_shim.Tensor
    with tf_shim.installed(reference_dir) as tf:
        for k, f in extra.items():
            setattr(tf, k, tf_shim._returns_tensor(f))
        tf.math.log = tf_shim._returns_tensor(lambda x, **_: np.log(tf_shim._arr(x)))
        tf.random.uniform = tf_shim._returns_tensor(uniform)
        seq = types.ModuleType("tensorflow.keras.preprocessing.sequence")
        seq.pad_sequences = pad_sequences
        pre = types.ModuleType("tensorflow.keras.preprocessing")
        pre.__path__, pre.sequence = [], seq
        tf.keras.preprocessing = pre
        mods = {"tensorflow.keras.preprocessing": pre, "tensorflow.keras.preprocessing.sequence": seq}
        sys.modules.update(mods)
        tensor.dtype = property(lambda self: _DType(np.ndarray.dtype.__get__(self)))
        tensor.shape = property(lambda self: _Shape(np.ndarray.shape.__get__(self)), lambda self, v: np.ndarray.shape.__set__(self, v))
        try:
            yield state
        finally:
            del tensor.dtype, tensor.shape
            for n in mods:
                sys.modules.pop(n, None)
            sys.modules.pop("ats_vit", None)
            if saved is not None:
                sys.modules["ats_vit"] = saved


def load_weights(model, w, dtype):
    """The oracle's weights into a reference ats_vit.ViT by attribute path (ats_vit.py:283-297)."""
    w = {k: np.asarray(v, dtype) for k, v in w.items()}
    model.patch_embedding.layers[1].set_weights([w["patch.kernel"], w["patch.bias"]])
    model.pos_embedding.assign(w["pos_embedding"])
    model.cls_token.assign(w["cls_token"])
    for L, (attn, ff) in enumerate(model.transformer.layers):
        p = f"layers.{L}."
        attn.norm.set_weights([w[p + "attn_norm.gamma"], w[p + "attn_norm.beta"]])
        attn.fn.to_qkv.set_weights([w[p + "to_qkv.kernel"]])
        attn.fn.to_out.layers[0].set_weights([w[p + "to_out.kernel"], w[p + "to_out.bias"]])
        ff.norm.set_weights([w[p + "ff_norm.gamma"], w[p + "ff_norm.beta"]])
        ff.fn.net.layers[0].set_weights([w[p + "fc1.kernel"], w[p + "fc1.bias"]])
        ff.fn.net.layers[3].set_weights([w[p + "fc2.kernel"], w[p + "fc2.bias"]])
    model.mlp_head.layers[0].set_weights([w["head_norm.gamma"], w["head_norm.beta"]])
    model.mlp_head.layers[1].set_weights([w["head.kernel"], w["head.bias"]])


def reference_run(reference_dir, cases, dtype=np.float64, seed=SEED):
    """{name: dict(logits, token_ids, noise_shapes)} of the reference's unmodified ats_vit.ViT over the shim in `dtype`, each called
    with the draw counter at 0 after one building call; noise_shapes: the [b, K, n - 1] of every tf.random.uniform call (one per
    layer that sampled).  Importing the module runs its usage block (a 4 x 256^2 forward)."""
    import importlib
    from oracle import tf_shim
    out = {}
    tf_shim.set_dtype(dtype)
    try:
        with installed(reference_dir, seed) as state:
            mod = importlib.import_module("ats_vit")
            for name, cfg in cases.items():
                img = images(cfg, BATCH).astype(dtype)
                model = mod.ViT(image_size=cfg["image"], patch_size=cfg["patch"], num_classes=5, dim=cfg["dim"],
                                depth=len(cfg["max_tokens_per_depth"]), max_tokens_per_depth=cfg["max_tokens_per_depth"],
                                heads=cfg["heads"], mlp_dim=cfg["mlp_dim"], dim_head=cfg["dim_head"])
                model(img)
                load_weights(model, weights(cfg), dtype)
                state["d"], state["shapes"] = 0, []
                logits, ids = model(img, True)
                out[name] = dict(logits=np.asarray(logits).view(np.ndarray).copy(), token_ids=np.asarray(ids).view(np.ndarray).copy(),
                                 noise_shapes=np.asarray(state["shapes"], np.int64).reshape(-1, 3))
    finally:
        tf_shim.set_dtype(np.float32)
    return out

"""Float64 restatement of MAE.call (reference mae.py:49-92) and SimMIM.call (simmim.py:82-129) with the engine's defined mask noise
(include/vitb200.h): u[b, j] = (word 0 of Philox4x32-10 >> 8) * 2^-24, key = the 64-bit seed, counter (j, b, d_lo, d_hi), d counting
the calls since the seed was set.  MAE's masks are the stable argsort of u (ascending, ties to the smaller id), SimMIM's the stable
top_k (descending, ties to the smaller id); the first int(masking_ratio * n) ids are masked.

Also here: the cases of the fixtures (tests/golden/make_mim_golden.py), their weights, and the reference run over the numpy stand-in
for TensorFlow with tf.random.uniform returning that noise."""
import contextlib
import importlib

import numpy as np
from scipy.special import erf

from ats_oracle import _ln, bf16_round, philox4x32_10


def noise(b, n, seed=0, d=0):
    """u [b, n] in [0, 1): one MAE / SimMIM call's mask noise at draw counter d."""
    bb, jj = np.meshgrid(np.arange(b), np.arange(n), indexing="ij")
    ctr = np.stack([jj.astype(np.uint64), bb.astype(np.uint64), np.full(bb.shape, d & 0xFFFFFFFF, np.uint64),
                    np.full(bb.shape, d >> 32, np.uint64)], -1)
    x = philox4x32_10(ctr, (seed & 0xFFFFFFFF, seed >> 32))[..., 0]
    return (x >> 8).astype(np.float64) * 2.0 ** -24


def permutation(u, simmim):
    """Each image's ids, the masked ones first: argsort of u (MAE) or of -u (SimMIM's top_k), ties to the smaller id."""
    return np.argsort(-u if simmim else u, axis=-1, kind="stable").astype(np.int32)


def mask_indices(kind, b, n, seed=0, d=0):
    return permutation(noise(b, n, seed, d), kind == "simmim")


def has_tie(u):
    """Whether some image's noise holds two equal values."""
    s = np.sort(u, -1)
    return bool((np.diff(s, axis=-1) == 0).any())


def num_masked(ratio, n):
    return int(ratio * n)                                            # mae.py:57, simmim.py:106: Python's int() of a double


def to_patches(img, ph, pw):
    """'b (h p1) (w p2) c -> b (h w) (p1 p2 c)' (vit.py:142)."""
    b, H, W, c = img.shape
    return img.reshape(b, H // ph, ph, W // pw, pw, c).transpose(0, 1, 3, 2, 4, 5).reshape(b, (H // ph) * (W // pw), ph * pw * c)


def _transformer(x, w, prefix, depth, heads, dh, st, mm):
    """vit.Transformer.call (vit.py:95-104): pre-norm attention (to_out when its weights exist) and MLP, no final norm."""
    f = lambda k: np.asarray(w[k], np.float64)
    b, n, _ = x.shape
    for L in range(depth):
        p = f"{prefix}{L}."
        y = _ln(x, f(p + "attn_norm.gamma"), f(p + "attn_norm.beta"))
        qkv = mm(y, f(p + "to_qkv.kernel"))
        q, k, v = (st(t).reshape(b, n, heads, dh).transpose(0, 2, 1, 3) for t in np.split(qkv, 3, -1))
        dots = q @ k.transpose(0, 1, 3, 2) * dh ** -0.5
        dots = dots - dots.max(-1, keepdims=True)
        attn = np.exp(dots)
        attn /= attn.sum(-1, keepdims=True)
        out = st((attn @ v).transpose(0, 2, 1, 3).reshape(b, n, heads * dh))
        if p + "to_out.kernel" in w:
            out = mm(out, f(p + "to_out.kernel")) + f(p + "to_out.bias")
        x = st(x + out)
        y = _ln(x, f(p + "ff_norm.gamma"), f(p + "ff_norm.beta"))
        h1 = mm(y, f(p + "fc1.kernel")) + f(p + "fc1.bias")
        h1 = 0.5 * h1 * (1.0 + erf(h1 / np.sqrt(2.0)))
        x = st(x + mm(h1, f(p + "fc2.kernel")) + f(p + "fc2.bias"))
    return x


def forward(kind, w, img, cfg, seed=0, d=0, bf16_storage=False):
    """MAE / SimMIM call in float64.  kind: "mae" or "simmim"; w: the weight dict (include/vitb200.h names), img [b, H, W, 3];
    cfg: patch (ph, pw), dim, depth, heads, dim_head, ratio and (MAE) decoder_dim, decoder_depth, decoder_heads, decoder_dim_head.
    bf16_storage: what the bf16 engine stores rounded to bfloat16 (every Dense's operands and result, the position rows, q|k|v,
    the attention output, the residual stream after every sub-block, the decoder input, pred), everything else in float64: a lower
    estimate of what bf16 storage alone costs.  Returns dict(loss, pred [b, nm, pd], masked_patches, indices [b, n], u)."""
    f = lambda k: np.asarray(w[k], np.float64)
    st = bf16_round if bf16_storage else (lambda a: a)
    mm = (lambda a, k: bf16_round(bf16_round(a) @ bf16_round(k))) if bf16_storage else (lambda a, k: a @ k)
    x0 = np.asarray(img, np.float64)
    b = x0.shape[0]
    ph, pw = cfg["patch"]
    patches = to_patches(x0, ph, pw)
    n = patches.shape[1]
    nm = num_masked(cfg["ratio"], n)
    u = noise(b, n, seed, d)
    perm = permutation(u, kind == "simmim")
    take = lambda a, ids: np.take_along_axis(a, ids[..., None].astype(np.int64), 1)
    pos = f("pos_embedding")[0, 1:n + 1]
    masked_patches = take(patches, perm[:, :nm])
    if kind == "mae":
        kept = perm[:, nm:]
        x = st(mm(take(patches, kept), f("patch.kernel")) + f("patch.bias") + st(pos[kept]))   # embed-then-gather, per row
        x = _transformer(x, w, "layers.", cfg["depth"], cfg["heads"], cfg["dim_head"], st, mm)
        if "enc_to_dec.kernel" in w:
            x = st(mm(x, f("enc_to_dec.kernel")) + f("enc_to_dec.bias"))
        dpe = f("decoder_pos_emb.embeddings")
        z = st(np.concatenate([f("mask_token") + dpe[perm[:, :nm]], x + dpe[kept]], 1))
        z = _transformer(z, w, "decoder.layers.", cfg["decoder_depth"], cfg["decoder_heads"], cfg["decoder_dim_head"], st, mm)
        pred = st(mm(z[:, :nm], f("to_pixels.kernel")) + f("to_pixels.bias"))
        loss = np.mean(pred ** 2)                                    # mae.py:90: tf.square(pred, masked_patches) squares pred
    else:
        x = st(mm(patches, f("patch.kernel")) + f("patch.bias") + st(pos))
        m = np.zeros((b, n), bool)
        np.put_along_axis(m, perm[:, :nm].astype(np.int64), True, 1)
        x = np.where(m[..., None], st(f("mask_token") + pos), x)
        x = _transformer(x, w, "layers.", cfg["depth"], cfg["heads"], cfg["dim_head"], st, mm)
        pred = st(mm(take(x, perm[:, :nm]), f("to_pixels.kernel")) + f("to_pixels.bias"))
        loss = np.mean(np.abs(pred - masked_patches)) / nm           # simmim.py:128
    return dict(loss=float(loss), pred=pred, masked_patches=masked_patches, indices=perm, u=u, num_masked=nm)


# ------------------------------------------------------------------------------------------------ cases and weights
def _layer_weights(rng, pre, dim, heads, dh, mlp, stress):
    s = 1.0 if stress else 0.0
    inner = heads * dh
    w = {pre + "attn_norm.gamma": 1 + s * 0.1 * rng.standard_normal(dim), pre + "attn_norm.beta": s * 0.1 * rng.standard_normal(dim),
         pre + "to_qkv.kernel": rng.standard_normal((dim, 3 * inner)) * dim ** -0.5,
         pre + "ff_norm.gamma": 1 + s * 0.1 * rng.standard_normal(dim), pre + "ff_norm.beta": s * 0.1 * rng.standard_normal(dim),
         pre + "fc1.kernel": rng.standard_normal((dim, mlp)) * dim ** -0.5, pre + "fc1.bias": s * 0.1 * rng.standard_normal(mlp),
         pre + "fc2.kernel": rng.standard_normal((mlp, dim)) * mlp ** -0.5, pre + "fc2.bias": s * 0.1 * rng.standard_normal(dim)}
    if not (heads == 1 and dh == dim):                               # vit.py:53
        w[pre + "to_out.kernel"] = rng.standard_normal((inner, dim)) * inner ** -0.5
        w[pre + "to_out.bias"] = s * 0.1 * rng.standard_normal(dim)
    return w


def weights(kind, cfg, variant="init", seed=0):
    """The engine's weights of a case: 'init' (Keras-like scale: zero biases, unit LayerNorms, N(0, 1) mask token, uniform(-0.05,
    0.05) decoder positions) or 'stress' (non-trivial biases, LayerNorms and larger positions)."""
    rng = np.random.default_rng(seed + (0 if variant == "init" else 1000))
    stress = variant == "stress"
    ph, pw = cfg["patch"]
    H, W = cfg["image"]
    dim, pd = cfg["dim"], ph * pw * 3
    npos = (H // ph) * (W // pw) + 1
    w = {"pos_embedding": rng.standard_normal((1, npos, dim)) * (1.0 if stress else 0.5),
         "patch.kernel": rng.standard_normal((pd, dim)) * pd ** -0.5, "patch.bias": (0.1 if stress else 0.0) * rng.standard_normal(dim)}
    for L in range(cfg["depth"]):
        w.update(_layer_weights(rng, f"layers.{L}.", dim, cfg["heads"], cfg["dim_head"], cfg["mlp_dim"], stress))
    Dd = cfg["decoder_dim"] if kind == "mae" else dim
    w["mask_token"] = rng.standard_normal(Dd)
    if kind == "mae":
        if dim != Dd:
            w["enc_to_dec.kernel"] = rng.standard_normal((dim, Dd)) * dim ** -0.5
            w["enc_to_dec.bias"] = (0.1 if stress else 0.0) * rng.standard_normal(Dd)
        for L in range(cfg["decoder_depth"]):
            w.update(_layer_weights(rng, f"decoder.layers.{L}.", Dd, cfg["decoder_heads"], cfg["decoder_dim_head"], 4 * Dd, stress))
        w["decoder_pos_emb.embeddings"] = rng.uniform(-0.05, 0.05, (npos, Dd)) * (10.0 if stress else 1.0)
    w["to_pixels.kernel"] = rng.standard_normal((Dd, pd)) * Dd ** -0.5
    w["to_pixels.bias"] = (0.1 if stress else 0.0) * rng.standard_normal(pd)
    return {k: np.asarray(v, np.float32) for k, v in w.items()}


def images(cfg, b, seed=1, size=None):
    h, w = size or cfg["image"]
    return np.random.default_rng(seed).standard_normal((b, h, w, 3)).astype(np.float32)


BATCH, SEED = 2, 0
# (kind, cfg): image / patch sizes, the encoder ViT and the MIM arguments; call: the image size of the call when it is not `image`
CASES = {
    "mae_dense": ("mae", dict(image=(32, 32), patch=(8, 8), dim=64, depth=2, heads=2, dim_head=32, mlp_dim=128, ratio=0.75,
                              decoder_dim=48, decoder_depth=1, decoder_heads=3, decoder_dim_head=16)),
    "mae_identity": ("mae", dict(image=(32, 32), patch=(4, 4), dim=64, depth=1, heads=2, dim_head=32, mlp_dim=64, ratio=0.6,
                                 decoder_dim=64, decoder_depth=2, decoder_heads=4, decoder_dim_head=16)),
    "mae_no_to_out": ("mae", dict(image=(24, 24), patch=(4, 4), dim=40, depth=1, heads=2, dim_head=20, mlp_dim=80, ratio=0.5,
                                  decoder_dim=24, decoder_depth=2, decoder_heads=1, decoder_dim_head=24)),
    "mae_rect": ("mae", dict(image=(24, 40), patch=(4, 8), dim=72, depth=1, heads=3, dim_head=24, mlp_dim=96, ratio=0.75,
                             decoder_dim=36, decoder_depth=1, decoder_heads=2, decoder_dim_head=18)),
    "mae_small_image": ("mae", dict(image=(32, 32), patch=(4, 4), dim=64, depth=1, heads=2, dim_head=32, mlp_dim=64, ratio=0.75,
                                    decoder_dim=32, decoder_depth=1, decoder_heads=2, decoder_dim_head=16, call=(16, 24))),
    "mae_ratio29": ("mae", dict(image=(40, 40), patch=(4, 4), dim=64, depth=1, heads=2, dim_head=32, mlp_dim=64, ratio=0.29,
                                decoder_dim=32, decoder_depth=1, decoder_heads=2, decoder_dim_head=16)),
    "simmim_base": ("simmim", dict(image=(32, 32), patch=(8, 8), dim=64, depth=2, heads=2, dim_head=32, mlp_dim=128, ratio=0.5)),
    "simmim_odd": ("simmim", dict(image=(24, 24), patch=(4, 4), dim=40, depth=1, heads=2, dim_head=20, mlp_dim=80, ratio=0.3)),
    "simmim_rect": ("simmim", dict(image=(24, 40), patch=(8, 4), dim=72, depth=1, heads=3, dim_head=24, mlp_dim=96, ratio=0.5)),
    "simmim_small_image": ("simmim", dict(image=(32, 32), patch=(4, 4), dim=64, depth=1, heads=2, dim_head=32, mlp_dim=64, ratio=0.5,
                                          call=(24, 16))),
    "simmim_ratio29": ("simmim", dict(image=(40, 40), patch=(4, 4), dim=64, depth=1, heads=2, dim_head=32, mlp_dim=64, ratio=0.29)),
    # README configurations (README.md:685-735: encoder ViT 256^2 / 32, dim 1024, depth 6, heads 8, mlp 2048) at batch 2
    "mae_readme": ("mae", dict(image=(256, 256), patch=(32, 32), dim=1024, depth=6, heads=8, dim_head=64, mlp_dim=2048, ratio=0.75,
                               decoder_dim=512, decoder_depth=6, decoder_heads=8, decoder_dim_head=64)),
    "simmim_readme": ("simmim", dict(image=(256, 256), patch=(32, 32), dim=1024, depth=6, heads=8, dim_head=64, mlp_dim=2048, ratio=0.5)),
}
# a seed whose noise holds a tie inside one image (found by tie_seed below), for the cases that pin the tie order
TIE_CASES = {
    "mae_tie": ("mae", dict(image=(64, 64), patch=(2, 2), dim=64, depth=1, heads=2, dim_head=32, mlp_dim=64, ratio=0.5,
                            decoder_dim=32, decoder_depth=1, decoder_heads=2, decoder_dim_head=16)),
    "simmim_tie": ("simmim", dict(image=(64, 64), patch=(2, 2), dim=64, depth=1, heads=2, dim_head=32, mlp_dim=64, ratio=0.5)),
}


def tie_seed(b, n, start=0):
    """The first seed >= start whose draw-0 noise of a batch of b images with n patches holds a tie."""
    s = start
    while not has_tie(noise(b, n, s, 0)):
        s += 1
    return s


def case_seed(name):
    kind, cfg = ALL_CASES[name]
    if name in TIE_CASES:
        H, W = cfg["image"]
        return tie_seed(BATCH, (H // cfg["patch"][0]) * (W // cfg["patch"][1]))
    return SEED


ALL_CASES = {**CASES, **TIE_CASES}


def call_size(cfg):
    return cfg.get("call", cfg["image"])


# ------------------------------------------------------------------------------------------------ the reference over the shim
@contextlib.contextmanager
def installed(reference_dir, seed=0):
    """oracle/tf_shim.installed(reference_dir) with tf.random.uniform returning the engine's noise for the call's [b, n] shape,
    the draw counter counting the calls (yielded as state['d']); state['argsort'] / ['top_k'] / ['to_pixels'] / ['to_patch']
    record what those produced in the last call."""
    from oracle import tf_shim
    state = {"d": 0}

    def uniform(shape, *_, **__):
        b, n = (int(s) for s in shape)
        u = noise(b, n, seed, state["d"])
        state["d"] += 1
        return u.astype(tf_shim.get_dtype())

    with tf_shim.installed(reference_dir) as tf:
        tf.random.uniform = tf_shim._returns_tensor(uniform)
        argsort, top_k = tf.argsort, tf.math.top_k

        def rec_argsort(*a, **k):
            r = argsort(*a, **k)
            state["argsort"] = np.asarray(r).copy()
            return r

        def rec_top_k(*a, **k):
            r = top_k(*a, **k)
            state["top_k"] = np.asarray(r.indices).copy()
            return r
        tf.argsort, tf.math.top_k = rec_argsort, rec_top_k
        yield state


def _record(state, key, fn):
    def wrapped(*a, **k):
        r = fn(*a, **k)
        state[key] = np.asarray(r).view(np.ndarray).copy()
        return r
    return wrapped


def load_weights(model, kind, w, enc_w, dtype):
    """The engine's weights into a reference MAE / SimMIM by attribute path (mae.py:35-47, simmim.py:77-86); enc_w: the full ViT
    weights of its encoder (cls_token and mlp_head are never used)."""
    from oracle import ref_bind
    cast = lambda d: {k: np.asarray(v, dtype) for k, v in d.items()}
    w, enc_w = cast(w), cast(enc_w)
    ref_bind.load_weights(model.encoder, "vit", enc_w)
    model.mask_token.assign(w["mask_token"])
    if kind == "mae":
        if "enc_to_dec.kernel" in w:
            model.enc_to_dec.set_weights([w["enc_to_dec.kernel"], w["enc_to_dec.bias"]])
        ref_bind._set_transformer(model.decoder, w, "decoder.layers.", "vit")
        model.decoder_pos_emb.embeddings.assign(w["decoder_pos_emb.embeddings"])
    model.to_pixels.set_weights([w["to_pixels.kernel"], w["to_pixels.bias"]])


def encoder_weights(w, cfg, num_classes=5, seed=7):
    """ViT weights of the reference encoder: the engine's encoder weights plus a cls token and an mlp_head, which MAE / SimMIM
    never read."""
    rng = np.random.default_rng(seed)
    e = {k: v for k, v in w.items() if k == "pos_embedding" or k.startswith(("patch.", "layers."))}
    e.update({"cls_token": rng.standard_normal((1, 1, cfg["dim"])), "head_norm.gamma": np.ones(cfg["dim"]),
              "head_norm.beta": np.zeros(cfg["dim"]), "head.kernel": rng.standard_normal((cfg["dim"], num_classes)) * 0.1,
              "head.bias": np.zeros(num_classes)})
    return {k: np.asarray(v, np.float32) for k, v in e.items()}


def reference_run(reference_dir, name, variant, dtype=np.float64):
    """dict(loss, pred, masked_patches, indices) of the reference's unmodified MAE / SimMIM over the shim in `dtype`, called
    with the draw counter at 0 after one building call.  indices: MAE's whole argsort [b, n], SimMIM's top_k ids [b, nm]."""
    from oracle import tf_shim
    kind, cfg = ALL_CASES[name]
    seed = case_seed(name)
    w = weights(kind, cfg, variant)
    img = images(cfg, BATCH, size=call_size(cfg)).astype(dtype)
    tf_shim.set_dtype(dtype)
    try:
        with installed(reference_dir, seed) as state:
            vit = importlib.import_module("vit")
            enc = vit.ViT(image_size=cfg["image"], patch_size=cfg["patch"], num_classes=5, dim=cfg["dim"], depth=cfg["depth"],
                          heads=cfg["heads"], mlp_dim=cfg["mlp_dim"], dim_head=cfg["dim_head"])
            H, W = cfg["image"]
            if kind == "mae":
                mod = importlib.import_module("mae")
                model = mod.MAE(image_size=H, encoder=enc, decoder_dim=cfg["decoder_dim"], masking_ratio=cfg["ratio"],
                                decoder_depth=cfg["decoder_depth"], decoder_heads=cfg["decoder_heads"], decoder_dim_head=cfg["decoder_dim_head"])
            else:
                mod = importlib.import_module("simmim")
                model = mod.SimMIM(image_size=H, encoder=enc, masking_ratio=cfg["ratio"])
            model(img)                                               # builds the lazily created variables
            load_weights(model, kind, w, encoder_weights(w, cfg), dtype)
            model.to_pixels = _record(state, "pred", model.to_pixels)         # instrumentation on the instance
            model.to_patch = _record(state, "patches", model.to_patch)
            state["d"] = 0
            loss = float(np.asarray(model(img)))
    finally:
        tf_shim.set_dtype(np.float32)
    nm = num_masked(cfg["ratio"], state["patches"].shape[1])
    ids = state["argsort"] if kind == "mae" else state["top_k"]
    masked = np.take_along_axis(state["patches"], ids[:, :nm, None].astype(np.int64), 1)
    return dict(loss=loss, pred=state["pred"], masked_patches=masked, indices=ids.astype(np.int32))

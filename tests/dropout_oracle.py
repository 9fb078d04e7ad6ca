"""Training-mode dropout of ViT, DeepViT, CaiT and CrossViT (include/vitb200.h, vb_set_dropout) in float64, two ways:

- `spec(...)`: a numpy restatement of the four forwards with every Dropout site masked from the engine's Philox stream, the sites
  numbered by hand in the reference's call order;
- `reference(...)`: the reference's own classes, unmodified, over the numpy stand-in for TensorFlow (oracle/tf_shim.py), with the
  stand-in's Dropout drawing from the same stream inside `philox_dropout(seed, draw)`: there it numbers its calls from 0 and masks
  its input viewed as [M, N] (leading axes flattened).

The two agreeing pins the site numbering to the reference's own execution order."""
import contextlib
import json

import numpy as np
from einops import rearrange

import oracle
from oracle import ref_bind, tf_shim
from oracle.spec_numpy import dense, gelu, layer_norm, patch_embed, softmax
from ats_oracle import philox4x32_10

SEED = 0x5EED_D50F_0123_4567
WEIGHT_SEED, IMAGE_SEED, BATCH = 11, 12, 2
WEIGHTS = ("init", "stress")

# name -> (constructor kwargs with kind, image (h, w) of the call or None for image_size).  Together they reach every dropout GEMM
# instance: M = 2 x 65 = 130 rows (two row tiles, the last ragged), mlp_dim 1536 at dim 64 (the width whose inference fc1 takes the
# 192-wide tile), dim 48 (the bf16 SIMT fallback), an image smaller than image_size, no out-projection, LayerScale and a class stack,
# CrossViT with and without ProjectInOut's projections, and dropout only / emb_dropout only / both.
CASES = {
    "vit_cls": (dict(kind="vit", image_size=64, patch_size=8, num_classes=10, dim=64, depth=2, heads=2, dim_head=32, mlp_dim=1536,
                     dropout=0.1, emb_dropout=0.1), None),
    "vit_mean_rect": (dict(kind="vit", image_size=(32, 48), patch_size=8, num_classes=7, dim=64, depth=1, heads=2, dim_head=32,
                           mlp_dim=128, pool="mean", dropout=0.25, emb_dropout=0.0), None),
    "vit_noproj": (dict(kind="vit", image_size=32, patch_size=8, num_classes=5, dim=64, depth=2, heads=1, dim_head=64, mlp_dim=64,
                        dropout=0.1, emb_dropout=0.2), None),
    "vit_odd": (dict(kind="vit", image_size=32, patch_size=8, num_classes=6, dim=48, depth=1, heads=2, dim_head=24, mlp_dim=80,
                     dropout=0.0, emb_dropout=0.3), None),
    "vit_small_image": (dict(kind="vit", image_size=64, patch_size=8, num_classes=5, dim=64, depth=1, heads=2, dim_head=32,
                             mlp_dim=128, dropout=0.5, emb_dropout=0.1), (32, 48)),
    "deepvit": (dict(kind="deepvit", image_size=32, patch_size=8, num_classes=10, dim=64, depth=2, heads=4, dim_head=16, mlp_dim=128,
                     dropout=0.1, emb_dropout=0.1), None),
    "cait": (dict(kind="cait", image_size=32, patch_size=8, num_classes=10, dim=64, depth=2, cls_depth=2, heads=4, dim_head=16,
                  mlp_dim=128, dropout=0.1, emb_dropout=0.1), None),
    "crossvit_proj": (dict(kind="crossvit", image_size=64, num_classes=10, sm_dim=64, lg_dim=128, sm_patch_size=8, lg_patch_size=16,
                           sm_enc_depth=1, lg_enc_depth=2, sm_enc_heads=2, lg_enc_heads=2, sm_enc_mlp_dim=64, lg_enc_mlp_dim=128,
                           sm_enc_dim_head=32, lg_enc_dim_head=32, cross_attn_depth=2, cross_attn_heads=2, cross_attn_dim_head=32,
                           depth=2, dropout=0.1, emb_dropout=0.1), None),
    "crossvit_samedim": (dict(kind="crossvit", image_size=32, num_classes=6, sm_dim=64, lg_dim=64, sm_patch_size=8, lg_patch_size=16,
                              sm_enc_depth=1, lg_enc_depth=1, sm_enc_heads=2, lg_enc_heads=2, sm_enc_mlp_dim=64, lg_enc_mlp_dim=64,
                              sm_enc_dim_head=32, lg_enc_dim_head=32, cross_attn_depth=1, cross_attn_heads=2, cross_attn_dim_head=32,
                              depth=1), None),     # the reference's defaults: dropout = emb_dropout = 0.1 (cross_vit.py:252-253)
}


def fixture_name(name, gen):
    return f"dropout_{name}__{gen}__refshim.npz"


def rates(name):
    kw = CASES[name][0]
    return kw.get("dropout", 0.1 if kw["kind"] == "crossvit" else 0.0), kw.get("emb_dropout", 0.1 if kw["kind"] == "crossvit" else 0.0)


def config(name):
    kw = dict(CASES[name][0])
    kind = kw.pop("kind")
    kw.pop("dropout", None)
    kw.pop("emb_dropout", None)
    return oracle.make_config(kind, **kw)


def weights(name, gen):
    cfg = config(name)
    return (oracle.init_weights if gen == "init" else oracle.stress_weights)(cfg, WEIGHT_SEED)


def images(name):
    cfg = config(name)
    hw = CASES[name][1]
    return oracle.make_image(cfg, BATCH, IMAGE_SEED, *(hw or (None, None)))


# ----------------------------------------------------------------------------------------------------------- the stream
def keep_mask(seed, draw, site, M, N, rate):
    """keep bool [M, N] of site `site` at draw `draw` (include/vitb200.h)."""
    m = np.arange(M, dtype=np.uint64)[:, None]
    n = np.arange(N, dtype=np.uint64)[None, :]
    m, n = np.broadcast_arrays(m, n)
    ctr = np.stack([n >> np.uint64(1), ((m >> np.uint64(4)) << np.uint64(3)) | (m & np.uint64(7)),
                    np.full(m.shape, site, np.uint64), np.full(m.shape, draw & 0xFFFFFFFF, np.uint64)], -1)
    x = philox4x32_10(ctr, (seed & 0xFFFFFFFF, seed >> 32))
    idx = (2 * ((m >> np.uint64(3)) & np.uint64(1)) + (n & np.uint64(1))).astype(np.int64)
    word = np.take_along_axis(x, idx[..., None], -1)[..., 0]
    u = (word >> np.uint32(8)).astype(np.float64) * 2.0 ** -24
    return u >= np.float64(np.float32(rate))


def apply(x, seed, draw, site, rate):
    """Dropout(rate) of site `site` on x viewed as [M, N]: kept values times 1 / (1 - rate) in x's dtype, the rest 0."""
    if rate == 0:
        return x
    keep = keep_mask(seed, draw, site, int(np.prod(x.shape[:-1])), x.shape[-1], rate).reshape(x.shape)
    return np.where(keep, x * np.asarray(1.0 / (1.0 - rate), x.dtype), np.zeros((), x.dtype))


class _Sites:
    def __init__(self, seed, draw):
        self.seed, self.draw, self.next = seed, draw, 0

    def __call__(self, x, rate):
        s = self.next
        self.next += 1
        return apply(x, self.seed, self.draw, s, rate)


# ----------------------------------------------------------------------------------------------------------- numpy spec
def _heads(t, h):
    return rearrange(t, 'b n (h d) -> b h n d', h=h)


def _attend(q, k, v, dh, mix_pre=None, mix_post=None, reattn=None, w=None, pre=None):
    dots = np.einsum('bhid,bhjd->bhij', q, k) * dh ** -0.5
    if mix_pre is not None:
        dots = np.einsum('bhij,hg->bgij', dots, mix_pre)                     # cait.py:123
    attn = softmax(dots)
    if mix_post is not None:
        attn = np.einsum('bhij,hg->bgij', attn, mix_post)                    # cait.py:125
    if reattn is not None:                                                    # deepvit.py:83-84
        attn = np.einsum('bhij,hg->bgij', attn, reattn)
        attn = rearrange(layer_norm(rearrange(attn, 'b h i j -> b i j h'), w, pre + "reattn_norm"), 'b i j h -> b h i j')
    return rearrange(np.einsum('bhij,bhjd->bhid', attn, v), 'b h n d -> b n (h d)')


def _attn_vit(x, w, pre, cfg, drop, r):
    q, k, v = (_heads(t, cfg["heads"]) for t in np.split(dense(x, w, pre + "to_qkv", bias=False), 3, axis=-1))
    out = _attend(q, k, v, cfg["dim_head"], reattn=w.get(pre + "reattn_weights") if cfg["kind"] == "deepvit" else None, w=w, pre=pre)
    if pre + "to_out.kernel" not in w:                                        # vit.py:53: no Dense, no Dropout
        return out
    return drop(dense(out, w, pre + "to_out"), r)


def _attn_qkv(x, w, pre, heads, dh, drop, r, context=None, talking=False):
    ctx = x if context is None else np.concatenate([x, context], axis=1)
    q = _heads(dense(x, w, pre + "to_q", bias=False), heads)
    k, v = (_heads(t, heads) for t in np.split(dense(ctx, w, pre + "to_kv", bias=False), 2, axis=-1))
    out = _attend(q, k, v, dh, w.get(pre + "mix_pre") if talking else None, w.get(pre + "mix_post") if talking else None)
    return drop(dense(out, w, pre + "to_out"), r)


def _mlp(x, w, pre, drop, r):
    return drop(dense(drop(gelu(dense(x, w, pre + "fc1")), r), w, pre + "fc2"), r)


def spec(name, gen, draw, seed=SEED, dtype=np.float64):
    """Logits [b, num_classes] of the case's training-mode call at draw `draw`."""
    cfg = config(name)
    w = {k: np.asarray(v, dtype) for k, v in weights(name, gen).items()}
    img = np.asarray(images(name), dtype)
    r, re = rates(name)
    drop = _Sites(seed, draw)
    kind = cfg["kind"]
    if kind in ("vit", "deepvit"):
        x = patch_embed(img, w, "patch", cfg["patch_h"], cfg["patch_w"])
        b, n, d = x.shape
        x = np.concatenate([np.broadcast_to(w["cls_token"], (b, 1, d)), x], axis=1) + w["pos_embedding"][:, :n + 1]
        x = drop(x, re)
        for L in range(cfg["depth"]):
            pre = f"layers.{L}."
            x = _attn_vit(layer_norm(x, w, pre + "attn_norm"), w, pre, cfg, drop, r) + x
            x = _mlp(layer_norm(x, w, pre + "ff_norm"), w, pre, drop, r) + x
        x = x.mean(axis=1) if cfg["pool"] == "mean" else x[:, 0]
        return dense(layer_norm(x, w, "head_norm"), w, "head")
    if kind == "cait":
        x = patch_embed(img, w, "patch", cfg["patch_h"], cfg["patch_w"])
        b, n, d = x.shape
        x = drop(x + w["pos_embedding"][:, :n], re)

        def stack(x, name, depth, context=None):
            for L in range(depth):
                pre = f"{name}.layers.{L}."
                a = _attn_qkv(layer_norm(x, w, pre + "attn_norm"), w, pre, cfg["heads"], cfg["dim_head"], drop, r, context, True)
                x = a * w[pre + "attn_scale"] + x
                x = _mlp(layer_norm(x, w, pre + "ff_norm"), w, pre, drop, r) * w[pre + "ff_scale"] + x
            return x
        x = stack(x, "patch_transformer", cfg["depth"])
        x = stack(np.broadcast_to(w["cls_token"], (b, 1, d)), "cls_transformer", cfg["cls_depth"], x)
        return dense(layer_norm(x[:, 0], w, "head_norm"), w, "head")
    toks = {}
    for br in ("sm", "lg"):
        p = cfg[f"{br}_patch_size"]
        x = patch_embed(img, w, f"{br}_embed.patch", p, p)
        b, n, d = x.shape
        x = np.concatenate([np.broadcast_to(w[f"{br}_embed.cls_token"], (b, 1, d)), x], axis=1) + w[f"{br}_embed.pos_embedding"][:, :n + 1]
        toks[br] = drop(x, re)

    def encoder(x, pre, br):
        for L in range(cfg[f"{br}_enc_depth"]):
            p = f"{pre}layers.{L}."
            x = _attn_qkv(layer_norm(x, w, p + "attn_norm"), w, p, cfg[f"{br}_enc_heads"], cfg[f"{br}_enc_dim_head"], drop, r) + x
            x = _mlp(layer_norm(x, w, p + "ff_norm"), w, p, drop, r) + x
        return layer_norm(x, w, pre + "final_norm")

    def cross(cls, ctx, pre):
        x = cls
        proj = (pre + "project_in.kernel") in w
        if proj:
            x = dense(x, w, pre + "project_in")
        x = _attn_qkv(layer_norm(x, w, pre + "norm"), w, pre, cfg["cross_attn_heads"], cfg["cross_attn_dim_head"], drop, r, ctx)
        if proj:
            x = dense(x, w, pre + "project_out")
        return x + cls

    sm, lg = toks["sm"], toks["lg"]
    for D in range(cfg["depth"]):
        sm = encoder(sm, f"blocks.{D}.sm_enc.", "sm")
        lg = encoder(lg, f"blocks.{D}.lg_enc.", "lg")
        sm_cls, sm_p, lg_cls, lg_p = sm[:, :1], sm[:, 1:], lg[:, :1], lg[:, 1:]
        for R in range(cfg["cross_attn_depth"]):
            sm_cls = cross(sm_cls, lg_p, f"blocks.{D}.cross.{R}.sm_attend_lg.")
            lg_cls = cross(lg_cls, sm_p, f"blocks.{D}.cross.{R}.lg_attend_sm.")
        sm = np.concatenate([sm_cls, sm_p], axis=1)
        lg = np.concatenate([lg_cls, lg_p], axis=1)
    return dense(layer_norm(sm[:, 0], w, "sm_head_norm"), w, "sm_head") + dense(layer_norm(lg[:, 0], w, "lg_head_norm"), w, "lg_head")


# ----------------------------------------------------------------------------------------------------------- the reference
@contextlib.contextmanager
def philox_dropout(seed, draw):
    """Within the block the stand-in's Dropout numbers its calls from 0 and masks from the engine's stream (`apply`); outside it
    keeps its numpy-RNG behaviour.  Yields the site counter (its `next` is the number of Dropout calls so far)."""
    sites = _Sites(seed, draw)
    original = tf_shim.Dropout.call

    def call(self, inputs, training=None):
        s = sites.next
        sites.next += 1
        if not training or self.rate == 0.0:
            return inputs
        return tf_shim._t(apply(tf_shim._arr(inputs), seed, draw, s, self.rate))

    tf_shim.Dropout.call = call
    try:
        yield sites
    finally:
        tf_shim.Dropout.call = original


def reference(ref_dir, name, gen, draw, dtype=np.float64, seed=SEED):
    """The reference's own class over the stand-in, model(img, training=True) in Philox mode -> (logits, Dropout calls)."""
    kind, kw = ref_bind.ctor_kwargs(CASES[name][0])
    kw["dropout"], kw["emb_dropout"] = rates(name)      # ctor_kwargs zeroes CrossViT's defaults, which inference ignores
    w = {k: v.astype(dtype) for k, v in weights(name, gen).items()}
    img = images(name).astype(dtype)
    tf_shim.set_dtype(dtype)
    try:
        with tf_shim.installed(ref_dir):
            model = ref_bind.build_model(kind, kw, w, img)
            with philox_dropout(seed, draw) as sites:
                out = ref_bind.to_numpy(model(img, training=True))
            return out, sites.next
    finally:
        tf_shim.set_dtype(np.float32)


def site_count(name):
    """The Dropout calls of one forward, counted as the engine numbers them."""
    cfg = config(name)
    kind = cfg["kind"]
    if kind == "crossvit":
        per = lambda br: 3 * cfg[f"{br}_enc_depth"]   # noqa: E731
        return 2 + cfg["depth"] * (per("sm") + per("lg") + 2 * cfg["cross_attn_depth"])
    per_layer = 2 if (kind == "vit" and cfg["heads"] == 1 and cfg["dim_head"] == cfg["dim"]) else 3
    return 1 + per_layer * (cfg["depth"] + cfg.get("cls_depth", 0))


def meta(name, gen):
    return json.dumps(dict(case=CASES[name][0], image=CASES[name][1], variant=gen, seed=SEED, weight_seed=WEIGHT_SEED,
                           image_seed=IMAGE_SEED, batch=BATCH, generator="tests/golden/make_dropout_golden.py"))

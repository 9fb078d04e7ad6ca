"""Float64 restatement of MPP.call (reference mpp.py:168-218) as include/vitb200.h defines it, with the engine's draws: one
Philox4x32-10 block per (image, position) at MAE's key and counter (j, b, d_lo, d_hi), words 0-3 the mask noise, the random-patch
coin, the random patch id and the replace coin.

- Mask: k = ceil(mask_prob * n) in double; the masked ids are the top_k of u0 (descending, ties to the smaller id).
- Corruption per masked position: the original patch at the random id where the random-patch coin is true, then the pixel-space
  mask_token where the replace coin is true.  corrupt=False gives what the reference computes under TF 2, where `.numpy()` returns
  a copy and both writes are lost.
- Encoder: patch Dense + positions by position, the cls row cls_token + pos_embedding[0], the encoder's layers over n + 1 rows.
- Loss: to_bits on the masked rows (ids ascending); softmax_cross_entropy_with_logits(labels=logits, logits=targets [M, 1])
  broadcasts the targets to [M, K] before the softmax, so every row's loss is ln(K) * sum_c logits[row, c].

Also here: the fixture cases (tests/golden/make_mpp_golden.py), their weights, and the unmodified reference run over the numpy
stand-in for TensorFlow with tf.random.uniform returning the engine's words and `.numpy()` returning a copy."""
import contextlib
import importlib
import math

import numpy as np

from ats_oracle import bf16_round, philox4x32_10
from mim_oracle import _layer_weights, _transformer, images, to_patches

BATCH, SEED = 2, 0


def words(b, n, seed=0, d=0):
    """The four Philox words [b, n, 4] (uint64 holding uint32) of one call at draw counter d."""
    bb, jj = np.meshgrid(np.arange(b), np.arange(n), indexing="ij")
    ctr = np.stack([jj.astype(np.uint64), bb.astype(np.uint64), np.full(bb.shape, d & 0xFFFFFFFF, np.uint64),
                    np.full(bb.shape, d >> 32, np.uint64)], -1)
    return philox4x32_10(ctr, (seed & 0xFFFFFFFF, seed >> 32))


def unit(w, dtype=np.float64):
    return ((w >> 8).astype(np.float64) * 2.0 ** -24).astype(dtype)


def random_ids(w2, n):
    return ((w2.astype(np.uint64) * np.uint64(n)) >> np.uint64(32)).astype(np.int64)


def num_masked(mask_prob, n):
    return math.ceil(mask_prob * n)                                  # mpp.py:80, in double


def draws(b, n, cfg, seed=0, d=0):
    """dict(mask_ids [b, k] ascending, mask [b, n], rand_coin, random_id, replace_coin [b, n], source [b, n], u0)."""
    x = words(b, n, seed, d)
    k = num_masked(cfg["mask_prob"], n)
    u0 = unit(x[..., 0])
    top = np.argsort(-u0, axis=-1, kind="stable")[:, :k]
    mask = np.zeros((b, n), bool)
    np.put_along_axis(mask, top, True, 1)
    rp, rep = cfg["random_patch_prob"], cfg["replace_prob"]
    # the coins compare float32 noise with the Python double rounded to float32, as TF converts it
    rand_coin = unit(x[..., 1], np.float32) < np.float32(rp / (1 - rep)) if rp > 0 else np.zeros((b, n), bool)
    random_id = random_ids(x[..., 2], n)
    replace_coin = unit(x[..., 3], np.float32) < np.float32(rep)
    source = np.broadcast_to(np.arange(n), (b, n)).copy()
    source = np.where(mask & rand_coin, random_id, source)
    source = np.where(mask & replace_coin, -1, source)
    return dict(mask_ids=np.sort(top, -1).astype(np.int32), mask=mask, rand_coin=rand_coin, random_id=random_id,
                replace_coin=replace_coin, source=source.astype(np.int32), u0=u0)


def forward(w, img, cfg, seed=0, d=0, bf16_storage=False, corrupt=True):
    """MPP call in float64 (bf16_storage: the bf16 engine's stored tensors rounded, as mim_oracle.forward).  Returns
    dict(loss, logits [b, k, K], mask_ids, source, ...the draws)."""
    f = lambda key: np.asarray(w[key], np.float64)
    st = bf16_round if bf16_storage else (lambda a: a)
    mm = (lambda a, k: bf16_round(bf16_round(a) @ bf16_round(k))) if bf16_storage else (lambda a, k: a @ k)
    x0 = np.asarray(img, np.float64)
    b = x0.shape[0]
    p = cfg["patch"]
    patches = to_patches(x0, p, p)
    n = patches.shape[1]
    dr = draws(b, n, cfg, seed, d)
    if corrupt:
        src = dr["source"].astype(np.int64)
        taken = np.take_along_axis(patches, np.maximum(src, 0)[..., None], 1)
        patches = np.where((src < 0)[..., None], f("mask_token")[None, None], taken)
    pos = f("pos_embedding")[0]
    x = st(mm(patches, f("patch.kernel")) + f("patch.bias") + st(pos[1:n + 1]))
    cls = np.broadcast_to(st(f("cls_token")[0, 0] + pos[0]), (b, 1, x.shape[-1]))
    x = np.concatenate([cls, x], 1)
    x = _transformer(x, w, "layers.", cfg["depth"], cfg["heads"], cfg["dim_head"], st, mm)
    rows = np.take_along_axis(x[:, 1:], dr["mask_ids"][..., None].astype(np.int64), 1)
    logits = st(mm(rows, f("to_bits.kernel")) + f("to_bits.bias"))
    K = logits.shape[-1]
    loss = math.log(K) * float(logits.sum(-1).mean())
    return dict(loss=loss, logits=logits, **dr)


# ------------------------------------------------------------------------------------------------ cases and weights
def classes(cfg):
    return 2 ** (3 * cfg.get("bits", 3))


def weights(cfg, variant="init", seed=0):
    """The engine's MPP weights of a case: the encoder ViT's (cls_token included, no mlp_head), mask_token [patch_dim] and
    to_bits; 'init' at Keras-like scale, 'stress' with non-trivial biases, LayerNorms and larger positions."""
    rng = np.random.default_rng(seed + (0 if variant == "init" else 1000))
    stress = variant == "stress"
    p = cfg["patch"]
    H, W = cfg["image"]
    dim, pd, K = cfg["dim"], p * p * 3, classes(cfg)
    npos = (H // p) * (W // p) + 1
    w = {"pos_embedding": rng.standard_normal((1, npos, dim)) * (1.0 if stress else 0.5),
         "cls_token": rng.standard_normal((1, 1, dim)),
         "patch.kernel": rng.standard_normal((pd, dim)) * pd ** -0.5, "patch.bias": (0.1 if stress else 0.0) * rng.standard_normal(dim)}
    for L in range(cfg["depth"]):
        w.update(_layer_weights(rng, f"layers.{L}.", dim, cfg["heads"], cfg["dim_head"], cfg["mlp_dim"], stress))
    w["mask_token"] = rng.standard_normal(pd)
    w["to_bits.kernel"] = rng.standard_normal((dim, K)) * dim ** -0.5
    w["to_bits.bias"] = (0.1 if stress else 0.0) * rng.standard_normal(K)
    return {k: np.asarray(v, np.float32) for k, v in w.items()}


_SMALL = dict(image=(32, 32), patch=8, dim=64, depth=2, heads=2, dim_head=32, mlp_dim=128, mask_prob=0.3, replace_prob=0.5,
              random_patch_prob=0.5)
CASES = {
    # mpp.py:221-240: ViT 256^2 / 32, dim 1024, depth 6, heads 8, mlp 2048; mask 0.15, random patch 0.30, replace 0.50
    "mpp_usage": dict(image=(256, 256), patch=32, dim=1024, depth=6, heads=8, dim_head=64, mlp_dim=2048, mask_prob=0.15,
                      replace_prob=0.5, random_patch_prob=0.3),
    "mpp_no_random": dict(_SMALL, random_patch_prob=0.0),
    "mpp_coin_above_one": dict(_SMALL, replace_prob=0.8, random_patch_prob=0.3),       # 0.3 / (1 - 0.8) = 1.5
    "mpp_ceil": dict(_SMALL, image=(40, 40), patch=4, depth=1, mlp_dim=64, mask_prob=0.07),   # 0.07 * 100 = 7.000000000000001: k = 8
    "mpp_rect": dict(_SMALL, image=(24, 40), depth=1),
    "mpp_small_image": dict(_SMALL, patch=4, depth=1, call=(16, 24)),
    "mpp_bits1": dict(_SMALL, depth=1, bits=1),
    "mpp_bits4": dict(_SMALL, image=(16, 16), depth=1, bits=4),
    "mpp_odd": dict(_SMALL, image=(24, 24), patch=4, dim=40, depth=1, heads=2, dim_head=20, mlp_dim=80),
    "mpp_batch1": dict(_SMALL, batch=1),
}
TIE_CASES = {"mpp_tie": dict(_SMALL, image=(64, 64), patch=2, depth=1, mlp_dim=64, mask_prob=0.5, bits=1)}
ALL_CASES = {**CASES, **TIE_CASES}


def batch(cfg):
    return cfg.get("batch", BATCH)


def call_size(cfg):
    return cfg.get("call", cfg["image"])


def tie_seed(b, n, k, start=0):
    """The first seed >= start whose draw-0 mask noise holds a tie across some image's top-k boundary."""
    s = start
    while True:
        u = np.sort(words(b, n, s, 0)[..., 0] >> 8, -1)[:, ::-1]
        if (u[:, k - 1] == u[:, k]).any():
            return s
        s += 1


def case_seed(name):
    cfg = ALL_CASES[name]
    if name in TIE_CASES:
        H, W = cfg["image"]
        n = (H // cfg["patch"]) * (W // cfg["patch"])
        return tie_seed(batch(cfg), n, num_masked(cfg["mask_prob"], n))
    return SEED


def spec(name, variant, **kw):
    cfg = ALL_CASES[name]
    return forward(weights(cfg, variant), images(cfg, batch(cfg), size=call_size(cfg)), cfg, seed=case_seed(name), **kw)


# ------------------------------------------------------------------------------------------------ the reference over the shim
def _cross_entropy_broadcast(labels, logits, axis=-1, **_):
    """tf.nn.softmax_cross_entropy_with_logits as TF's kernel computes it: `logits` broadcast to the shape of `labels` before
    the softmax.  Equal to the stand-in's own version whenever the two shapes are equal."""
    from oracle import tf_shim
    labels, logits = np.broadcast_arrays(np.asarray(labels), np.asarray(logits))
    return -(labels * tf_shim._log_softmax(logits, axis)).sum(axis=axis)


@contextlib.contextmanager
def installed(reference_dir, seed, cfg):
    """oracle/tf_shim.installed(reference_dir) with MPP's draws: tf.random.uniform returns, call by call, the engine's words in
    the order mpp.py draws them (0-3, or 0 and 3 when random_patch_prob == 0; the int draw as (word 2 * maxval) >> 32), the draw
    counter advancing once per MPP call (yielded as state['d']); `.numpy()` returns a copy, as TF 2's EagerTensor.numpy() does;
    and softmax_cross_entropy_with_logits broadcasts before its softmax, as TF's kernel does."""
    from oracle import tf_shim
    order = (0, 1, 2, 3) if cfg["random_patch_prob"] > 0 else (0, 3)
    state = {"d": 0, "i": 0}

    def uniform(shape, minval=0, maxval=None, dtype=None, **_):
        b, n = (int(s) for s in shape)
        word = order[state["i"]]
        x = words(b, n, seed, state["d"])[..., word]
        state["i"] += 1
        if state["i"] == len(order):
            state["i"] = 0
            state["d"] += 1
        dt = np.dtype(dtype or tf_shim.get_dtype())
        if np.issubdtype(dt, np.integer):
            state["random_id"] = random_ids(x, int(maxval))
            return state["random_id"].astype(dt)
        return unit(x, dt)

    numpy = tf_shim.Tensor.numpy
    tf_shim.Tensor.numpy = lambda self: self.view(np.ndarray).copy()
    try:
        with tf_shim.installed(reference_dir) as tf:
            tf.random.uniform = tf_shim._returns_tensor(uniform)
            tf.nn.softmax_cross_entropy_with_logits = tf_shim._returns_tensor(_cross_entropy_broadcast)
            yield state
    finally:
        tf_shim.Tensor.numpy = numpy


def reference_run(reference_dir, name, variant, dtype=np.float64):
    """dict(loss, logits [b, k, K], mask_ids, rand_coin, random_id, replace_coin) of the reference's unmodified MPP over the shim
    in `dtype`, called with the draw counter at 0 after one building call.  The coins are what prob_mask_like returned (an
    all-false rand_coin when the reference draws none)."""
    from oracle import ref_bind, tf_shim
    cfg = ALL_CASES[name]
    seed = case_seed(name)
    w = weights(cfg, variant)
    img = images(cfg, batch(cfg), size=call_size(cfg)).astype(dtype)
    tf_shim.set_dtype(dtype)
    try:
        with installed(reference_dir, seed, cfg) as state:
            import io
            import sys
            saved, sys.stdout = sys.stdout, io.StringIO()
            try:
                mod = importlib.import_module("mpp")                 # builds the usage block's model at import
            finally:
                sys.stdout = saved
            vit = importlib.import_module("vit")
            enc = vit.ViT(image_size=cfg["image"], patch_size=cfg["patch"], num_classes=5, dim=cfg["dim"], depth=cfg["depth"],
                          heads=cfg["heads"], mlp_dim=cfg["mlp_dim"], dim_head=cfg["dim_head"])
            model = mod.MPP(image_size=cfg["image"][0], transformer=enc, patch_size=cfg["patch"], output_channel_bits=cfg.get("bits", 3),
                            mask_prob=cfg["mask_prob"], replace_prob=cfg["replace_prob"], random_patch_prob=cfg["random_patch_prob"])
            model(img)                                               # builds to_bits
            enc_w = {k: np.asarray(v, dtype) for k, v in w.items() if not k.startswith(("to_bits.", "mask_token"))}
            enc_w.update({"head_norm.gamma": np.ones(cfg["dim"], dtype), "head_norm.beta": np.zeros(cfg["dim"], dtype),
                          "head.kernel": np.zeros((cfg["dim"], 5), dtype), "head.bias": np.zeros(5, dtype)})
            ref_bind.load_weights(model.transformer, "vit", enc_w)
            model.mask_token.assign(np.asarray(w["mask_token"], dtype).reshape(1, 1, -1))
            model.to_bits.set_weights([np.asarray(w["to_bits.kernel"], dtype), np.asarray(w["to_bits.bias"], dtype)])
            coins, rec = [], {}
            plain_coin, plain_mask = mod.prob_mask_like, mod.get_mask_subset_with_prob
            to_bits = model.to_bits

            def coin(t, prob):
                r = plain_coin(t, prob)
                coins.append(np.asarray(r).copy())
                return r

            def mask_of(t, prob):
                r = plain_mask(t, prob)
                rec["mask"] = np.asarray(r).copy()
                return r

            def bits(x, *a, **k):
                r = to_bits(x, *a, **k)
                rec["logits"] = np.asarray(r).view(np.ndarray).copy()
                return r
            mod.prob_mask_like, mod.get_mask_subset_with_prob, model.to_bits = coin, mask_of, bits
            state["d"], state["i"] = 0, 0
            loss = float(np.asarray(model(img)))
    finally:
        tf_shim.set_dtype(np.float32)
    mask = rec["mask"]
    b, n = mask.shape
    ids = np.stack([np.nonzero(m)[0] for m in mask]).astype(np.int32)
    logits = np.take_along_axis(rec["logits"][:, 1:], ids[..., None].astype(np.int64), 1)
    rand_coin = coins[0] if len(coins) == 2 else np.zeros((b, n), bool)
    return dict(loss=loss, logits=logits, mask_ids=ids, rand_coin=rand_coin, random_id=state.get("random_id"), replace_coin=coins[-1])

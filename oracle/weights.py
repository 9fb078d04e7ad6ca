"""Canonical configs, weight names/shapes (SURVEY.md App. B) and seeded generators.

TEST INFRASTRUCTURE (see oracle/__init__.py).  Follows the reference constructors:
  ViT      vit_tensorflow/vit.py:107-157
  DeepViT  vit_tensorflow/deepvit.py:112-137 (+ Attention :46-71)
  CaiT     vit_tensorflow/cait.py:155-178 (+ LayerScale :33-45, Attention :85-105)
  CrossViT vit_tensorflow/cross_vit.py:232-288 (+ ImageEmbedder :199-217,
           Transformer :95-107, ProjectInOut :118-126, CrossTransformer :141-150)
  parallel ViT  vit_tensorflow/parallel_vit.py:120-165 (+ Parallel :36-42, Transformer :99-117)
  patch-merger ViT  vit_tensorflow/vit_with_patch_merger.py:134-172 (+ PatchMerger :42-47, Transformer :104-115)
  T2TViT   vit_tensorflow/t2t.py:50-94 (+ RearrangeUnfoldTransformer :17-36)

Weight layouts are the Keras layouts: Dense kernel ``[in, out]``, bias ``[out]``,
LayerNormalization gamma/beta ``[dim]``.
"""
from __future__ import annotations

import collections
import numpy as np


def _pair(t):
    return t if isinstance(t, tuple) else (t, t)


def make_config(kind: str, **kw) -> dict:
    """Normalise constructor kwargs to a flat config dict, applying the reference defaults."""
    kind = kind.lower()
    if kind in ("vit", "deepvit", "parallel_vit"):
        cfg = dict(kind=kind, pool="cls", dim_head=64, channels=3)
        if kind == "parallel_vit":
            cfg["num_parallel_branches"] = 2                          # parallel_vit.py:130
        cfg.update(kw)
        ih, iw = _pair(cfg["image_size"])
        ph, pw = _pair(cfg["patch_size"])
        assert ih % ph == 0 and iw % pw == 0, 'Image dimensions must be divisible by the patch size.'
        assert cfg["pool"] in {"cls", "mean"}, 'pool type must be either cls (cls token) or mean (mean pooling)'
        cfg.update(image_h=ih, image_w=iw, patch_h=ph, patch_w=pw,
                   num_patches=(ih // ph) * (iw // pw))
    elif kind == "cait":
        cfg = dict(kind=kind, dim_head=64, channels=3)
        cfg.update(kw)
        s, p = cfg["image_size"], cfg["patch_size"]
        assert s % p == 0, 'Image dimensions must be divisible by the patch size.'
        cfg.update(image_h=s, image_w=s, patch_h=p, patch_w=p, num_patches=(s // p) ** 2)
    elif kind == "crossvit":
        cfg = dict(kind=kind, channels=3, sm_patch_size=12, sm_enc_depth=1, sm_enc_heads=8,
                   sm_enc_mlp_dim=2048, sm_enc_dim_head=64, lg_patch_size=16, lg_enc_depth=4,
                   lg_enc_heads=8, lg_enc_mlp_dim=2048, lg_enc_dim_head=64, cross_attn_depth=2,
                   cross_attn_heads=8, cross_attn_dim_head=64, depth=3)
        cfg.update(kw)
        s = cfg["image_size"]
        for p in (cfg["sm_patch_size"], cfg["lg_patch_size"]):
            assert s % p == 0, 'Image dimensions must be divisible by the patch size.'
        cfg.update(image_h=s, image_w=s)
    elif kind == "patch_merger_vit":
        # vit_with_patch_merger.py:134-146 (ViT) and :104-109 (Transformer): no cls token, mean pooling in mlp_head (:168-172)
        cfg = dict(kind=kind, dim_head=64, channels=3, patch_merge_layer=None, patch_merge_num_tokens=8)
        cfg.update(kw)
        ih, iw = _pair(cfg["image_size"])
        ph, pw = _pair(cfg["patch_size"])
        assert ih % ph == 0 and iw % pw == 0, 'Image dimensions must be divisible by the patch size.'
        pml = cfg["patch_merge_layer"]
        cfg.update(image_h=ih, image_w=iw, patch_h=ph, patch_w=pw, num_patches=(ih // ph) * (iw // pw), pool="mean",
                   patch_merge_layer_index=(pml if pml is not None else cfg["depth"] // 2) - 1)   # :108
    elif kind == "t2t_vit":
        # t2t.py:50-94
        cfg = dict(kind=kind, pool="cls", channels=3, dim_head=64, t2t_layers=((7, 4), (3, 2), (3, 2)))
        cfg.update(kw)
        assert cfg["pool"] in {"cls", "mean"}, 'pool type must be either cls (cls token) or mean (mean pooling)'
        assert all(cfg.get(k) is not None for k in ("depth", "heads", "mlp_dim")), 'depth, heads, and mlp_dim must be supplied'
        cfg["t2t_layers"] = tuple((int(k), int(s)) for k, s in cfg["t2t_layers"])
        s = cfg["image_size"]
        out, layer_dim, dims = s, cfg["channels"], []
        for k, st in cfg["t2t_layers"]:
            layer_dim *= k * k                                            # t2t.py:63
            out = int(((out - k + 2 * (st // 2)) / st) + 1)               # conv_output_size t2t.py:14-15,66
            dims.append(layer_dim)
        cfg.update(image_h=s, image_w=s, t2t_dims=tuple(dims), num_patches=out * out)
    else:
        raise ValueError(f"unknown model kind {kind!r}")
    return cfg


def t2t_token_grid(cfg, h=None, w=None):
    """Token grid after every soft-split of T2T: tf.image.extract_patches(..., padding='SAME') yields ceil(size / stride)
    positions per axis (t2t.py:43); the last entry is the grid the main transformer sees."""
    h = cfg["image_h"] if h is None else h
    w = cfg["image_w"] if w is None else w
    grids = []
    for _, st in cfg["t2t_layers"]:
        h, w = -(-h // st), -(-w // st)
        grids.append((h, w))
    return grids


# ----------------------------------------------------------------------------- specs
# init kinds: 'glorot' (Dense kernel), 'zeros' (bias, beta), 'ones' (gamma), 'normal' (N(0,1)
# tf.random.normal Variables), ('fill', v) LayerScale.

def _dense(specs, name, din, dout, bias=True):
    specs[name + ".kernel"] = ((din, dout), "glorot")
    if bias:
        specs[name + ".bias"] = ((dout,), "zeros")


def _ln(specs, name, dim):
    specs[name + ".gamma"] = ((dim,), "ones")
    specs[name + ".beta"] = ((dim,), "zeros")


def _layerscale_eps(depth_index_plus_1: int) -> float:
    # cait.py:36-41 (keyed on layer index + 1, cait.py:142-143)
    d = depth_index_plus_1
    if d <= 18:
        return 0.1
    if d <= 24:
        return 1e-5
    return 1e-6


def _vit_layer(specs, pre, dim, heads, dim_head, mlp_dim, *, kind):
    inner = heads * dim_head
    _ln(specs, pre + "attn_norm", dim)
    if kind in ("vit", "deepvit"):
        _dense(specs, pre + "to_qkv", dim, 3 * inner, bias=False)
    else:  # cait / crossvit attention: to_q + to_kv (cait.py:94-95, cross_vit.py:61-62)
        _dense(specs, pre + "to_q", dim, inner, bias=False)
        _dense(specs, pre + "to_kv", dim, 2 * inner, bias=False)
    if kind == "deepvit":
        specs[pre + "reattn_weights"] = ((heads, heads), "normal")
        _ln(specs, pre + "reattn_norm", heads)
    if kind == "cait":
        specs[pre + "mix_pre"] = ((heads, heads), "normal")
        specs[pre + "mix_post"] = ((heads, heads), "normal")
    project_out = not (kind == "vit" and heads == 1 and dim_head == dim)  # vit.py:53 only
    if project_out:
        _dense(specs, pre + "to_out", inner, dim)
    _ln(specs, pre + "ff_norm", dim)
    _dense(specs, pre + "fc1", dim, mlp_dim)
    _dense(specs, pre + "fc2", mlp_dim, dim)


def weight_specs(cfg: dict) -> "collections.OrderedDict[str, tuple]":
    specs: collections.OrderedDict = collections.OrderedDict()
    kind = cfg["kind"]
    C = cfg["channels"]
    if kind in ("vit", "deepvit", "parallel_vit"):
        dim = cfg["dim"]
        pd = cfg["patch_h"] * cfg["patch_w"] * C
        specs["pos_embedding"] = ((1, cfg["num_patches"] + 1, dim), "normal")
        specs["cls_token"] = ((1, 1, dim), "normal")
        _dense(specs, "patch", pd, dim)
        for L in range(cfg["depth"]):
            if kind == "parallel_vit":
                # branch i = (Parallel attention fn i, Parallel feed-forward fn i) of layer L (parallel_vit.py:109-112):
                # Keras path model.transformer.layers[L][0].fns[i] / [L][1].fns[i]
                for i in range(cfg["num_parallel_branches"]):
                    _vit_layer(specs, f"layers.{L}.branch{i}.", dim, cfg["heads"], cfg["dim_head"], cfg["mlp_dim"], kind="vit")
            else:
                _vit_layer(specs, f"layers.{L}.", dim, cfg["heads"], cfg["dim_head"], cfg["mlp_dim"], kind=kind)
        _ln(specs, "head_norm", dim)
        _dense(specs, "head", dim, cfg["num_classes"])
    elif kind == "cait":
        dim = cfg["dim"]
        pd = cfg["patch_h"] * cfg["patch_w"] * C
        specs["pos_embedding"] = ((1, cfg["num_patches"], dim), "normal")  # cait.py:168 (no +1)
        specs["cls_token"] = ((1, 1, dim), "normal")
        _dense(specs, "patch", pd, dim)
        for stack, depth in (("patch_transformer", cfg["depth"]), ("cls_transformer", cfg["cls_depth"])):
            for L in range(depth):
                pre = f"{stack}.layers.{L}."
                specs[pre + "attn_scale"] = ((1, 1, dim), ("fill", _layerscale_eps(L + 1)))
                specs[pre + "ff_scale"] = ((1, 1, dim), ("fill", _layerscale_eps(L + 1)))
                _vit_layer(specs, pre, dim, cfg["heads"], cfg["dim_head"], cfg["mlp_dim"], kind="cait")
        _ln(specs, "head_norm", dim)
        _dense(specs, "head", dim, cfg["num_classes"])
    elif kind == "patch_merger_vit":
        dim = cfg["dim"]
        pd = cfg["patch_h"] * cfg["patch_w"] * C
        specs["pos_embedding"] = ((1, cfg["num_patches"] + 1, dim), "normal")   # vit_with_patch_merger.py:163 (only [:n] is used, :178)
        _dense(specs, "patch", pd, dim)
        for L in range(cfg["depth"]):
            _vit_layer(specs, f"layers.{L}.", dim, cfg["heads"], cfg["dim_head"], cfg["mlp_dim"], kind="vit")
        _ln(specs, "patch_merger.norm", dim)                                       # :46
        specs["patch_merger.queries"] = ((cfg["patch_merge_num_tokens"], dim), "normal")   # :47
        _ln(specs, "head_norm", dim)
        _dense(specs, "head", dim, cfg["num_classes"])
    elif kind == "t2t_vit":
        dim = cfg["dim"]
        dims = cfg["t2t_dims"]
        for i, d in enumerate(dims[:-1]):
            # RearrangeUnfoldTransformer's Transformer(dim=d, heads=1, depth=1, dim_head=d, mlp_dim=d) (t2t.py:69-70,35):
            # heads == 1 and dim_head == dim -> no out-projection (vit.py:53)
            _vit_layer(specs, f"t2t.{i}.layers.0.", d, 1, d, d, kind="vit")
        _dense(specs, "patch", dims[-1], dim)                                      # t2t.py:73
        specs["pos_embedding"] = ((1, cfg["num_patches"] + 1, dim), "normal")      # :76
        specs["cls_token"] = ((1, 1, dim), "normal")                               # :77
        for L in range(cfg["depth"]):
            _vit_layer(specs, f"layers.{L}.", dim, cfg["heads"], cfg["dim_head"], cfg["mlp_dim"], kind="vit")
        _ln(specs, "head_norm", dim)
        _dense(specs, "head", dim, cfg["num_classes"])
    elif kind == "crossvit":
        s = cfg["image_size"]
        for br in ("sm", "lg"):
            dim, p = cfg[f"{br}_dim"], cfg[f"{br}_patch_size"]
            n_p = (s // p) ** 2
            _dense(specs, f"{br}_embed.patch", p * p * C, dim)
            specs[f"{br}_embed.pos_embedding"] = ((1, n_p + 1, dim), "normal")
            specs[f"{br}_embed.cls_token"] = ((1, 1, dim), "normal")
        for D in range(cfg["depth"]):
            for br in ("sm", "lg"):
                dim = cfg[f"{br}_dim"]
                for L in range(cfg[f"{br}_enc_depth"]):
                    _vit_layer(specs, f"blocks.{D}.{br}_enc.layers.{L}.", dim, cfg[f"{br}_enc_heads"],
                               cfg[f"{br}_enc_dim_head"], cfg[f"{br}_enc_mlp_dim"], kind="crossvit")
                _ln(specs, f"blocks.{D}.{br}_enc.final_norm", dim)  # cross_vit.py:100,113
            for R in range(cfg["cross_attn_depth"]):
                # cross_vit.py:148-149: ProjectInOut(dim_in, dim_out, PreNorm(Attention(dim_out)))
                for name, din, dout in ((f"blocks.{D}.cross.{R}.sm_attend_lg.", cfg["sm_dim"], cfg["lg_dim"]),
                                        (f"blocks.{D}.cross.{R}.lg_attend_sm.", cfg["lg_dim"], cfg["sm_dim"])):
                    if din != dout:
                        _dense(specs, name + "project_in", din, dout)
                        _dense(specs, name + "project_out", dout, din)
                    _ln(specs, name + "norm", dout)
                    inner = cfg["cross_attn_heads"] * cfg["cross_attn_dim_head"]
                    _dense(specs, name + "to_q", dout, inner, bias=False)
                    _dense(specs, name + "to_kv", dout, 2 * inner, bias=False)
                    _dense(specs, name + "to_out", inner, dout)
        for br in ("sm", "lg"):
            _ln(specs, f"{br}_head_norm", cfg[f"{br}_dim"])
            _dense(specs, f"{br}_head", cfg[f"{br}_dim"], cfg["num_classes"])
    return specs


def init_weights(cfg: dict, seed: int = 0) -> "collections.OrderedDict[str, np.ndarray]":
    """The reference's init distributions (Dense glorot-uniform / zeros, LN ones/zeros,
    tf.random.normal Variables N(0,1), LayerScale fill) from a seeded numpy generator."""
    rng = np.random.default_rng(seed)
    out = collections.OrderedDict()
    for name, (shape, init) in weight_specs(cfg).items():
        if init == "glorot":
            lim = np.sqrt(6.0 / (shape[0] + shape[1]))
            w = rng.uniform(-lim, lim, size=shape)
        elif init == "zeros":
            w = np.zeros(shape)
        elif init == "ones":
            w = np.ones(shape)
        elif init == "normal":
            w = rng.standard_normal(shape)
        elif isinstance(init, tuple) and init[0] == "fill":
            w = np.full(shape, init[1])
        else:
            raise AssertionError(init)
        out[name] = np.ascontiguousarray(w, dtype=np.float32)
    return out


def stress_weights(cfg: dict, seed: int = 1) -> "collections.OrderedDict[str, np.ndarray]":
    """Like init_weights but with non-zero biases, non-unit LN gamma/beta and O(1) LayerScale,
    so that bias / affine / scale wiring bugs cannot hide behind the Keras defaults."""
    rng = np.random.default_rng(seed)
    out = init_weights(cfg, seed)
    for name, (shape, init) in weight_specs(cfg).items():
        if init == "zeros":
            out[name] = (0.2 * rng.standard_normal(shape)).astype(np.float32)
        elif init == "ones":
            out[name] = (1.0 + 0.2 * rng.standard_normal(shape)).astype(np.float32)
        elif isinstance(init, tuple) and init[0] == "fill":
            out[name] = (0.5 + 0.5 * rng.uniform(size=shape)).astype(np.float32)
    return out


def make_image(cfg: dict, batch: int, seed: int = 0, h: int | None = None, w: int | None = None) -> np.ndarray:
    """Synthetic NHWC float32 image batch."""
    rng = np.random.default_rng(seed)
    h = cfg["image_h"] if h is None else h
    w = cfg["image_w"] if w is None else w
    return rng.standard_normal((batch, h, w, cfg["channels"]), dtype=np.float32)


# ----------------------------------------------------------------------------- FLOPs
def _layer_flops(nq, nk, dim, heads, dim_head, mlp_dim, *, mixes=0, project_out=True):
    inner = heads * dim_head
    f = 2 * nq * dim * inner + 2 * nk * dim * 2 * inner      # q + kv projections
    f += 2 * 2 * heads * nq * nk * dim_head                   # QK^T and PV
    f += mixes * 2 * nq * nk * heads * heads                  # head-mix einsums
    if project_out:
        f += 2 * nq * inner * dim
    f += 4 * nq * dim * mlp_dim
    return f


def flops_per_image(cfg: dict) -> float:
    """Algorithmic FLOPs (2*MAC over every matmul at the true n), SURVEY.md App. C."""
    kind = cfg["kind"]
    C = cfg["channels"]
    if kind in ("vit", "deepvit", "parallel_vit"):
        n_p, dim = cfg["num_patches"], cfg["dim"]
        n = n_p + 1
        f = 2 * n_p * cfg["patch_h"] * cfg["patch_w"] * C * dim
        po = not (kind != "deepvit" and cfg["heads"] == 1 and cfg["dim_head"] == dim)
        f += cfg["depth"] * cfg.get("num_parallel_branches", 1) * _layer_flops(n, n, dim, cfg["heads"], cfg["dim_head"], cfg["mlp_dim"],
                                         mixes=1 if kind == "deepvit" else 0, project_out=po)
        f += 2 * dim * cfg["num_classes"]
        return float(f)
    if kind == "cait":
        n_p, dim = cfg["num_patches"], cfg["dim"]
        f = 2 * n_p * cfg["patch_h"] * cfg["patch_w"] * C * dim
        f += cfg["depth"] * _layer_flops(n_p, n_p, dim, cfg["heads"], cfg["dim_head"], cfg["mlp_dim"], mixes=2)
        f += cfg["cls_depth"] * _layer_flops(1, n_p + 1, dim, cfg["heads"], cfg["dim_head"], cfg["mlp_dim"], mixes=2)
        f += 2 * dim * cfg["num_classes"]
        return float(f)
    if kind == "patch_merger_vit":
        n, dim = cfg["num_patches"], cfg["dim"]
        f = 2 * n * cfg["patch_h"] * cfg["patch_w"] * C * dim
        po = not (cfg["heads"] == 1 and cfg["dim_head"] == dim)
        for L in range(cfg["depth"]):
            f += _layer_flops(n, n, dim, cfg["heads"], cfg["dim_head"], cfg["mlp_dim"], project_out=po)
            if L == cfg["patch_merge_layer_index"]:
                f += 4 * cfg["patch_merge_num_tokens"] * n * dim               # queries . x^T and attn . x
                n = cfg["patch_merge_num_tokens"]
        f += 2 * dim * cfg["num_classes"]
        return float(f)
    if kind == "t2t_vit":
        f = 0
        grids = t2t_token_grid(cfg)
        for i, d in enumerate(cfg["t2t_dims"][:-1]):
            n = grids[i][0] * grids[i][1]
            f += _layer_flops(n, n, d, 1, d, d, project_out=False)
        n_p, dim = grids[-1][0] * grids[-1][1], cfg["dim"]
        f += 2 * n_p * cfg["t2t_dims"][-1] * dim
        po = not (cfg["heads"] == 1 and cfg["dim_head"] == dim)
        f += cfg["depth"] * _layer_flops(n_p + 1, n_p + 1, dim, cfg["heads"], cfg["dim_head"], cfg["mlp_dim"], project_out=po)
        f += 2 * dim * cfg["num_classes"]
        return float(f)
    if kind == "crossvit":
        s = cfg["image_size"]
        f = 0
        n = {}
        for br in ("sm", "lg"):
            p, dim = cfg[f"{br}_patch_size"], cfg[f"{br}_dim"]
            n[br] = (s // p) ** 2 + 1
            f += 2 * (n[br] - 1) * p * p * C * dim
        for _ in range(cfg["depth"]):
            for br in ("sm", "lg"):
                f += cfg[f"{br}_enc_depth"] * _layer_flops(n[br], n[br], cfg[f"{br}_dim"], cfg[f"{br}_enc_heads"],
                                                          cfg[f"{br}_enc_dim_head"], cfg[f"{br}_enc_mlp_dim"])
            inner = cfg["cross_attn_heads"] * cfg["cross_attn_dim_head"]
            for din, dout, nk in ((cfg["sm_dim"], cfg["lg_dim"], n["lg"]), (cfg["lg_dim"], cfg["sm_dim"], n["sm"])):
                g = 0
                if din != dout:
                    g += 2 * din * dout * 2
                g += 2 * dout * inner + 2 * nk * dout * 2 * inner + 4 * cfg["cross_attn_heads"] * nk * cfg["cross_attn_dim_head"]
                g += 2 * inner * dout
                f += cfg["cross_attn_depth"] * g
        f += 2 * (cfg["sm_dim"] + cfg["lg_dim"]) * cfg["num_classes"]
        return float(f)
    raise ValueError(kind)

"""Host-side mirror of the reference's model classes over the libvitb200 C-ABI.

    ViT       vit_tensorflow/vit.py:106-177          DeepViT   vit_tensorflow/deepvit.py:112-157
    CaiT      vit_tensorflow/cait.py:155-194         CrossViT  vit_tensorflow/cross_vit.py:232-303
    parallel_vit.ViT  parallel_vit.py:120-185        DistillableViT  distill.py:47-58 (forward)
    T2TViT    vit_tensorflow/t2t.py:50-116           vit_with_patch_merger.ViT / PatchMerger  vit_with_patch_merger.py:42-55,134-185
    efficient.ViT  vit_tensorflow/efficient.py:12-55 (injected transformer between the engine's embed and head stages)
    CvT       vit_tensorflow/cvt.py:149-202
    TwinsSVT  vit_tensorflow/twins_svt.py:215-268
    CrossFormer  vit_tensorflow/crossformer.py:205-269

Same constructor kwargs, defaults and assertion messages; `model(img, training=True, **kwargs) -> logits`
with `img` NHWC float32 `[b, H, W, 3]` and logits float32 `[b, num_classes]`.  Everything below the call is
hand-written sm_90a CUDA behind `include/vitb200.h`; this file only validates arguments, owns the weight dict
(Keras layouts, SURVEY.md App. B) and marshals pointers.  Two extra keyword-only constructor arguments that the
reference does not have: `precision` ("bf16" tensor-core path, default; "fp32" exact gate path) and `device`.

Semantics notes (SURVEY.md App. D): inference only -- dropout is the identity, so a non-zero
dropout / emb_dropout / layer_dropout with `training=True` (the reference's default!) cannot be reproduced and
raises unless `training=False` is passed (CaiT's layer_dropout is active even then in the reference,
cait.py:147, so it must be 0).
"""
from __future__ import annotations

import collections
import ctypes as C

import numpy as np

from . import _lib


def pair(t):  # vit.py:11
    return t if isinstance(t, tuple) else (t, t)


def _layerscale_eps(depth):  # cait.py:36-41
    if depth <= 18:
        return 0.1
    if depth <= 24:
        return 1e-5
    return 1e-6


class _Array(np.ndarray):
    """What the host classes hand back: a float32 numpy array that also answers `.numpy()`.  The reference's outputs are eager
    TensorFlow tensors and its wrappers call `.numpy()` on them and on anything derived from them -- `tokens.numpy()[batch_range,
    unmasked_indices]` (mae.py:63), `encoded.numpy()[batch_range, masked_indices]`, `patches.numpy()` (simmim.py:119,125) -- so a
    plain ndarray would break those wrappers; arithmetic on an `_Array` yields an `_Array`, so derived values keep the method."""

    def numpy(self):
        return self.view(np.ndarray)

    def __array_wrap__(self, obj, context=None, return_scalar=False):
        out = super().__array_wrap__(obj, context, return_scalar)
        return out[()] if isinstance(out, np.ndarray) and out.ndim == 0 else out    # reductions give numpy scalars, as on ndarray


def _as_tensor(a):
    return a.view(_Array)


class _Transformer:
    """`model.transformer(tokens)` (vit.py:99-104): the entry the reference's wrappers call with any n."""

    def __init__(self, model):
        self._m = model

    def __call__(self, x, training=True):
        return self._m.forward_tokens(x)


class _Layer:
    """A callable standing where the reference has a Keras layer (`patch_embedding.layers[i]`, `mlp_head`, `dropout`)."""

    def __init__(self, fn):
        self._fn = fn

    def __call__(self, x, training=True):
        return self._fn(x)


class _DenseLayer(_Layer):
    """Stands where the reference has an `nn.Dense`: callable, plus the Keras variable list the wrappers read the patch
    size from -- `patch_to_emb.weights[0].shape[0]` (mae.py:38, simmim.py:80).  `weights` = [kernel [in, units], bias [units]]
    as read-only views of the arrays the model holds (assign through `set_weights_dict`)."""

    def __init__(self, fn, model, name):
        super().__init__(fn)
        self._m, self._name = model, name

    @property
    def kernel(self):
        return self._m._weight_view(self._name + ".kernel")

    @property
    def bias(self):
        return self._m._weight_view(self._name + ".bias")

    @property
    def weights(self):
        return [self.kernel, self.bias]

    def get_weights(self):
        return [w.copy() for w in self.weights]


class _PatchEmbedding(_Layer):
    """`model.patch_embedding` (vit.py:141-144): Sequential([Rearrange, Dense]); the wrappers take `.layers[:2]` apart
    (mae.py:37, simmim.py:79) or call `.layers[-1]` (mpp.py:200)."""

    def __init__(self, model):
        super().__init__(model.forward_patch_embedding)
        self.layers = [_Layer(model.to_patch), _DenseLayer(model.patch_to_emb, model, "patch")]


class _EngineModel:
    """Common machinery: engine handle, weight dict, forward call."""

    _kind = None

    def _create(self, precision, device, **cfgkw):
        self.precision = precision
        self.device = int(device)
        cfg = _lib.VbConfig()
        cfg.struct_size = C.sizeof(_lib.VbConfig)
        cfg.kind = _lib.KIND[self._kind]
        if precision not in _lib.PRECISION:
            raise ValueError(f"precision must be one of {sorted(_lib.PRECISION)}")
        cfg.precision = _lib.PRECISION[precision]
        cfg.channels = 3
        for k, v in cfgkw.items():
            setattr(cfg, k, int(v))
        self._cfg = cfg
        self._lib = _lib.load()
        h = C.c_void_p()
        _lib.check(self._lib.vb_create(C.byref(cfg), self.device, C.byref(h)))
        self._h = h
        self._finalized = False
        self._specs = collections.OrderedDict()
        name, shape, ndim = C.c_char_p(), (C.c_int64 * 4)(), C.c_int32()
        for i in range(self._lib.vb_num_weights(h)):
            _lib.check(self._lib.vb_weight_info(h, i, C.byref(name), shape, C.byref(ndim)), h)
            self._specs[name.value.decode()] = tuple(int(shape[j]) for j in range(ndim.value))
        self._weights = collections.OrderedDict()

    # ---- weights -------------------------------------------------------------------------------------
    def weight_specs(self):
        return collections.OrderedDict(self._specs)

    def init_weights(self, seed=None):
        """The reference's initial distributions: Dense glorot-uniform / zero bias (Keras defaults),
        LayerNormalization ones/zeros, tf.random.normal Variables N(0,1) (vit.py:146-147, deepvit.py:57,
        cait.py:97-98), LayerScale fill (cait.py:36-44)."""
        rng = np.random.default_rng(seed)
        w = collections.OrderedDict()
        for name, shape in self._specs.items():
            leaf = name.rsplit(".", 1)[-1]
            if leaf == "kernel":
                receptive = int(np.prod(shape[:-2]))          # Conv2D kernel [k, k, cin, cout]: fans count the window (1 for Dense)
                lim = np.sqrt(6.0 / (receptive * (shape[-2] + shape[-1])))
                a = rng.uniform(-lim, lim, size=shape)
            elif leaf in ("bias", "beta"):
                a = np.zeros(shape)
            elif leaf == "gamma":
                a = np.ones(shape)
            elif leaf in ("attn_scale", "ff_scale"):
                layer = int(name.split(".layers.")[1].split(".")[0])
                a = np.full(shape, _layerscale_eps(layer + 1))
            elif leaf == "positional_emb":                   # CCT cct.py:251-254
                a = (sinusoidal_embedding(shape[1], shape[2]) if self._positional_embedding == "sine"
                     else _truncated_normal(rng, shape, 0.2))
            else:  # pos_embedding, cls_token, reattn_weights, mix_pre, mix_post
                a = rng.standard_normal(shape)
            w[name] = a.astype(np.float32)
        self.set_weights_dict(w)

    def set_weights_dict(self, weights):
        """weights: mapping name -> array in the Keras layout (SURVEY.md App. B).  Missing names keep their value."""
        for name, arr in weights.items():
            if name not in self._specs:
                raise KeyError(f"{type(self).__name__} has no weight named {name!r}")
            a = np.ascontiguousarray(arr, dtype=np.float32)
            if tuple(a.shape) != self._specs[name]:
                raise ValueError(f"weight {name!r}: expected shape {self._specs[name]}, got {tuple(a.shape)}")
            shape = (C.c_int64 * a.ndim)(*a.shape)
            _lib.check(self._lib.vb_set_weight(self._h, name.encode(), a.ctypes.data_as(C.c_void_p), shape, a.ndim), self._h)
            self._weights[name] = a
        self._finalized = False

    def get_weights_dict(self):
        return collections.OrderedDict((k, v.copy()) for k, v in self._weights.items())

    def get_weight(self, name):
        return self._weights[name]

    # `model.pos_embedding` / `model.cls_token` as the reference's wrappers use them: `.shape` (mae.py:33), slicing
    # `encoder.pos_embedding[:, 1:(n + 1)]` (mae.py:54, simmim.py:95), `pos_embedding[:, :(n + 1)]` (mpp.py:208), einops
    # `repeat(transformer.cls_token, ...)` (mpp.py:204) and arithmetic with token arrays: the float32 numpy array the model
    # currently holds for that weight (read-only view; assign through set_weights_dict).
    def _weight_view(self, name):
        if name not in self._specs:
            raise AttributeError(f"{type(self).__name__} has no weight '{name}'")
        a = self._weights[name].view()
        a.flags.writeable = False
        return a.view(_Array)

    @property
    def pos_embedding(self):
        return self._weight_view("pos_embedding")

    @property
    def cls_token(self):
        return self._weight_view("cls_token")

    def load_weights(self, path):
        with np.load(path) as z:
            self.set_weights_dict({k: z[k] for k in z.files})

    def save_weights(self, path):
        np.savez(path, **self._weights)

    def _finalize(self):
        if not self._finalized:
            _lib.check(self._lib.vb_finalize(self._h), self._h)
            self._finalized = True

    def build(self, input_shape=None):  # Keras API used by mae.py:32; weights exist from construction here
        self._finalize()

    # ---- forward ------------------------------------------------------------------------------------
    def _check_training(self, training):
        if training and any(r != 0 for r in self._dropout_rates):
            raise NotImplementedError(
                "libvitb200 implements inference semantics: stochastic dropout (rate > 0 with training=True, the "
                "reference's default) is not reproducible; pass training=False or construct with dropout = 0")

    def __call__(self, img, training=True, **kwargs):
        """Reference call surface (vit.py:159): numpy NHWC float image batch -> numpy float32 logits."""
        self._check_training(training)
        x = np.ascontiguousarray(img, dtype=np.float32)
        if x.ndim != 4 or x.shape[3] != 3:
            raise ValueError("img must be NHWC float [b, H, W, 3]")
        b, h, w, _ = x.shape
        out = np.empty((b, self.num_classes), np.float32)
        self.forward_raw(x.ctypes.data, _lib.MEM_HOST, b, h, w, out.ctypes.data, _lib.MEM_HOST, None)
        return _as_tensor(out)

    call = __call__

    def forward_raw(self, img_ptr, img_mem, batch, h, w, logits_ptr, logits_mem, stream=None):
        """Pointer-level forward: host or device (e.g. torch tensor .data_ptr()) buffers, optional cudaStream_t."""
        self._finalize()
        _lib.check(self._lib.vb_forward(self._h, C.c_void_p(img_ptr), img_mem, batch, h, w, C.c_void_p(logits_ptr), logits_mem,
                                        C.c_void_p(stream) if stream else None), self._h)

    def forward_tokens(self, tokens):
        self._finalize()
        x = np.ascontiguousarray(tokens, dtype=np.float32)
        if x.ndim != 3 or x.shape[2] != self._cfg.dim:
            raise ValueError(f"transformer(tokens): expected [batch, n, {self._cfg.dim}] tokens, got {x.shape}")
        b, n, _ = x.shape
        out = np.empty_like(x)
        _lib.check(self._lib.vb_forward_tokens(self._h, x.ctypes.data_as(C.c_void_p), _lib.MEM_HOST, b, n,
                                               out.ctypes.data_as(C.c_void_p), _lib.MEM_HOST, None), self._h)
        return _as_tensor(out)

    # ---- the stages of `call` on their own (SURVEY.md 8f f1/f4) ------------------------------------------
    def _img(self, img):
        x = np.ascontiguousarray(img, dtype=np.float32)
        if x.ndim != 4 or x.shape[3] != 3:
            raise ValueError("img must be NHWC float [b, H, W, 3]")
        return x

    def forward_embed(self, img):
        """`call` up to the transformer (vit.py:160-166): patch embedding, cls token, positions -> [b, rows, dim]."""
        self._finalize()
        x = self._img(img)
        b, h, w, _ = x.shape
        rows = self._lib.vb_embed_rows(self._h, h, w)
        if rows < 0:
            _lib.check(-rows, self._h)
        out = np.empty((b, rows, self._cfg.dim), np.float32)
        _lib.check(self._lib.vb_forward_embed(self._h, x.ctypes.data_as(C.c_void_p), _lib.MEM_HOST, b, h, w,
                                              out.ctypes.data_as(C.c_void_p), _lib.MEM_HOST, None), self._h)
        return _as_tensor(out)

    def forward_head(self, tokens):
        """`call` after the transformer (vit.py:170-175): pooling + mlp_head; [b, n, dim] (or [b, dim]) -> logits."""
        self._finalize()
        x = np.ascontiguousarray(tokens, dtype=np.float32)
        if x.ndim == 2:
            x = x[:, None, :]
        b, n, d = x.shape
        if d != self._cfg.dim:
            raise ValueError(f"tokens must have last dimension {self._cfg.dim}")
        out = np.empty((b, self.num_classes), np.float32)
        _lib.check(self._lib.vb_forward_head(self._h, x.ctypes.data_as(C.c_void_p), _lib.MEM_HOST, b, n,
                                             out.ctypes.data_as(C.c_void_p), _lib.MEM_HOST, None), self._h)
        return _as_tensor(out)

    def to_patch(self, img):
        """`patch_embedding.layers[0]`: Rearrange('b (h p1) (w p2) c -> b (h w) (p1 p2 c)') (vit.py:142)."""
        x = self._img(img)
        b, h, w, c = x.shape
        ph, pw = self._cfg.patch_h, self._cfg.patch_w
        if ph <= 0 or pw <= 0 or h % ph or w % pw:
            raise ValueError("Image dimensions must be divisible by the patch size.")
        out = np.empty((b, (h // ph) * (w // pw), ph * pw * c), np.float32)
        _lib.check(self._lib.vb_to_patch(self._h, x.ctypes.data_as(C.c_void_p), _lib.MEM_HOST, b, h, w,
                                         out.ctypes.data_as(C.c_void_p), _lib.MEM_HOST, None), self._h)
        return _as_tensor(out)

    def patch_to_emb(self, patches):
        """`patch_embedding.layers[1]`: the Dense(dim) on patch vectors [..., patch_dim] (vit.py:143)."""
        self._finalize()
        x = np.ascontiguousarray(patches, dtype=np.float32)
        pd = self._specs["patch.kernel"][0]
        if x.shape[-1] != pd:
            raise ValueError(f"patches must have last dimension {pd}")
        rows = int(np.prod(x.shape[:-1]))
        out = np.empty(x.shape[:-1] + (self._cfg.dim,), np.float32)
        _lib.check(self._lib.vb_patch_to_emb(self._h, x.ctypes.data_as(C.c_void_p), _lib.MEM_HOST, rows,
                                             out.ctypes.data_as(C.c_void_p), _lib.MEM_HOST, None), self._h)
        return _as_tensor(out)

    def forward_patch_embedding(self, img):
        """`model.patch_embedding(img)` (vit.py:160)."""
        if self._kind == "t2t_vit":
            raise NotImplementedError("T2TViT: the tokens-to-token module runs inside forward_embed(img) (with cls token and "
                                      "positions); only patch_embedding.layers[-1] (the Dense) is exposed separately")
        return self.patch_to_emb(self.to_patch(img))

    def _attach_stage_attributes(self):
        """The attribute surface the reference's wrappers use (SURVEY.md 3.5): patch_embedding(.layers), pos_embedding,
        cls_token, dropout, mlp_head."""
        self.patch_embedding = _PatchEmbedding(self)
        self.dropout = _Layer(lambda x: x)               # inference semantics: identity (vit.py:148,166)
        self.mlp_head = _Layer(self.forward_head)

    PROFILE_CLASSES = ("gemm_wgmma", "attention", "layernorm", "im2col", "other", "gemm_wgmma_gelu", "gemm_wgmma_residual")

    def profile(self, on=True):
        """Record CUDA events around every kernel class on the launch stream (for the roofline report)."""
        _lib.check(self._lib.vb_profile_enable(self._h, int(bool(on))), self._h)

    def profile_read(self, reset=True):
        n = len(self.PROFILE_CLASSES)
        ms, fl, by, calls = (C.c_double * n)(), (C.c_double * n)(), (C.c_double * n)(), (C.c_int64 * n)()
        _lib.check(self._lib.vb_profile_read(self._h, ms, fl, by, calls, int(bool(reset))), self._h)
        return {c: dict(ms=ms[i], flops=fl[i], bytes=by[i], launches=int(calls[i])) for i, c in enumerate(self.PROFILE_CLASSES)}

    @property
    def last_launch_count(self):
        return int(self._lib.vb_last_launch_count(self._h))

    def graph_stats(self):
        """CUDA-graph activity of `forward_raw` on a stream (vb_graph_stats), cumulative: captures, replays, failed captures and
        the reason of the last failure ("" if none)."""
        cap, rep, fail, why = C.c_int64(), C.c_int64(), C.c_int64(), C.c_char_p()
        _lib.check(self._lib.vb_graph_stats(self._h, C.byref(cap), C.byref(rep), C.byref(fail), C.byref(why)), self._h)
        return dict(captures=cap.value, replays=rep.value, failures=fail.value, last_failure=(why.value or b"").decode())

    def close(self):
        h, self._h = getattr(self, "_h", None), None
        if h:
            self._lib.vb_destroy(h)

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class ViT(_EngineModel):
    """vit.py:106-177."""
    _kind = "vit"

    def __init__(self, image_size, patch_size, num_classes, dim, depth, heads, mlp_dim,
                 pool='cls', dim_head=64, dropout=0.0, emb_dropout=0.0, *, precision="bf16", device=0, seed=None):
        image_height, image_width = pair(image_size)
        patch_height, patch_width = pair(patch_size)
        assert image_height % patch_height == 0 and image_width % patch_width == 0, 'Image dimensions must be divisible by the patch size.'
        assert pool in {'cls', 'mean'}, 'pool type must be either cls (cls token) or mean (mean pooling)'
        self.num_classes, self.pool, self.dim = num_classes, pool, dim
        self._dropout_rates = (dropout, emb_dropout)
        self._create(precision, device, image_h=image_height, image_w=image_width, patch_h=patch_height, patch_w=patch_width,
                     num_classes=num_classes, dim=dim, depth=depth, heads=heads, dim_head=dim_head, mlp_dim=mlp_dim,
                     pool=0 if pool == 'cls' else 1)
        self.init_weights(seed)
        # attribute surface used by the reference's wrappers (SURVEY.md section 3.5)
        self._attach_stage_attributes()
        self.transformer = _Transformer(self)


class ParallelViT(_EngineModel):
    """parallel_vit.py:120-185 (`parallel_vit.ViT`): every layer sums `num_parallel_branches` attention blocks and then as
    many feed-forward blocks, each behind its own LayerNorm (Parallel parallel_vit.py:36-42, Transformer :99-117)."""
    _kind = "parallel_vit"

    def __init__(self, image_size, patch_size, num_classes, dim, depth, heads, mlp_dim, pool='cls', num_parallel_branches=2,
                 dim_head=64, dropout=0.0, emb_dropout=0.0, *, precision="bf16", device=0, seed=None):
        image_height, image_width = pair(image_size)
        patch_height, patch_width = pair(patch_size)
        assert image_height % patch_height == 0 and image_width % patch_width == 0, 'Image dimensions must be divisible by the patch size.'
        assert pool in {'cls', 'mean'}, 'pool type must be either cls (cls token) or mean (mean pooling)'
        self.num_classes, self.pool, self.dim = num_classes, pool, dim
        self._dropout_rates = (dropout, emb_dropout)
        self._create(precision, device, image_h=image_height, image_w=image_width, patch_h=patch_height, patch_w=patch_width,
                     num_classes=num_classes, dim=dim, depth=depth, heads=heads, dim_head=dim_head, mlp_dim=mlp_dim,
                     pool=0 if pool == 'cls' else 1, parallel_branches=num_parallel_branches)
        self.init_weights(seed)
        self._attach_stage_attributes()


class DistillableViT(ViT):
    """distill.py:47-58 (DistillMixin.call distill.py:16-45): a ViT whose call takes an optional distillation token
    `[1, 1, dim]`; with it the call returns `(logits, distill_tokens [b, dim])`, without it plain ViT logits.
    Forward only -- DistillWrapper's losses (distill.py:100-170) stay with the caller."""

    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self.args, self.kwargs = args, kwargs
        self.dim, self.num_classes = kwargs["dim"], kwargs["num_classes"]

    def __call__(self, img, distill_token=None, training=True):
        if distill_token is None:
            return super().__call__(img, training=training)
        self._check_training(training)
        self._finalize()
        x = np.ascontiguousarray(img, dtype=np.float32)
        if x.ndim != 4 or x.shape[3] != 3:
            raise ValueError("img must be NHWC float [b, H, W, 3]")
        tok = np.ascontiguousarray(distill_token, dtype=np.float32).reshape(-1)
        if tok.size != self.dim:
            raise ValueError(f"distill_token must hold dim = {self.dim} values, got shape {np.shape(distill_token)}")
        b, h, w, _ = x.shape
        logits = np.empty((b, self.num_classes), np.float32)
        dist = np.empty((b, self.dim), np.float32)
        _lib.check(self._lib.vb_forward_distill(self._h, x.ctypes.data_as(C.c_void_p), _lib.MEM_HOST, b, h, w,
                                                tok.ctypes.data_as(C.c_void_p), logits.ctypes.data_as(C.c_void_p),
                                                dist.ctypes.data_as(C.c_void_p), _lib.MEM_HOST, None), self._h)
        return _as_tensor(logits), _as_tensor(dist)

    call = __call__


class DeepViT(ViT):
    """deepvit.py:112-157 (integer image/patch sizes only, :117-118)."""
    _kind = "deepvit"

    def __init__(self, image_size, patch_size, num_classes, dim, depth, heads, mlp_dim,
                 pool='cls', dim_head=64, dropout=0.0, emb_dropout=0.0, *, precision="bf16", device=0, seed=None):
        assert image_size % patch_size == 0, 'Image dimensions must be divisible by the patch size.'
        super().__init__(image_size, patch_size, num_classes, dim, depth, heads, mlp_dim, pool, dim_head, dropout,
                         emb_dropout, precision=precision, device=device, seed=seed)


class CaiT(_EngineModel):
    """cait.py:155-194."""
    _kind = "cait"

    def __init__(self, image_size, patch_size, num_classes, dim, depth, cls_depth, heads, mlp_dim,
                 dim_head=64, dropout=0.0, emb_dropout=0.0, layer_dropout=0.0, *, precision="bf16", device=0, seed=None):
        assert image_size % patch_size == 0, 'Image dimensions must be divisible by the patch size.'
        if layer_dropout != 0:
            raise NotImplementedError("layer_dropout drops layers even at inference in the reference (cait.py:147); "
                                      "parity is only defined for layer_dropout = 0")
        self.num_classes, self.dim = num_classes, dim
        self._dropout_rates = (dropout, emb_dropout)
        self._create(precision, device, image_h=image_size, image_w=image_size, patch_h=patch_size, patch_w=patch_size,
                     num_classes=num_classes, dim=dim, depth=depth, cls_depth=cls_depth, heads=heads, dim_head=dim_head,
                     mlp_dim=mlp_dim)
        self.init_weights(seed)
        self._attach_stage_attributes()


class CrossViT(_EngineModel):
    """cross_vit.py:232-303."""
    _kind = "crossvit"

    def __init__(self, image_size, num_classes, sm_dim, lg_dim, sm_patch_size=12, sm_enc_depth=1, sm_enc_heads=8,
                 sm_enc_mlp_dim=2048, sm_enc_dim_head=64, lg_patch_size=16, lg_enc_depth=4, lg_enc_heads=8,
                 lg_enc_mlp_dim=2048, lg_enc_dim_head=64, cross_attn_depth=2, cross_attn_heads=8, cross_attn_dim_head=64,
                 depth=3, dropout=0.1, emb_dropout=0.1, *, precision="bf16", device=0, seed=None):
        assert image_size % sm_patch_size == 0, 'Image dimensions must be divisible by the patch size.'
        assert image_size % lg_patch_size == 0, 'Image dimensions must be divisible by the patch size.'
        self.num_classes = num_classes
        self._dropout_rates = (dropout, emb_dropout)
        self._create(precision, device, image_h=image_size, image_w=image_size, num_classes=num_classes, sm_dim=sm_dim,
                     lg_dim=lg_dim, sm_patch_size=sm_patch_size, sm_enc_depth=sm_enc_depth, sm_enc_heads=sm_enc_heads,
                     sm_enc_mlp_dim=sm_enc_mlp_dim, sm_enc_dim_head=sm_enc_dim_head, lg_patch_size=lg_patch_size,
                     lg_enc_depth=lg_enc_depth, lg_enc_heads=lg_enc_heads, lg_enc_mlp_dim=lg_enc_mlp_dim,
                     lg_enc_dim_head=lg_enc_dim_head, cross_attn_depth=cross_attn_depth, cross_attn_heads=cross_attn_heads,
                     cross_attn_dim_head=cross_attn_dim_head, cross_depth=depth)
        self.init_weights(seed)


class T2TViT(_EngineModel):
    """t2t.py:50-116.  `transformer=` injection (t2t.py:82-86): pass any callable over [b, n, dim] numpy tokens (e.g. another
    engine model's `.transformer`); then depth / heads / mlp_dim may be omitted and the engine runs the tokens-to-token
    module and the head around it."""
    _kind = "t2t_vit"

    def __init__(self, image_size, num_classes, dim, depth=None, heads=None, mlp_dim=None, pool='cls', channels=3, dim_head=64,
                 dropout=0.0, emb_dropout=0.0, transformer=None, t2t_layers=((7, 4), (3, 2), (3, 2)), *, precision="bf16",
                 device=0, seed=None):
        assert pool in {'cls', 'mean'}, 'pool type must be either cls (cls token) or mean (mean pooling)'
        if transformer is None:
            assert all(v is not None for v in (depth, heads, mlp_dim)), 'depth, heads, and mlp_dim must be supplied'
        else:
            depth, heads, mlp_dim = 0, 1, 1          # the engine holds no main-transformer layers
        if channels != 3:
            raise NotImplementedError("libvitb200 takes NHWC images with 3 channels")
        if isinstance(image_size, tuple):
            raise ValueError("T2TViT takes an integer image_size (t2t.py:66)")
        t2t_layers = tuple((int(k), int(s)) for k, s in t2t_layers)
        if not 1 <= len(t2t_layers) <= 4:
            raise NotImplementedError("libvitb200 supports 1 to 4 t2t_layers")
        self.num_classes, self.pool, self.dim = num_classes, pool, dim
        self._dropout_rates = (dropout, emb_dropout)
        kw = {}
        for i, (k, s) in enumerate(t2t_layers):
            kw[f"t2t_k{i}"], kw[f"t2t_s{i}"] = k, s
        self._create(precision, device, image_h=image_size, image_w=image_size, num_classes=num_classes, dim=dim, depth=depth,
                     heads=heads, dim_head=dim_head, mlp_dim=mlp_dim, pool=0 if pool == 'cls' else 1,
                     t2t_num_layers=len(t2t_layers), **kw)
        self.init_weights(seed)
        self._attach_stage_attributes()
        # t2t.py:58-74: patch_embedding is Sequential([RearrangeUnfoldTransformer..., Dense]); only its last layer (the Dense,
        # what mpp.py:200 calls) is exposed on its own -- the soft splits run inside vb_forward_embed
        self.patch_embedding.layers = [_Layer(self.patch_to_emb)]
        self._injected = transformer
        self.transformer = transformer if transformer is not None else _Transformer(self)

    def __call__(self, img, training=True, **kwargs):
        if self._injected is None:
            return super().__call__(img, training=training)
        self._check_training(training)
        x = self.forward_embed(img)                                   # t2t.py:97-103
        x = np.asarray(self._injected(x, training=training), dtype=np.float32)   # :105
        return self.forward_head(x)                                   # :107-112

    call = __call__


class PatchMergerViT(_EngineModel):
    """vit_with_patch_merger.py:134-185 (`vit_with_patch_merger.ViT`): no cls token, a PatchMerger after layer
    `patch_merge_layer` (default depth // 2) shrinking the stream to `patch_merge_num_tokens` rows, mean pooling."""
    _kind = "patch_merger_vit"

    def __init__(self, image_size, patch_size, num_classes, dim, depth, heads, mlp_dim, patch_merge_layer=None,
                 patch_merge_num_tokens=8, dim_head=64, dropout=0.0, emb_dropout=0.0, *, precision="bf16", device=0, seed=None):
        image_height, image_width = pair(image_size)
        patch_height, patch_width = pair(patch_size)
        assert image_height % patch_height == 0 and image_width % patch_width == 0, 'Image dimensions must be divisible by the patch size.'
        self.num_classes, self.dim = num_classes, dim
        self._dropout_rates = (dropout, emb_dropout)
        index = (patch_merge_layer if patch_merge_layer is not None else depth // 2) - 1   # vit_with_patch_merger.py:108
        self._create(precision, device, image_h=image_height, image_w=image_width, patch_h=patch_height, patch_w=patch_width,
                     num_classes=num_classes, dim=dim, depth=depth, heads=heads, dim_head=dim_head, mlp_dim=mlp_dim, pool=1,
                     patch_merge_layer_index=index, patch_merge_num_tokens=patch_merge_num_tokens)
        self.init_weights(seed)
        self._attach_stage_attributes()


class PatchMerger:
    """vit_with_patch_merger.py:42-55 as a standalone layer: `PatchMerger(dim, num_tokens_out)(x [b, n, dim]) -> [b, num_tokens_out, dim]`.
    Weights: `queries` N(0,1) [num_tokens_out, dim] (:47), `norm_gamma` / `norm_beta` (LayerNormalization :46)."""

    def __init__(self, dim, num_tokens_out, *, precision="bf16", seed=None):
        self.dim, self.num_tokens_out, self.precision = dim, num_tokens_out, precision
        self.queries = np.random.default_rng(seed).standard_normal((num_tokens_out, dim)).astype(np.float32)
        self.norm_gamma = np.ones(dim, np.float32)
        self.norm_beta = np.zeros(dim, np.float32)

    def __call__(self, x, training=True):
        x = np.ascontiguousarray(x, dtype=np.float32)
        if x.ndim != 3 or x.shape[2] != self.dim:
            raise ValueError(f"x must be [b, n, {self.dim}]")
        return _as_tensor(_lib.op_patch_merger(x, self.norm_gamma, self.norm_beta, self.queries, precision=self.precision)[0])

    call = __call__


class EfficientViT(_EngineModel):
    """efficient.py:12-55 (`efficient.ViT`): the ViT shell around an injected `transformer` -- any callable
    `transformer(tokens [b, n + 1, dim], training=...) -> [b, n + 1, dim]` (the reference passes Keras layers from
    efficient-attention libraries; another engine model's `.transformer` works too).  The engine runs the patch embedding,
    cls token and positions (efficient.py:40-45, `vb_forward_embed`) and pooling + mlp_head (:48-55, `vb_forward_head`)."""
    _kind = "vit"

    def __init__(self, image_size, patch_size, num_classes, dim, transformer, pool='cls', *, precision="bf16", device=0, seed=None):
        image_size_h, image_size_w = pair(image_size)
        assert image_size_h % patch_size == 0 and image_size_w % patch_size == 0, 'image dimensions must be divisible by the patch size'
        assert pool in {'cls', 'mean'}, 'pool type must be either cls (cls token) or mean (mean pooling)'
        self.num_classes, self.pool, self.dim = num_classes, pool, dim
        self._dropout_rates = ()
        self._create(precision, device, image_h=image_size_h, image_w=image_size_w, patch_h=patch_size, patch_w=patch_size,
                     num_classes=num_classes, dim=dim, depth=0, heads=1, dim_head=1, mlp_dim=1, pool=0 if pool == 'cls' else 1)
        self.init_weights(seed)
        self._attach_stage_attributes()
        self.transformer = transformer

    def __call__(self, img, training=True, **kwargs):
        x = self.forward_embed(img)                                              # efficient.py:40-45
        x = np.asarray(self.transformer(x, training=training), dtype=np.float32)  # :46
        return self.forward_head(x)                                              # :48-55

    call = __call__


def sinusoidal_embedding(n_channels, dim):
    """TransformerClassifier.sinusoidal_embedding (cct.py:269-275) as the code spells it: the angles as Python floats, cast to
    float32, then sin / cos in float32 on the even / odd columns.  -> float32 [1, n_channels, dim]."""
    pe = np.asarray([[p / (10000 ** (2 * (i // 2) / dim)) for i in range(dim)] for p in range(n_channels)]).astype(np.float32)
    pe[:, 0::2] = np.sin(pe[:, 0::2])
    pe[:, 1::2] = np.cos(pe[:, 1::2])
    return pe[None]


def _truncated_normal(rng, shape, stddev):
    """tf.random.truncated_normal: N(0, stddev) with draws beyond two standard deviations redrawn."""
    a = rng.standard_normal(shape)
    bad = np.abs(a) > 2.0
    while bad.any():
        a[bad] = rng.standard_normal(int(bad.sum()))
        bad = np.abs(a) > 2.0
    return a * stddev


def cct_token_grid(h, w, n_conv_layers, stride, pooling_stride):
    """Token grid of the CCT Tokenizer (cct.py:188-215): every Conv2D and MaxPool2D uses SAME padding, ceil(size / stride)."""
    for _ in range(n_conv_layers):
        h, w = -(-h // stride), -(-w // stride)
        h, w = -(-h // pooling_stride), -(-w // pooling_stride)
    return h, w


class TransformerClassifier:
    """The constructor-argument handling of the reference's TransformerClassifier (cct.py:217-242), which CCT forwards its
    *args / **kwargs to: same parameter list, so positional extras and the kwargs CCT sets itself raise the same TypeError
    (multiple values), unknown kwargs are swallowed and an unknown positional_embedding falls back to 'sine'.  Holds the
    resolved configuration; the layers are the engine's."""

    def __init__(self, seq_pool=True, embedding_dim=768, num_layers=12, num_heads=12, mlp_ratio=4.0, num_classes=1000,
                 dropout_rate=0.1, attention_dropout=0.1, stochastic_depth_rate=0.1, positional_embedding='sine',
                 sequence_length=None, *args, **kwargs):
        positional_embedding = positional_embedding if positional_embedding in ['sine', 'learnable', 'none'] else 'sine'
        self.embedding_dim, self.num_layers, self.num_heads, self.num_classes = embedding_dim, num_layers, num_heads, num_classes
        self.mlp_dim = int(embedding_dim * mlp_ratio)                                 # cct.py:235
        self.positional_embedding, self.sequence_length, self.seq_pool = positional_embedding, sequence_length, seq_pool
        self.dropout_rates = (dropout_rate, attention_dropout, stochastic_depth_rate)
        assert sequence_length is not None or positional_embedding == 'none', \
            f"Positional embedding is set to {positional_embedding} and" \
            f" the sequence length was not specified."


class CCT(_EngineModel):
    """cct.py:307-345: convolutional tokenizer (n_conv_layers x Conv2D SAME -> ReLU -> MaxPool2D SAME), positional embedding,
    post-attention-norm encoder layers (x = norm1(x + attn(pre_norm(x))); x = x + mlp(x)), sequence pooling, fc.

    Inference only: the reference hard-codes attention_dropout = stochastic_depth_rate = 0.1 (cct.py:336-338) and its call
    resolves `training=None` to the classifier's default True, so every call without `training=False` is stochastic there;
    here such a call raises NotImplementedError.  Images are NHWC with 3 channels; with a 'sine' / 'learnable' embedding they
    must give the token count of `img_size`, with 'none' fewer tokens are zero-padded to it (cct.py:278-280).
    Weights (SURVEY.md App. B): tokenizer.conv.{i}.kernel [k, k, cin, cout], positional_emb [1, n, dim],
    layers.L.{attn_norm, to_qkv, to_out, norm1, fc1, fc2}, norm, attention_pool [dim, 1] + [1], head."""
    _kind = "cct"

    def __init__(self, img_size=224, embedding_dim=768, n_input_channels=3, n_conv_layers=1, kernel_size=7, stride=2,
                 pooling_kernel_size=3, pooling_stride=2, *args, precision="bf16", device=0, seed=None, **kwargs):
        img_height, img_width = pair(img_size)
        if n_input_channels != 3:
            raise NotImplementedError("libvitb200 takes NHWC images with 3 channels")
        seq_h, seq_w = cct_token_grid(img_height, img_width, n_conv_layers, stride, pooling_stride)
        tc = TransformerClassifier(sequence_length=seq_h * seq_w, embedding_dim=embedding_dim, seq_pool=True, dropout_rate=0.,
                                   attention_dropout=0.1, stochastic_depth_rate=0.1, *args, **kwargs)   # cct.py:330-339
        if embedding_dim % tc.num_heads != 0:
            raise ValueError(f"CCT: embedding_dim ({embedding_dim}) must be divisible by num_heads ({tc.num_heads})")
        self.num_classes, self.dim = tc.num_classes, embedding_dim
        self.sequence_length = tc.sequence_length
        self._positional_embedding = tc.positional_embedding
        self._dropout_rates = tc.dropout_rates
        self._create(precision, device, image_h=img_height, image_w=img_width, num_classes=tc.num_classes, dim=embedding_dim,
                     depth=tc.num_layers, heads=tc.num_heads, dim_head=embedding_dim // tc.num_heads, mlp_dim=tc.mlp_dim,
                     cct_conv_layers=n_conv_layers, cct_kernel=kernel_size, cct_stride=stride, cct_pool_kernel=pooling_kernel_size,
                     cct_pool_stride=pooling_stride, cct_pos_emb=_lib.CCT_POS[tc.positional_embedding])
        self.init_weights(seed)

    def _check_training(self, training):
        if training is None or training:
            raise NotImplementedError(
                "CCT runs inference only: the reference's call resolves training=None to True and then applies its "
                "hard-coded attention dropout and stochastic depth of 0.1 (cct.py:336-338); pass training=False")

    def __call__(self, img, training=None, **kwargs):
        """cct.py:342: NHWC float image batch -> float32 logits [b, num_classes]; training must be False."""
        return super().__call__(img, training=training)

    call = __call__


def _cct(num_layers, num_heads, mlp_ratio, embedding_dim, kernel_size=3, stride=None, *args, **kwargs):   # cct.py:51-61
    stride = stride if stride is not None else max(1, (kernel_size // 2) - 1)
    return CCT(num_layers=num_layers, num_heads=num_heads, mlp_ratio=mlp_ratio, embedding_dim=embedding_dim,
               kernel_size=kernel_size, stride=stride, *args, **kwargs)


def cct_2(*args, **kwargs):   # cct.py:16-48
    return _cct(num_layers=2, num_heads=2, mlp_ratio=1, embedding_dim=128, *args, **kwargs)


def cct_4(*args, **kwargs):
    return _cct(num_layers=4, num_heads=2, mlp_ratio=1, embedding_dim=128, *args, **kwargs)


def cct_6(*args, **kwargs):
    return _cct(num_layers=6, num_heads=4, mlp_ratio=2, embedding_dim=256, *args, **kwargs)


def cct_7(*args, **kwargs):
    return _cct(num_layers=7, num_heads=4, mlp_ratio=2, embedding_dim=256, *args, **kwargs)


def cct_8(*args, **kwargs):
    return _cct(num_layers=8, num_heads=4, mlp_ratio=2, embedding_dim=256, *args, **kwargs)


def cct_14(*args, **kwargs):
    return _cct(num_layers=14, num_heads=6, mlp_ratio=3, embedding_dim=384, *args, **kwargs)


def cct_16(*args, **kwargs):
    return _cct(num_layers=16, num_heads=6, mlp_ratio=3, embedding_dim=384, *args, **kwargs)


CCT_CTOR_KEYS = ("img_size", "embedding_dim", "n_input_channels", "n_conv_layers", "kernel_size", "stride", "pooling_kernel_size",
                 "pooling_stride", "num_layers", "num_heads", "mlp_ratio", "num_classes", "positional_embedding")


def levit_cast_tuple(val, l=3):
    """levit.py:18-20: an int is repeated, a short tuple padded with its last element, a long one kept (the assert catches it)."""
    val = val if isinstance(val, tuple) else (val,)
    return (*val, *((val[-1],) * max(l - len(val), 0)))


class LeViT(_EngineModel):
    """levit.py:164-226: a four-convolution stem, `stages` stacks of BatchNorm attention with a learned relative-position bias and
    hard-swish MLPs, a stride-2 "shrink" attention between stages, global average pooling, mlp_head (and distill_head).

    Inference only: the reference's call defaults to training=True, which makes every BatchNormalization use the batch's statistics
    and the dropout layers draw masks; a call without training=False raises NotImplementedError here.  The feature map after the
    stem must be image_size // 16 square (levit.py:194): such an image_size is refused at construction, and an image whose stem
    output has another size is refused at call time.
    Weights (SURVEY.md App. B) keep the reference's attribute paths: conv_embedding.{i}, backbone.{t}.layers.{l}.0 (attention:
    to_q / to_k / to_v .0 conv + .1 BatchNormalization, pos_bias.embeddings, to_out.1 conv + .2 BatchNormalization),
    backbone.{t}.layers.{l}.1.net.{0,3} (MLP), mlp_head, distill_head."""
    _kind = "levit"

    def __init__(self, image_size, num_classes, dim, depth, heads, mlp_mult, stages=3, dim_key=32, dim_value=64, dropout=0.0,
                 num_distill_classes=None, *, precision="bf16", device=0, seed=None):
        dims = levit_cast_tuple(dim, stages)
        depths = levit_cast_tuple(depth, stages)
        layer_heads = levit_cast_tuple(heads, stages)
        assert all(map(lambda t: len(t) == stages, (dims, depths, layer_heads))), \
            'dimensions, depths, and heads must be a tuple that is less than the designated number of stages'
        f = image_size
        for _ in range(4):
            f = -(-f // 2)
        if f != image_size // 16:
            raise ValueError(f"LeViT: image_size {image_size} gives a {f} x {f} map after the four stride-2 stem convolutions, but "
                             f"the position biases are built for image_size // 16 = {image_size // 16} (levit.py:194); the "
                             "reference fails at its first call")
        if stages > _lib.LEVIT_MAX_STAGES:
            raise ValueError(f"LeViT: at most {_lib.LEVIT_MAX_STAGES} stages")
        self.num_classes, self.num_distill_classes = num_classes, num_distill_classes
        self.dims, self.depths, self.layer_heads = dims, depths, layer_heads
        self.image_size, self.dim_key, self.dim_value, self.mlp_mult, self.stages = image_size, dim_key, dim_value, mlp_mult, stages
        self._dropout_rates = (dropout,)
        self.precision = precision
        self.device = int(device)
        cfg = _lib.VbConfig()
        cfg.struct_size = C.sizeof(_lib.VbConfig)
        cfg.kind = _lib.KIND["levit"]
        if precision not in _lib.PRECISION:
            raise ValueError(f"precision must be one of {sorted(_lib.PRECISION)}")
        cfg.precision = _lib.PRECISION[precision]
        cfg.channels, cfg.image_h, cfg.image_w, cfg.num_classes = 3, image_size, image_size, num_classes
        cfg.dim = dims[-1]                               # the pooled width (what the engine's handle records as dim)
        lv = _lib.VbLevitConfig()
        lv.struct_size = C.sizeof(_lib.VbLevitConfig)
        lv.stages = stages
        for i in range(stages):
            lv.dims[i], lv.depths[i], lv.heads[i] = dims[i], depths[i], layer_heads[i]
        lv.dim_key, lv.dim_value, lv.mlp_mult = dim_key, dim_value, mlp_mult
        lv.num_distill_classes = num_distill_classes or 0
        self._cfg, self._lv = cfg, lv
        self._lib = _lib.load()
        h = C.c_void_p()
        _lib.check(self._lib.vb_create_levit(C.byref(cfg), C.byref(lv), self.device, C.byref(h)))
        self._h = h
        self._finalized = False
        self._specs = collections.OrderedDict()
        name, shape, ndim = C.c_char_p(), (C.c_int64 * 4)(), C.c_int32()
        for i in range(self._lib.vb_num_weights(h)):
            _lib.check(self._lib.vb_weight_info(h, i, C.byref(name), shape, C.byref(ndim)), h)
            self._specs[name.value.decode()] = tuple(int(shape[j]) for j in range(ndim.value))
        self._weights = collections.OrderedDict()
        self.init_weights(seed)

    def init_weights(self, seed=None):
        """The reference's initialisers: glorot-uniform over the receptive field and zero biases (Conv2D / Dense), BatchNormalization
        gamma 1 / beta 0 / moving statistics 0 and 1 with the to_out gamma at 0 (levit.py:91), Embedding U(-0.05, 0.05)."""
        rng = np.random.default_rng(seed)
        w = collections.OrderedDict()
        for name, shape in self._specs.items():
            leaf = name.rsplit(".", 1)[-1]
            if leaf == "kernel":
                receptive = int(np.prod(shape[:-2]))
                lim = np.sqrt(6.0 / (receptive * (shape[-2] + shape[-1])))
                a = rng.uniform(-lim, lim, size=shape)
            elif leaf in ("bias", "beta", "moving_mean"):
                a = np.zeros(shape)
            elif leaf == "moving_variance":
                a = np.ones(shape)
            elif leaf == "gamma":
                a = np.zeros(shape) if ".to_out." in name else np.ones(shape)
            elif leaf == "embeddings":
                a = rng.uniform(-0.05, 0.05, size=shape)
            else:
                raise AssertionError(name)
            w[name] = a.astype(np.float32)
        self.set_weights_dict(w)

    def _check_training(self, training):
        if training is None or training:
            raise NotImplementedError(
                "LeViT runs inference only: with training=True (the reference's default, levit.py:214) every BatchNormalization "
                "normalises with the batch's own statistics and dropout draws masks; pass training=False")

    def __call__(self, img, training=True, **kwargs):
        """levit.py:214: NHWC float images -> logits [b, num_classes], or (logits, distill [b, num_distill_classes]) with a
        distillation head.  training must be False."""
        self._check_training(training)
        if self.num_distill_classes is None:
            return super().__call__(img, training=False)
        self._finalize()
        x = self._img(img)
        b, h, w, _ = x.shape
        logits = np.empty((b, self.num_classes), np.float32)
        dist = np.empty((b, self.num_distill_classes), np.float32)
        _lib.check(self._lib.vb_forward_distill(self._h, x.ctypes.data_as(C.c_void_p), _lib.MEM_HOST, b, h, w, None,
                                                logits.ctypes.data_as(C.c_void_p), dist.ctypes.data_as(C.c_void_p), _lib.MEM_HOST,
                                                None), self._h)
        return _as_tensor(logits), _as_tensor(dist)

    call = __call__


LEVIT_CTOR_KEYS = ("image_size", "num_classes", "dim", "depth", "heads", "mlp_mult", "stages", "dim_key", "dim_value", "dropout",
                   "num_distill_classes")


CVT_STAGE_KEYS = ("emb_dim", "emb_kernel", "emb_stride", "proj_kernel", "kv_proj_stride", "heads", "depth", "mlp_mult")


class CvT(_EngineModel):
    """cvt.py:149-202: three stages of Conv2D (SAME) + channel LayerNorm + Transformer, whose attention projects q and k|v with
    depthwise convolutions, BatchNormalization and 1x1 convolutions (heads of 64), then GlobalAvgPool2D and Dense.

    Inference only: the reference's call defaults to training=True, which makes every BatchNormalization use the batch's statistics
    and the dropout layers draw masks; a call without training=False raises NotImplementedError here.  There are no position
    embeddings and no image_size: any h x w image runs.  proj_kernel must be in [1, 7] and kv_proj_stride 1 or 2.
    Weights (SURVEY.md App. B) keep the reference's attribute paths: cvt_layers.{s}.0 (stem Conv2D), cvt_layers.{s}.1.g / .b
    (LayerNorm), cvt_layers.{s}.2.layers.{l}.0.norm / .0.fn.to_q.net.{0,1,2} / .0.fn.to_kv.net.{0,1,2} / .0.fn.to_out.0,
    cvt_layers.{s}.2.layers.{l}.1.norm / .1.fn.net.{0,3}, cvt_layers.3.1 (the Dense head)."""
    _kind = "cvt"

    def __init__(self,
                 num_classes,
                 s1_emb_dim=64,
                 s1_emb_kernel=7,
                 s1_emb_stride=4,
                 s1_proj_kernel=3,
                 s1_kv_proj_stride=2,
                 s1_heads=1,
                 s1_depth=1,
                 s1_mlp_mult=4,
                 s2_emb_dim=192,
                 s2_emb_kernel=3,
                 s2_emb_stride=2,
                 s2_proj_kernel=3,
                 s2_kv_proj_stride=2,
                 s2_heads=3,
                 s2_depth=2,
                 s2_mlp_mult=4,
                 s3_emb_dim=384,
                 s3_emb_kernel=3,
                 s3_emb_stride=2,
                 s3_proj_kernel=3,
                 s3_kv_proj_stride=2,
                 s3_heads=6,
                 s3_depth=10,
                 s3_mlp_mult=4,
                 dropout=0.,
                 *, precision="bf16", device=0, seed=None):
        kw = dict(locals())
        self.num_classes = num_classes
        self.stages = tuple({k: kw[f"s{i}_{k}"] for k in CVT_STAGE_KEYS} for i in (1, 2, 3))
        self._dropout_rates = (dropout,)
        for st in self.stages:
            if not 1 <= st["proj_kernel"] <= 7:
                raise ValueError(f"CvT: proj_kernel {st['proj_kernel']} is not supported (1 to 7)")
            if st["kv_proj_stride"] not in (1, 2):
                raise ValueError(f"CvT: kv_proj_stride {st['kv_proj_stride']} is not supported (1 or 2)")
        self.precision = precision
        self.device = int(device)
        cfg = _lib.VbConfig()
        cfg.struct_size = C.sizeof(_lib.VbConfig)
        cfg.kind = _lib.KIND["cvt"]
        if precision not in _lib.PRECISION:
            raise ValueError(f"precision must be one of {sorted(_lib.PRECISION)}")
        cfg.precision = _lib.PRECISION[precision]
        cfg.channels, cfg.num_classes = 3, num_classes
        cfg.dim = self.stages[-1]["emb_dim"]
        cv = _lib.VbCvtConfig()
        cv.struct_size = C.sizeof(_lib.VbCvtConfig)
        for i, st in enumerate(self.stages):
            for k in CVT_STAGE_KEYS:
                getattr(cv, k)[i] = int(st[k])
        self._cfg, self._cv = cfg, cv
        self._lib = _lib.load()
        h = C.c_void_p()
        _lib.check(self._lib.vb_create_cvt(C.byref(cfg), C.byref(cv), self.device, C.byref(h)))
        self._h = h
        self._finalized = False
        self._specs = collections.OrderedDict()
        name, shape, ndim = C.c_char_p(), (C.c_int64 * 4)(), C.c_int32()
        for i in range(self._lib.vb_num_weights(h)):
            _lib.check(self._lib.vb_weight_info(h, i, C.byref(name), shape, C.byref(ndim)), h)
            self._specs[name.value.decode()] = tuple(int(shape[j]) for j in range(ndim.value))
        self._weights = collections.OrderedDict()
        self.init_weights(seed)

    def init_weights(self, seed=None):
        """The reference's initialisers: glorot-uniform over the receptive field (a depthwise kernel [k, k, 1, dim] has fan_in k^2 and
        fan_out k^2 * dim) and zero biases, BatchNormalization gamma 1 / beta 0 / moving statistics 0 and 1, LayerNorm g 1 / b 0."""
        rng = np.random.default_rng(seed)
        w = collections.OrderedDict()
        for name, shape in self._specs.items():
            leaf = name.rsplit(".", 1)[-1]
            if leaf == "kernel":
                receptive = int(np.prod(shape[:-2]))
                lim = np.sqrt(6.0 / (receptive * (shape[-2] + shape[-1])))
                a = rng.uniform(-lim, lim, size=shape)
            elif leaf in ("bias", "beta", "moving_mean", "b"):
                a = np.zeros(shape)
            elif leaf in ("gamma", "moving_variance", "g"):
                a = np.ones(shape)
            else:
                raise AssertionError(name)
            w[name] = a.astype(np.float32)
        self.set_weights_dict(w)

    def _check_training(self, training):
        if training is None or training:
            raise NotImplementedError(
                "CvT runs inference only: with training=True (the reference's default, cvt.py:200) every BatchNormalization "
                "normalises with the batch's own statistics and dropout draws masks; pass training=False")

    def __call__(self, img, training=True, **kwargs):
        """cvt.py:200: NHWC float images of any size -> logits [b, num_classes].  training must be False."""
        return super().__call__(img, training=training)

    call = __call__


CVT_CTOR_KEYS = ("num_classes",) + tuple(f"s{i}_{k}" for i in (1, 2, 3) for k in CVT_STAGE_KEYS) + ("dropout",)


TWINS_STAGE_KEYS = ("emb_dim", "patch_size", "local_patch_size", "global_k", "depth")


def twins_size_error(stages, h, w):
    """The reference's shape rules (twins_svt.py:103,141,168, enforced there by einops and Keras) for an h x w image: None, or
    what the first stage that breaks one says."""
    for i, st in enumerate(stages, 1):
        ps = st["patch_size"]
        if h % ps or w % ps:
            return f"Twins-SVT stage {i}: the {h} x {w} map is not divisible by patch_size {ps}"
        h, w = h // ps, w // ps
        if i < len(stages) and (h % st["local_patch_size"] or w % st["local_patch_size"]):
            return f"Twins-SVT stage {i}: the {h} x {w} map is not divisible by local_patch_size {st['local_patch_size']}"
        if h < st["global_k"] or w < st["global_k"]:
            return f"Twins-SVT stage {i}: the {h} x {w} map is smaller than global_k {st['global_k']} (a VALID convolution)"
    return None


class TwinsSVT(_EngineModel):
    """twins_svt.py:215-268: four stages of PatchEmbedding (c-slowest patch vectors, 1x1 Conv2D), a Transformer of depth 1, the PEG
    (x + a depthwise SAME convolution) and a Transformer of depth s{i}_depth, then GlobalAvgPool2D and Dense.  A Transformer layer
    is local attention within local_patch_size windows, an MLP, global attention against the keys of a global_k x global_k stride
    global_k VALID convolution, and an MLP, each PreNorm and residual; stage 4 has no local attention and no first MLP.  Every stage
    has 8 heads of 64 and an MLP multiplier of 4, whatever emb_dim is: the reference never passes them to Transformer.

    There are no position embeddings and no image_size: any image whose maps are divisible by every patch_size and, in stages 1-3,
    local_patch_size, and are at least global_k on each side runs; other sizes raise ValueError naming the stage.  There is no
    BatchNormalization, so with dropout = 0 training=True computes what training=False does.  peg_kernel_size must be in [1, 7].
    Weights (SURVEY.md App. B) keep the reference's attribute paths: svt_layers.{s}.0.proj, svt_layers.{s}.{1|3}.layers.{l}.{0..3}
    .fn.norm / .fn.fn.{to_q, to_kv, to_out.0, net.0, net.3}, svt_layers.{s}.2.proj.fn (PEG), svt_layers.4.1 (the Dense head)."""
    _kind = "twins_svt"

    def __init__(self,
                 num_classes,
                 s1_emb_dim=64,
                 s1_patch_size=4,
                 s1_local_patch_size=7,
                 s1_global_k=7,
                 s1_depth=1,
                 s2_emb_dim=128,
                 s2_patch_size=2,
                 s2_local_patch_size=7,
                 s2_global_k=7,
                 s2_depth=1,
                 s3_emb_dim=256,
                 s3_patch_size=2,
                 s3_local_patch_size=7,
                 s3_global_k=7,
                 s3_depth=5,
                 s4_emb_dim=512,
                 s4_patch_size=2,
                 s4_local_patch_size=7,
                 s4_global_k=7,
                 s4_depth=4,
                 peg_kernel_size=3,
                 dropout=0.0,
                 *, precision="bf16", device=0, seed=None):
        kw = dict(locals())
        self.num_classes = num_classes
        self.stages = tuple({k: kw[f"s{i}_{k}"] for k in TWINS_STAGE_KEYS} for i in (1, 2, 3, 4))
        self.peg_kernel_size = peg_kernel_size
        self._dropout_rates = (dropout,)
        if not 1 <= peg_kernel_size <= 7:
            raise ValueError(f"Twins-SVT: peg_kernel_size {peg_kernel_size} is not supported (1 to 7)")
        self.precision = precision
        self.device = int(device)
        cfg = _lib.VbConfig()
        cfg.struct_size = C.sizeof(_lib.VbConfig)
        cfg.kind = _lib.KIND["twins_svt"]
        if precision not in _lib.PRECISION:
            raise ValueError(f"precision must be one of {sorted(_lib.PRECISION)}")
        cfg.precision = _lib.PRECISION[precision]
        cfg.channels, cfg.num_classes = 3, num_classes
        cfg.dim = self.stages[-1]["emb_dim"]
        tw = _lib.VbTwinsSvtConfig()
        tw.struct_size = C.sizeof(_lib.VbTwinsSvtConfig)
        for i, st in enumerate(self.stages):
            for k in TWINS_STAGE_KEYS:
                getattr(tw, k)[i] = int(st[k])
        tw.peg_kernel_size = int(peg_kernel_size)
        self._cfg, self._tw = cfg, tw
        self._lib = _lib.load()
        h = C.c_void_p()
        _lib.check(self._lib.vb_create_twins_svt(C.byref(cfg), C.byref(tw), self.device, C.byref(h)))
        self._h = h
        self._finalized = False
        self._specs = collections.OrderedDict()
        name, shape, ndim = C.c_char_p(), (C.c_int64 * 4)(), C.c_int32()
        for i in range(self._lib.vb_num_weights(h)):
            _lib.check(self._lib.vb_weight_info(h, i, C.byref(name), shape, C.byref(ndim)), h)
            self._specs[name.value.decode()] = tuple(int(shape[j]) for j in range(ndim.value))
        self._weights = collections.OrderedDict()
        self.init_weights(seed)

    def init_weights(self, seed=None):
        """The reference's initialisers: glorot-uniform over the receptive field (the PEG's depthwise kernel [k, k, 1, dim] has fan_in
        k^2 and fan_out k^2 * dim), zero biases, LayerNorm g 1 / b 0."""
        rng = np.random.default_rng(seed)
        w = collections.OrderedDict()
        for name, shape in self._specs.items():
            leaf = name.rsplit(".", 1)[-1]
            if leaf == "kernel":
                receptive = int(np.prod(shape[:-2]))
                lim = np.sqrt(6.0 / (receptive * (shape[-2] + shape[-1])))
                a = rng.uniform(-lim, lim, size=shape)
            elif leaf in ("bias", "b"):
                a = np.zeros(shape)
            elif leaf == "g":
                a = np.ones(shape)
            else:
                raise AssertionError(name)
            w[name] = a.astype(np.float32)
        self.set_weights_dict(w)

    def __call__(self, img, training=True, **kwargs):
        """twins_svt.py:266-268: NHWC float images -> logits [b, num_classes]; extra kwargs are accepted and ignored, as there."""
        x = np.asarray(img)
        if x.ndim == 4:
            err = twins_size_error(self.stages, x.shape[1], x.shape[2])
            if err is not None:
                raise ValueError(err)
        return super().__call__(img, training=training)

    call = __call__


TWINS_CTOR_KEYS = ("num_classes",) + tuple(f"s{i}_{k}" for i in (1, 2, 3, 4) for k in TWINS_STAGE_KEYS) + ("peg_kernel_size", "dropout")


def _cast_tuple(val, length=1):                     # crossformer.py:11-12
    return val if isinstance(val, tuple) else ((val,) * length)


def crossformer_size_error(stages, h, w):
    """The reference's shape rule (crossformer.py:144,146, enforced there by einops) for an h x w image: None, or what the first
    stage that breaks it says.  Each stage map is ceil(previous / stride) (the SAME convolutions)."""
    for i, st in enumerate(stages, 1):
        h, w = -(-h // st["stride"]), -(-w // st["stride"])
        for key, name in (("local_wsz", "local_window_size"), ("global_wsz", "global_window_size")):
            if h % st[key] or w % st[key]:
                return f"CrossFormer stage {i}: the {h} x {w} map is not divisible by {name} {st[key]}"
    return None


class CrossFormer(_EngineModel):
    """crossformer.py:205-269: four stages of a CrossEmbedLayer (one SAME Conv2D per kernel size at the stage's stride, the kernel
    sizes sorted, dim / 2, dim / 4, ... channels and the rest for the largest, concatenated) and a Transformer whose layers are
    short attention within local_window_size blocks, an MLP, long attention within global_window_size dilated windows and an MLP,
    each with its own LayerNorm and a residual; then the mean over the map and Dense(num_classes).  Attention has dim // 32 heads
    of 32 and a DynamicPositionBias scalar per in-window offset, shared by the heads.

    There are no position embeddings and no image_size: any image whose every stage map is divisible by that stage's local and
    global window sizes runs; other sizes raise ValueError naming the stage.  The engine runs a stage's cross-scale embedding as
    one convolution with the smaller kernels nested at the centre of the largest, which is exact for every image when the
    stage's kernel sizes share one parity and are all at least its stride (the reference's defaults are); other kernel sets,
    more than 4 kernel sizes and dims below 32 raise ValueError.  attn_dropout is accepted and unused, as in the reference; with
    ff_dropout > 0 only training=False runs.  Weights (SURVEY.md App. B) keep the reference's attribute paths:
    crossformer_layers.{s}.0.convs.{i}, crossformer_layers.{s}.1.layers.{l}.{0|2}.{norm, to_qkv, to_out, dpb.dpb_layers.{0..9}},
    crossformer_layers.{s}.1.layers.{l}.{1|3}.net.{0, 1, 4}, to_logits.1 (the Dense head)."""
    _kind = "crossformer"

    def __init__(self,
                 dim=(64, 128, 256, 512),
                 depth=(2, 2, 8, 2),
                 global_window_size=(8, 4, 2, 1),
                 local_window_size=7,
                 cross_embed_kernel_sizes=((4, 8, 16, 32), (2, 4), (2, 4), (2, 4)),
                 cross_embed_strides=(4, 2, 2, 2),
                 num_classes=1000,
                 attn_dropout=0.0,
                 ff_dropout=0.0,
                 *, precision="bf16", device=0, seed=None):
        dim = _cast_tuple(dim, 4)
        depth = _cast_tuple(depth, 4)
        global_window_size = _cast_tuple(global_window_size, 4)
        local_window_size = _cast_tuple(local_window_size, 4)
        cross_embed_kernel_sizes = _cast_tuple(cross_embed_kernel_sizes, 4)
        cross_embed_strides = _cast_tuple(cross_embed_strides, 4)
        assert len(dim) == 4
        assert len(depth) == 4
        assert len(global_window_size) == 4
        assert len(local_window_size) == 4
        assert len(cross_embed_kernel_sizes) == 4
        assert len(cross_embed_strides) == 4
        self.num_classes = num_classes
        self.stages = tuple(dict(dim=int(d), depth=int(n), global_wsz=int(g), local_wsz=int(lw), kernels=tuple(sorted(k)), stride=int(st))
                            for d, n, g, lw, k, st in zip(dim, depth, global_window_size, local_window_size, cross_embed_kernel_sizes,
                                                          cross_embed_strides))
        self._dropout_rates = (ff_dropout,)
        for i, st in enumerate(self.stages, 1):
            ks = st["kernels"]
            if st["dim"] < 32:
                raise ValueError(f"CrossFormer stage {i}: dim {st['dim']} is not supported (at least 32: dim // 32 heads of 32)")
            if not 1 <= len(ks) <= _lib.CROSSFORMER_MAX_KERNELS:
                raise ValueError(f"CrossFormer stage {i}: {len(ks)} cross-embedding kernel sizes {ks}; at most "
                                 f"{_lib.CROSSFORMER_MAX_KERNELS} are supported")
            if len({k % 2 for k in ks}) != 1 or min(ks) < st["stride"]:
                raise ValueError(f"CrossFormer stage {i}: kernel sizes {ks} at stride {st['stride']} are not supported: the nested "
                                 "cross-scale embedding needs kernel sizes of one parity, each at least the stride")
        self.precision = precision
        self.device = int(device)
        cfg = _lib.VbConfig()
        cfg.struct_size = C.sizeof(_lib.VbConfig)
        cfg.kind = _lib.KIND["crossformer"]
        if precision not in _lib.PRECISION:
            raise ValueError(f"precision must be one of {sorted(_lib.PRECISION)}")
        cfg.precision = _lib.PRECISION[precision]
        cfg.channels, cfg.num_classes = 3, num_classes
        cfg.dim = self.stages[-1]["dim"]
        cf = _lib.VbCrossformerConfig()
        cf.struct_size = C.sizeof(_lib.VbCrossformerConfig)
        for i, st in enumerate(self.stages):
            for k in ("dim", "depth", "global_wsz", "local_wsz", "stride"):
                getattr(cf, k)[i] = st[k]
            cf.n_kernels[i] = len(st["kernels"])
            for j, k in enumerate(st["kernels"]):
                cf.kernels[i][j] = int(k)
        self._cfg, self._cf = cfg, cf
        self._lib = _lib.load()
        h = C.c_void_p()
        _lib.check(self._lib.vb_create_crossformer(C.byref(cfg), C.byref(cf), self.device, C.byref(h)))
        self._h = h
        self._finalized = False
        self._specs = collections.OrderedDict()
        name, shape, ndim = C.c_char_p(), (C.c_int64 * 4)(), C.c_int32()
        for i in range(self._lib.vb_num_weights(h)):
            _lib.check(self._lib.vb_weight_info(h, i, C.byref(name), shape, C.byref(ndim)), h)
            self._specs[name.value.decode()] = tuple(int(shape[j]) for j in range(ndim.value))
        self._weights = collections.OrderedDict()
        self.init_weights(seed)

    def init_weights(self, seed=None):
        """The reference's initialisers: glorot-uniform over the receptive field for every Conv2D and Dense kernel, zero biases,
        LayerNorm g 1 / b 0 and LayerNormalization gamma 1 / beta 0."""
        rng = np.random.default_rng(seed)
        w = collections.OrderedDict()
        for name, shape in self._specs.items():
            leaf = name.rsplit(".", 1)[-1]
            if leaf == "kernel":
                receptive = int(np.prod(shape[:-2]))
                lim = np.sqrt(6.0 / (receptive * (shape[-2] + shape[-1])))
                a = rng.uniform(-lim, lim, size=shape)
            elif leaf in ("bias", "b", "beta"):
                a = np.zeros(shape)
            elif leaf in ("g", "gamma"):
                a = np.ones(shape)
            else:
                raise AssertionError(name)
            w[name] = a.astype(np.float32)
        self.set_weights_dict(w)

    def __call__(self, img, training=True, **kwargs):
        """crossformer.py:263-269: NHWC float images -> logits [b, num_classes]; extra kwargs are accepted and ignored, as there."""
        x = np.asarray(img)
        if x.ndim == 4:
            err = crossformer_size_error(self.stages, x.shape[1], x.shape[2])
            if err is not None:
                raise ValueError(err)
        return super().__call__(img, training=training)

    call = __call__


CROSSFORMER_CTOR_KEYS = ("dim", "depth", "global_window_size", "local_window_size", "cross_embed_kernel_sizes", "cross_embed_strides",
                         "num_classes", "attn_dropout", "ff_dropout")


def from_config(cfg: dict, precision="bf16", device=0, seed=None):
    """Build a model from an oracle-style config dict (kind + reference kwargs)."""
    if cfg["kind"] == "crossformer":
        return CrossFormer(**{k: v for k, v in cfg.items() if k in CROSSFORMER_CTOR_KEYS}, precision=precision, device=device, seed=seed)
    if cfg["kind"] == "twins_svt":
        return TwinsSVT(**{k: v for k, v in cfg.items() if k in TWINS_CTOR_KEYS}, precision=precision, device=device, seed=seed)
    if cfg["kind"] == "cvt":
        return CvT(**{k: v for k, v in cfg.items() if k in CVT_CTOR_KEYS}, precision=precision, device=device, seed=seed)
    if cfg["kind"] == "levit":
        return LeViT(**{k: v for k, v in cfg.items() if k in LEVIT_CTOR_KEYS}, precision=precision, device=device, seed=seed)
    if cfg["kind"] == "cct":
        return CCT(**{k: v for k, v in cfg.items() if k in CCT_CTOR_KEYS}, precision=precision, device=device, seed=seed)
    kw = {k: v for k, v in cfg.items() if k not in ("kind", "channels", "image_h", "image_w", "patch_h", "patch_w", "num_patches",
                                                    "patch_merge_layer_index", "t2t_dims")}
    if cfg["kind"] == "patch_merger_vit":
        kw.pop("pool", None)
    cls = {"vit": ViT, "deepvit": DeepViT, "cait": CaiT, "crossvit": CrossViT, "parallel_vit": ParallelViT,
           "patch_merger_vit": PatchMergerViT, "t2t_vit": T2TViT}[cfg["kind"]]
    if cfg["kind"] == "crossvit":
        kw.setdefault("dropout", 0.0)
        kw.setdefault("emb_dropout", 0.0)
    return cls(**kw, precision=precision, device=device, seed=seed)

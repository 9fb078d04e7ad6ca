"""Host-side mirror of the reference's model classes over the libvitb200 C-ABI.

    ViT       vit_tensorflow/vit.py:106-177          DeepViT   vit_tensorflow/deepvit.py:112-157
    CaiT      vit_tensorflow/cait.py:155-194         CrossViT  vit_tensorflow/cross_vit.py:232-303
    parallel_vit.ViT  parallel_vit.py:120-185        DistillableViT  distill.py:47-58 (forward)
    DistillableT2TViT  distill.py:61-72 (forward)    DistillableEfficientViT  distill.py:74-85 (raises as the reference does)
    T2TViT    vit_tensorflow/t2t.py:50-116           vit_with_patch_merger.ViT / PatchMerger  vit_with_patch_merger.py:42-55,134-185
    efficient.ViT  vit_tensorflow/efficient.py:12-55 (injected transformer between the engine's embed and head stages)
    CvT       vit_tensorflow/cvt.py:149-202
    TwinsSVT  vit_tensorflow/twins_svt.py:215-268
    CrossFormer  vit_tensorflow/crossformer.py:205-269
    NesT      vit_tensorflow/nest.py:150-216
    RegionViT vit_tensorflow/regionvit.py:184-263
    ScalableViT  vit_tensorflow/scalable_vit.py:250-319
    PiT       vit_tensorflow/pit.py:158-219
    MAE / SimMIM  vit_tensorflow/mae.py:17-92, simmim.py:72-129 (around a ViT encoder)
    DistillWrapper  vit_tensorflow/distill.py:87-134 (around a distillable student and any teacher)

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
import math

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
    _encoder_names = ()         # weights another model owns and initialises (MAE / SimMIM: the encoder's; DistillWrapper: the student's)
    _inference_only = None      # the message of a family whose every call without training=False raises NotImplementedError
    # tf.random.normal Variables, N(0, 1): vit.py:146-147, deepvit.py:57, cait.py:97-98, vit_with_patch_merger.py:47,
    # nest.py:129, mae.py:43, simmim.py:85, distill.py:101; vit_for_small_dataset.py:94's temperature is drawn too, then set
    # (SmallDatasetViT)
    _NORMAL_LEAVES = ("pos_embedding", "cls_token", "reattn_weights", "mix_pre", "mix_post", "queries", "pos_emb", "mask_token",
                      "temperature", "distillation_token")

    def _create(self, precision, device, ext=None, create="vb_create", **cfgkw):
        """`_config`, then every VbConfig field of `cfgkw` as int(value), then `_open`."""
        cfg = self._config(precision, device)
        for k, v in cfgkw.items():
            setattr(cfg, k, int(v))
        self._open(cfg, create, ext)

    def _config(self, precision, device):
        """The family's VbConfig at `precision` with 3 channels, for the caller to fill and hand to `_open`.  A field assigned
        directly refuses a non-integer with ctypes' TypeError; `_create` converts with int() instead."""
        self.precision = precision
        self.device = int(device)
        cfg = _lib.VbConfig()
        cfg.struct_size = C.sizeof(_lib.VbConfig)
        cfg.kind = _lib.KIND[self._kind]
        if precision not in _lib.PRECISION:
            raise ValueError(f"precision must be one of {sorted(_lib.PRECISION)}")
        cfg.precision = _lib.PRECISION[precision]
        cfg.channels = 3
        self._cfg = cfg
        return cfg

    def _open(self, cfg, create="vb_create", ext=None):
        """Create the engine handle and read its weight list.  A family with an extension config passes the filled struct as
        `ext` and its entry point as `create` (e.g. "vb_create_levit")."""
        self._lib = _lib.load()
        h = C.c_void_p()
        if ext is None:
            _lib.check(getattr(self._lib, create)(C.byref(cfg), self.device, C.byref(h)))
        else:
            ext.struct_size = C.sizeof(ext)
            _lib.check(getattr(self._lib, create)(C.byref(cfg), C.byref(ext), self.device, C.byref(h)))
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
        """The reference's initial distributions, drawn from one generator in weight-list order (see `_initial_value`)."""
        rng = np.random.default_rng(seed)
        self.set_weights_dict(collections.OrderedDict((name, self._initial_value(name, shape, rng).astype(np.float32))
                                                      for name, shape in self._specs.items() if name not in self._encoder_names))

    def _initial_value(self, name, shape, rng):
        """Keras' defaults by leaf name: Conv2D / Dense kernels glorot-uniform over the receptive field (a depthwise kernel
        [k, k, 1, dim] has fan_in k^2 and fan_out k^2 * dim), zero biases, LayerNorm / LayerNormalization / BatchNormalization
        gamma 1 and beta 0 with moving statistics 0 and 1, Embedding U(-0.05, 0.05); LayerScale fill (cait.py:36-44), CCT's
        positional embedding (cct.py:251-254) and the tf.random.normal Variables of _NORMAL_LEAVES."""
        leaf = name.rsplit(".", 1)[-1]
        if leaf == "kernel":
            receptive = int(np.prod(shape[:-2]))              # Conv2D kernel [k, k, cin, cout]: fans count the window (1 for Dense)
            lim = np.sqrt(6.0 / (receptive * (shape[-2] + shape[-1])))
            return rng.uniform(-lim, lim, size=shape)
        if leaf in ("bias", "beta", "b", "moving_mean"):
            return np.zeros(shape)
        if leaf in ("gamma", "g", "moving_variance"):
            return np.ones(shape)
        if leaf == "embeddings":
            return rng.uniform(-0.05, 0.05, size=shape)
        if leaf in ("attn_scale", "ff_scale"):
            layer = int(name.split(".layers.")[1].split(".")[0])
            return np.full(shape, _layerscale_eps(layer + 1))
        if leaf == "positional_emb":
            return (sinusoidal_embedding(shape[1], shape[2]) if self._positional_embedding == "sine"
                    else _truncated_normal(rng, shape, 0.2))
        if leaf in self._NORMAL_LEAVES:
            return rng.standard_normal(shape)
        raise AssertionError(f"{type(self).__name__}: no initial distribution for weight {name!r}")

    def set_weights_dict(self, weights):
        """weights: mapping name -> array in the Keras layout (SURVEY.md App. B).  Missing names keep their value."""
        for name, arr in weights.items():
            if name not in self._specs:
                raise KeyError(f"{type(self).__name__} has no weight named {name!r}")
            a = np.asarray(arr, dtype=np.float32, order="C")   # (not ascontiguousarray: a scalar weight keeps shape ())
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
        if self._inference_only is not None:
            if training is None or training:
                raise NotImplementedError(self._inference_only)
        elif training and any(r != 0 for r in self._dropout_rates):
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

    def __init_subclass__(cls, **kwargs):
        """Keras' name of the forward: every class's `call` is its own `__call__`, so it keeps that call's signature.  This
        replaces any `call` a subclass defines: a family changes its forward through `__call__`."""
        super().__init_subclass__(**kwargs)
        cls.call = cls.__call__

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
        return _forward_distill(self, img, distill_token)


def _distill_token(model, distill_token):
    """The caller's distillation token `[1, 1, dim]` (distill.py:101) as a flat float32 vector of `dim` values."""
    tok = np.ascontiguousarray(distill_token, dtype=np.float32).reshape(-1)
    if tok.size != model.dim:
        raise ValueError(f"distill_token must hold dim = {model.dim} values, got shape {np.shape(distill_token)}")
    return tok


def _forward_distill(model, img, distill_token):
    """DistillMixin.call with a token (distill.py:17-45) on the engine: vb_forward_distill -> (logits, distill_tokens [b, dim])."""
    model._finalize()
    x = model._img(img)
    tok = _distill_token(model, distill_token)
    b, h, w, _ = x.shape
    logits = np.empty((b, model.num_classes), np.float32)
    dist = np.empty((b, model.dim), np.float32)
    _lib.check(model._lib.vb_forward_distill(model._h, x.ctypes.data_as(C.c_void_p), _lib.MEM_HOST, b, h, w,
                                             tok.ctypes.data_as(C.c_void_p), logits.ctypes.data_as(C.c_void_p),
                                             dist.ctypes.data_as(C.c_void_p), _lib.MEM_HOST, None), model._h)
    return _as_tensor(logits), _as_tensor(dist)


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


class DistillableT2TViT(T2TViT):
    """distill.py:61-72 (DistillMixin.call distill.py:16-45): a T2TViT whose call takes an optional distillation token
    `[1, 1, dim]`; with it the call returns `(logits, distill_tokens [b, dim])`, without it plain T2TViT logits.  With an
    injected `transformer=` the call is composed on the host around it.  Forward only, as DistillableViT."""

    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self.args, self.kwargs = args, kwargs
        self.dim, self.num_classes = kwargs["dim"], kwargs["num_classes"]

    def __call__(self, img, distill_token=None, training=True):
        if distill_token is None:
            return super().__call__(img, training=training)
        self._check_training(training)
        if self._injected is None:
            return _forward_distill(self, img, distill_token)
        tok = _distill_token(self, distill_token)
        x = self.forward_embed(img)                                   # distill.py:19-24: n + 1 rows
        x = np.concatenate([x, np.broadcast_to(tok, (x.shape[0], 1, self.dim))], axis=1)   # :26-28: the token as the last row
        x = np.asarray(self._injected(x, training=training), dtype=np.float32)             # :30, _attend :69-72
        return self.forward_head(x[:, :-1]), _as_tensor(np.ascontiguousarray(x[:, -1]))    # :32-43


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


class DistillableEfficientViT(EfficientViT):
    """distill.py:74-85 as the reference runs it: its `_attend` reads `self.dropout` (:83), which efficient.ViT never defines
    (efficient.py:13-55), so every call, with or without a token, raises AttributeError (SURVEY.md App. D).  It constructs and
    carries `dim`, `num_classes`, `args` and `kwargs`, which DistillWrapper's constructor reads (distill.py:91-97)."""

    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        del self.dropout                                  # the shell's identity stand-in; efficient.ViT has no `dropout`
        self.args, self.kwargs = args, kwargs
        self.dim, self.num_classes = kwargs["dim"], kwargs["num_classes"]

    def __call__(self, img, distill_token=None, training=True):
        raise AttributeError(f"'{type(self).__name__}' object has no attribute 'dropout'")


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
    _inference_only = ("CCT runs inference only: the reference's call resolves training=None to True and then applies its "
                       "hard-coded attention dropout and stochastic depth of 0.1 (cct.py:336-338); pass training=False")

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

    def __call__(self, img, training=None, **kwargs):
        """cct.py:342: NHWC float image batch -> float32 logits [b, num_classes]; training must be False."""
        return super().__call__(img, training=training)


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
    _inference_only = ("LeViT runs inference only: with training=True (the reference's default, levit.py:214) every BatchNormalization "
                       "normalises with the batch's own statistics and dropout draws masks; pass training=False")

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
        cfg = self._config(precision, device)
        cfg.image_h, cfg.image_w, cfg.num_classes = image_size, image_size, num_classes
        cfg.dim = dims[-1]                               # the pooled width (what the engine's handle records as dim)
        lv = _lib.VbLevitConfig()
        lv.stages = stages
        for i in range(stages):
            lv.dims[i], lv.depths[i], lv.heads[i] = dims[i], depths[i], layer_heads[i]
        lv.dim_key, lv.dim_value, lv.mlp_mult = dim_key, dim_value, mlp_mult
        lv.num_distill_classes = num_distill_classes or 0
        self._lv = lv
        self._open(cfg, "vb_create_levit", lv)
        self.init_weights(seed)

    def _initial_value(self, name, shape, rng):
        if ".to_out." in name and name.endswith(".gamma"):    # the to_out BatchNormalization starts at 0 (levit.py:91)
            return np.zeros(shape)
        return super()._initial_value(name, shape, rng)

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
    _inference_only = ("CvT runs inference only: with training=True (the reference's default, cvt.py:200) every BatchNormalization "
                       "normalises with the batch's own statistics and dropout draws masks; pass training=False")

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
        cfg = self._config(precision, device)
        cfg.num_classes, cfg.dim = num_classes, self.stages[-1]["emb_dim"]
        cv = _lib.VbCvtConfig()
        for i, st in enumerate(self.stages):
            for k in CVT_STAGE_KEYS:
                getattr(cv, k)[i] = int(st[k])
        self._cv = cv
        self._open(cfg, "vb_create_cvt", cv)
        self.init_weights(seed)

    def __call__(self, img, training=True, **kwargs):
        """cvt.py:200: NHWC float images of any size -> logits [b, num_classes].  training must be False."""
        return super().__call__(img, training=training)


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
        cfg = self._config(precision, device)
        cfg.num_classes, cfg.dim = num_classes, self.stages[-1]["emb_dim"]
        tw = _lib.VbTwinsSvtConfig()
        for i, st in enumerate(self.stages):
            for k in TWINS_STAGE_KEYS:
                getattr(tw, k)[i] = int(st[k])
        tw.peg_kernel_size = int(peg_kernel_size)
        self._tw = tw
        self._open(cfg, "vb_create_twins_svt", tw)
        self.init_weights(seed)

    def __call__(self, img, training=True, **kwargs):
        """twins_svt.py:266-268: NHWC float images -> logits [b, num_classes]; extra kwargs are accepted and ignored, as there."""
        x = np.asarray(img)
        if x.ndim == 4:
            err = twins_size_error(self.stages, x.shape[1], x.shape[2])
            if err is not None:
                raise ValueError(err)
        return super().__call__(img, training=training)


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
        cfg = self._config(precision, device)
        cfg.num_classes, cfg.dim = num_classes, self.stages[-1]["dim"]
        cf = _lib.VbCrossformerConfig()
        for i, st in enumerate(self.stages):
            for k in ("dim", "depth", "global_wsz", "local_wsz", "stride"):
                getattr(cf, k)[i] = st[k]
            cf.n_kernels[i] = len(st["kernels"])
            for j, k in enumerate(st["kernels"]):
                cf.kernels[i][j] = int(k)
        self._cf = cf
        self._open(cfg, "vb_create_crossformer", cf)
        self.init_weights(seed)

    def __call__(self, img, training=True, **kwargs):
        """crossformer.py:263-269: NHWC float images -> logits [b, num_classes]; extra kwargs are accepted and ignored, as there."""
        x = np.asarray(img)
        if x.ndim == 4:
            err = crossformer_size_error(self.stages, x.shape[1], x.shape[2])
            if err is not None:
                raise ValueError(err)
        return super().__call__(img, training=training)


CROSSFORMER_CTOR_KEYS = ("dim", "depth", "global_window_size", "local_window_size", "cross_embed_kernel_sizes", "cross_embed_strides",
                         "num_classes", "attn_dropout", "ff_dropout")


def nest_plan(image_size, patch_size, dim, heads, num_hierarchies, block_repeats):
    """NesT.__init__'s construction (nest.py:163-194) as data: seq_len and the levels the zip of hierarchies, heads, dim pairs and
    the cast_tuple'd block_repeats leaves (a longer tuple is truncated, a shorter one gives fewer levels, each keeping its
    is_last / width / heads).  Raises what the reference raises for a bad block_repeats entry (range(depth), :131)."""
    assert (image_size % patch_size) == 0, 'Image dimensions must be divisible by the patch size.'
    if not 1 <= num_hierarchies <= _lib.NEST_MAX_LEVELS:
        raise ValueError(f"NesT: num_hierarchies {num_hierarchies} is not supported (1 to {_lib.NEST_MAX_LEVELS})")
    fmap_size = image_size // patch_size
    seq_len = (fmap_size // 2 ** (num_hierarchies - 1)) ** 2
    block_repeats = _cast_tuple(block_repeats, num_hierarchies)
    levels = []
    for i, depth in zip(range(num_hierarchies), block_repeats):
        len(range(depth))                               # the reference's `for _ in range(depth)`: TypeError for a non-int
        levels.append(dict(dim=dim * 2 ** i, heads=heads * 2 ** i, depth=int(depth), aggregate=i != num_hierarchies - 1))
    return dict(patch_size=patch_size, dim=dim, heads=heads, num_hierarchies=num_hierarchies, seq_len=seq_len, levels=levels,
                last_dim=dim * 2 ** (num_hierarchies - 1))


def nest_size_error(plan, h, w):
    """The reference's shape rules (nest.py:179,209,140-142 through einops, and the head LayerNorm's broadcast) for an h x w image:
    None, or what the first level that breaks one says."""
    p = plan["patch_size"]
    if h % p or w % p:
        return f"NesT: the {h} x {w} image is not divisible by patch_size {p}"
    h, w = h // p, w // p
    n = len(plan["levels"])
    for i, lv in enumerate(plan["levels"]):
        bs = 2 ** (n - 1 - i)
        if h % bs or w % bs:
            return f"NesT level {i}: the {h} x {w} map is not divisible into {bs} x {bs} blocks"
        if (h // bs) * (w // bs) > plan["seq_len"]:
            return (f"NesT level {i}: the {h} x {w} map has blocks of {h // bs} x {w // bs} tokens, more than seq_len "
                    f"{plan['seq_len']} positions")
        if lv["aggregate"]:
            h, w = -(-h // 2), -(-w // 2)
    final = plan["dim"] if n == 0 else plan["levels"][-1]["dim"] * (2 if plan["levels"][-1]["aggregate"] else 1)
    if final != plan["last_dim"]:
        return (f"NesT: the last map has {final} channels but the head's LayerNorm has {plan['last_dim']} (block_repeats has fewer "
                "than num_hierarchies - 1 entries)")
    return None


class NesT(_EngineModel):
    """nest.py:150-216: a patch embedding (patches with c fastest, 1x1 Conv2D), then per level i (bottom first, width dim * 2^i,
    heads * 2^i heads of dim // heads) the map split into 2^level x 2^level contiguous blocks, a Transformer (+ pos_emb[:h w], one
    scalar per in-block position on every channel; block_repeats[i] x [PreNorm attention within the block, PreNorm MLP], each
    residual) and, below the top, an Aggregate (Conv2D(3, SAME), LayerNorm, MaxPool2D(3, 2, SAME)); then LayerNorm per pixel, the
    mean over the map and Dense(num_classes).  Every LayerNorm is the module's own (eps 1e-5).

    block_repeats is zipped with the hierarchies as in the reference: a longer tuple is truncated and a shorter one builds fewer
    levels.  One handle runs any image whose sides are multiples of patch_size and whose maps are whole blocks of at most seq_len
    tokens at every level; other sizes raise ValueError naming the level.  There is no BatchNormalization, so with dropout = 0
    training=True computes what training=False does; with dropout > 0 only training=False runs.  Weights (SURVEY.md App. B) keep
    the reference's attribute paths: patch_embedding.1, nest_layers.{i}.0.pos_emb, nest_layers.{i}.0.layers.{l}.{0|1}.norm,
    ....0.fn.to_qkv / to_out.0, ....1.fn.net.{0|3}, nest_layers.{i}.1.ag_layers.{0|1}, mlp_head.0 (LayerNorm), mlp_head.2."""
    _kind = "nest"

    def __init__(self,
                 image_size,
                 patch_size,
                 num_classes,
                 dim,
                 heads,
                 num_hierarchies,
                 block_repeats,
                 mlp_mult=4,
                 dropout=0.0,
                 *, precision="bf16", device=0, seed=None):
        self.plan = nest_plan(image_size, patch_size, dim, heads, num_hierarchies, block_repeats)
        self.num_classes = num_classes
        self._dropout_rates = (dropout,)
        cfg = self._config(precision, device)
        cfg.num_classes, cfg.dim = num_classes, self.plan["last_dim"]
        nc = _lib.VbNestConfig()
        nc.patch_size, nc.dim, nc.heads, nc.num_hierarchies = patch_size, dim, heads, num_hierarchies
        nc.levels = len(self.plan["levels"])
        for i, lv in enumerate(self.plan["levels"]):
            nc.block_repeats[i] = lv["depth"]
        nc.mlp_mult, nc.seq_len = mlp_mult, self.plan["seq_len"]
        self._nc = nc
        self._open(cfg, "vb_create_nest", nc)
        self.init_weights(seed)

    def __call__(self, img, training=True, **kwargs):
        """nest.py:202-216: NHWC float images -> logits [b, num_classes]; extra kwargs are accepted and ignored, as there."""
        x = np.asarray(img)
        if x.ndim == 4:
            err = nest_size_error(self.plan, x.shape[1], x.shape[2])
            if err is not None:
                raise ValueError(err)
        return super().__call__(img, training=training)


NEST_CTOR_KEYS = ("image_size", "patch_size", "num_classes", "dim", "heads", "num_hierarchies", "block_repeats", "mlp_mult", "dropout")


def regionvit_maps(h, w, local_patch_size, window_size):
    """The (local, region) map sides of every RegionViT stage for an h x w image: the local encoder's SAME stride 4 (or two SAME
    stride 2) gives ceil(h / 4), the region encoder h // (local_patch_size * window_size), each Downsample ceil(. / 2)."""
    p = local_patch_size * window_size
    lh, lw, rh, rw = -(-h // 4), -(-w // 4), h // p, w // p
    maps = []
    for s in range(4):
        if s:
            lh, lw, rh, rw = -(-lh // 2), -(-lw // 2), -(-rh // 2), -(-rw // 2)
        maps.append(((lh, lw), (rh, rw)))
    return maps


def regionvit_size_error(h, w, local_patch_size, window_size):
    """The shape rules the reference enforces after its call-time asserts (regionvit.py:163-168 through einops and the concat,
    :153 through the Embedding lookup) for an h x w image: None, or what the first stage that breaks one says."""
    for s, ((lh, lw), (rh, rw)) in enumerate(regionvit_maps(h, w, local_patch_size, window_size), 1):
        where = f"RegionViT stage {s}: the {lh} x {lw} local map and the {rh} x {rw} region map "
        if lh < rh or lw < rw or lh % rh or lw % rw:
            return where + "do not make whole windows (the local map must be the region map times the window)"
        if lh // rh > window_size or lw // rw > window_size:
            return (where + f"make {lh // rh} x {lw // rw} windows, larger than window_size {window_size} (the relative-position "
                    "table's reach)")
    return None


class RegionViT(_EngineModel):
    """regionvit.py:184-263: local tokens from Conv2D(dim[0], 8, 4, SAME) (or the 3-conv tokenizer: Conv3x3 s2, LayerNorm, GELU,
    Conv3x3 s2, LayerNorm, GELU, Conv3x3), regional tokens from 'b (h p1) (w p2) c -> b h w (c p1 p2)' (p = local_patch_size *
    window_size) and a 1x1 Conv2D; per stage s the shared Downsample Conv2D(dim[s], 3, 2, SAME) of both maps (s >= 1), the PEG
    of the local map (s >= 1 with use_peg), then depth[s] R2L layers: the regional tokens attend among themselves, then every
    lh/rh x lw/rw window of local tokens attends together with its regional token under the window's relative-position bias,
    then the MLP; one Attention module (4 heads of 32) serves both attentions.  Head: the mean over the regional tokens,
    LayerNorm, Dense.  Every LayerNorm is Keras's (eps 1e-3).

    One handle runs any image the reference runs: sides divisible by the region patch size (the reference's assert messages) and,
    at every stage, a local map that is a whole number of windows of at most window_size x window_size tokens per regional
    token; other sizes raise ValueError naming the stage.  attn_dropout builds no layer in the reference and changes nothing;
    with ff_dropout > 0 only training=False runs.  Weights (SURVEY.md App. B) keep the reference's attribute paths:
    local_encoder[.{0,1,3,4,6}], region_encoder.1, region_layers.{s}.{0.conv|1.proj|2.local_rel_pos_bias},
    region_layers.{s}.2.layers.{l}.0.{norm, to_qkv, to_out}, ....1.net.{0,1,4}, to_logits.{1,2}."""
    _kind = "regionvit"

    def __init__(self,
                 dim=(64, 128, 256, 512),
                 depth=(2, 2, 8, 2),
                 window_size=7,
                 num_classes=1000,
                 tokenize_local_3_conv=False,
                 local_patch_size=4,
                 use_peg=False,
                 attn_dropout=0.0,
                 ff_dropout=0.0,
                 *, precision="bf16", device=0, seed=None):
        dim = _cast_tuple(dim, 4)                         # regionvit.py:197-200
        depth = _cast_tuple(depth, 4)
        assert len(dim) == 4, 'dim needs to be a single value or a tuple of length 4'
        assert len(depth) == 4, 'depth needs to be a single value or a tuple of length 4'
        self.dims, self.depths = tuple(int(d) for d in dim), tuple(int(d) for d in depth)
        self.window_size, self.local_patch_size = window_size, local_patch_size
        self.region_patch_size = local_patch_size * window_size
        self.tokenize_local_3_conv, self.use_peg = bool(tokenize_local_3_conv), bool(use_peg)
        self.num_classes = num_classes
        self._dropout_rates = (ff_dropout,)               # Attention never builds its Dropout (:80-91)
        cfg = self._config(precision, device)
        cfg.num_classes, cfg.dim = num_classes, self.dims[-1]
        rc = _lib.VbRegionvitConfig()
        for i in range(4):
            rc.dims[i], rc.depth[i] = self.dims[i], self.depths[i]
        rc.window_size, rc.local_patch_size = window_size, local_patch_size
        rc.tokenize_local_3_conv, rc.use_peg, rc.mlp_mult = int(self.tokenize_local_3_conv), int(self.use_peg), 4
        self._rc = rc
        self._open(cfg, "vb_create_regionvit", rc)
        self.init_weights(seed)

    def __call__(self, x, training=True, **kwargs):
        """regionvit.py:249-263: NHWC float images -> logits [b, num_classes]; extra kwargs are accepted and ignored, as there."""
        a = np.asarray(x)
        if a.ndim == 4:
            h, w = a.shape[1], a.shape[2]
            assert h % self.region_patch_size == 0 and w % self.region_patch_size == 0, \
                'height and width must be divisible by region patch size'
            assert h % self.local_patch_size == 0 and w % self.local_patch_size == 0, \
                'height and width must be divisible by local patch size'
            err = regionvit_size_error(h, w, self.local_patch_size, self.window_size)
            if err is not None:
                raise ValueError(err)
        return super().__call__(x, training=training)


class ATSViT(_EngineModel):
    """ats_vit.py:260-318 (`ats_vit.ViT`, adaptive token sampling): a ViT whose layer L keeps at most max_tokens_per_depth[L]
    tokens, drawn by Gumbel-max from the cls token's attention weighted by the value norms, whenever the batch's padded token
    count exceeds that number.  The pool is always the cls token and to_out is always present.  The draws are random whatever
    `training` is; the noise is the engine's Philox stream (include/vitb200.h), keyed by set_sampling_seed (0 at construction)
    and advancing with every layer that samples, so repeated calls draw fresh tokens.  An image's result depends on the rest of
    its batch, as in the reference.  With dropout > 0 only training=False runs.  Weights keep ViT's names (SURVEY.md App. B)."""
    _kind = "ats_vit"

    def __init__(self, image_size, patch_size, num_classes, dim, depth, max_tokens_per_depth, heads, mlp_dim, dim_head=64,
                 dropout=0.0, emb_dropout=0.0, *, precision="bf16", device=0, seed=None):
        image_height, image_width = pair(image_size)
        patch_height, patch_width = pair(patch_size)
        assert image_height % patch_height == 0 and image_width % patch_width == 0, 'Image dimensions must be divisible by the patch size.'
        assert len(max_tokens_per_depth) == depth, 'max_tokens_per_depth must be a tuple of length that is equal to the depth of the transformer'
        assert sorted(max_tokens_per_depth, reverse=True) == list(max_tokens_per_depth), 'max_tokens_per_depth must be in decreasing order'
        assert min(max_tokens_per_depth) > 0, 'max_tokens_per_depth must have at least 1 token at any layer'
        if depth > _lib.ATS_MAX_DEPTH:
            raise ValueError(f"ATS-ViT: depth must be at most {_lib.ATS_MAX_DEPTH}")
        self.num_classes, self.dim = num_classes, dim
        self.max_tokens_per_depth = tuple(int(k) for k in max_tokens_per_depth)
        self._dropout_rates = (dropout, emb_dropout)
        ac = _lib.VbAtsVitConfig()
        for i, k in enumerate(self.max_tokens_per_depth):
            ac.max_tokens_per_depth[i] = k
        self._ac = ac
        self._create(precision, device, ext=ac, create="vb_create_ats_vit", image_h=image_height, image_w=image_width,
                     patch_h=patch_height, patch_w=patch_width, num_classes=num_classes, dim=dim, depth=depth, heads=heads,
                     dim_head=dim_head, mlp_dim=mlp_dim)
        self.init_weights(seed)

    def set_sampling_seed(self, seed):
        """The Philox key of the sampling noise; also restarts its draw counter, so the next calls repeat the draws made after
        the previous set_sampling_seed(seed) (on the same images and batch)."""
        _lib.check(self._lib.vb_ats_set_seed(self._h, int(seed) & 0xFFFFFFFFFFFFFFFF), self._h)

    def forward_ats(self, img, stream=None):
        """One forward: (logits [b, num_classes], token_ids [b, count]) with the reference's id layout (ats_vit.py:313-316).
        stream: a cudaStream_t, as in forward_raw (the forward is captured into a CUDA graph on its second call there)."""
        self._finalize()
        x = self._img(img)
        b, h, w, _ = x.shape
        logits = np.empty((b, self.num_classes), np.float32)
        self._last_batch = b
        ids = np.empty((b, self._last_pitch(h, w) - 1), np.int32)
        count = C.c_int32()
        _lib.check(self._lib.vb_forward_ats(self._h, x.ctypes.data_as(C.c_void_p), _lib.MEM_HOST, b, h, w, logits.ctypes.data_as(C.c_void_p),
                                            ids.ctypes.data_as(C.c_void_p), C.byref(count), C.c_void_p(stream) if stream else None),
                   self._h)
        return logits, ids[:, :count.value].copy()

    def _last_pitch(self, h, w):
        """Rows of the last layer: P_0 = patches + 1, P_{L+1} = 1 + min(P_L - 1, K_L)."""
        p = (h // self._cfg.patch_h) * (w // self._cfg.patch_w) + 1
        for k in self.max_tokens_per_depth:
            p = 1 + min(p - 1, k)
        return p

    def last_draws(self, layer):
        """After a forward: (draws [b, K] as argmax + 1 in the reference's left-padded layout, counts [b] of tokens kept, sampled)
        of a layer that can sample; when it did not sample (the batch already had at most K tokens) sampled is False and the
        draws are -1."""
        k = self.max_tokens_per_depth[layer]
        b = self._last_batch
        draws, counts, sampled = np.empty((b, k), np.int32), np.empty((b,), np.int32), C.c_int32()
        _lib.check(self._lib.vb_ats_last_draws(self._h, layer, draws.ctypes.data_as(C.c_void_p), counts.ctypes.data_as(C.c_void_p),
                                               C.byref(sampled)), self._h)
        return draws, counts, bool(sampled.value)

    def forward_raw(self, img_ptr, img_mem, batch, h, w, logits_ptr, logits_mem, stream=None):
        self._last_batch = batch
        super().forward_raw(img_ptr, img_mem, batch, h, w, logits_ptr, logits_mem, stream)

    def __call__(self, img, return_sampled_token_ids=False, training=True, **kwargs):
        """ats_vit.py:300-318: NHWC images -> logits, or (logits, token_ids) with return_sampled_token_ids."""
        self._check_training(training)
        logits, ids = self.forward_ats(img)
        if return_sampled_token_ids:
            return _as_tensor(logits), _as_tensor(ids)
        return _as_tensor(logits)


class _WrapperModel(_EngineModel):
    """A handle of its own that also registers the weights of the model it wraps (the attribute `_wrapped_name`): those stay
    the wrapped model's, and their current values are pushed into this handle before every call that follows a change."""
    _wrapped_name = None

    def _share_weights(self):
        self._encoder_names = tuple(n for n in self._specs if n in getattr(self, self._wrapped_name)._specs)
        self._pushed = {}

    def set_weights_dict(self, weights):
        """The model's own weights (SURVEY.md App. B); the wrapped model's are set on it and picked up by the next call."""
        shared = [n for n in weights if n in self._encoder_names]
        if shared:
            w = self._wrapped_name
            raise KeyError(f"{type(self).__name__}: {shared[0]!r} belongs to the {w}: set it with {w}.set_weights_dict")
        super().set_weights_dict(weights)

    def _push_wrapped(self):
        src = getattr(self, self._wrapped_name)
        changed = collections.OrderedDict((n, src.get_weight(n)) for n in self._encoder_names
                                          if self._pushed.get(n) is not src.get_weight(n))
        if changed:
            _EngineModel.set_weights_dict(self, changed)
            self._pushed.update(changed)

    def _finalize(self):
        self._push_wrapped()
        super()._finalize()


class _MaskedImageModel(_WrapperModel):
    """What MAE and SimMIM share: a handle of their own built from the encoder ViT's configuration, the encoder's current weights
    pushed into it before every call that follows a change, the engine's mask noise (set_seed) and the call itself."""
    _wrapped_name = "encoder"

    def _build(self, image_size, encoder, masking_ratio, seed, decoder=(0, 0, 0, 0), mc=None):
        if not (isinstance(encoder, ViT) and encoder._kind == "vit"):
            raise TypeError(f"{type(self).__name__}: the encoder must be a vit_tensorflow_b200.ViT (or DistillableViT), got "
                            f"{type(encoder).__name__}")
        encoder.build(input_shape=(1, image_size, image_size, 3))      # mae.py:32, simmim.py:77
        self.encoder = encoder
        self.masking_ratio = masking_ratio
        self._dropout_rates = encoder._dropout_rates
        ec = encoder._cfg
        mc = _lib.VbMimConfig() if mc is None else mc                   # MPP passes its VbMppConfig
        mc.masking_ratio = float(masking_ratio)
        mc.decoder_dim, mc.decoder_depth, mc.decoder_heads, mc.decoder_dim_head = (int(v) for v in decoder)
        self._mc = mc
        self._create(encoder.precision, encoder.device, ext=mc, create="vb_create_mim", image_h=ec.image_h, image_w=ec.image_w,
                     patch_h=ec.patch_h, patch_w=ec.patch_w, num_classes=ec.num_classes, dim=ec.dim, depth=ec.depth, heads=ec.heads,
                     dim_head=ec.dim_head, mlp_dim=ec.mlp_dim)
        self._share_weights()
        self.init_weights(seed)                                         # the model's own weights: the encoder keeps its own

    def set_seed(self, seed):
        """The Philox key of the mask noise (include/vitb200.h); also restarts its draw counter, so the next calls repeat the masks
        drawn after the previous set_seed(seed).  The seed is 0 at construction."""
        _lib.check(self._lib.vb_mim_set_seed(self._h, int(seed) & 0xFFFFFFFFFFFFFFFF), self._h)

    def _shapes(self, h, w):
        ph, pw = self._cfg.patch_h, self._cfg.patch_w
        if h % ph or w % pw:
            raise ValueError("Image dimensions must be divisible by the patch size.")
        n = (h // ph) * (w // pw)
        return n, int(self.masking_ratio * n), ph * pw * 3

    def forward_raw(self, img_ptr, img_mem, batch, h, w, loss_ptr, out_mem, stream=None, pred_ptr=None, patches_ptr=None,
                    indices_ptr=None):
        """Pointer-level call (vb_forward_mim): host or device buffers, optional cudaStream_t; pred / masked_patches [batch,
        num_masked, patch_dim] and indices [batch, n] are written when their pointers are given."""
        self._finalize()
        p = [C.c_void_p(v) if v else None for v in (pred_ptr, patches_ptr, indices_ptr)]
        _lib.check(self._lib.vb_forward_mim(self._h, C.c_void_p(img_ptr), img_mem, batch, h, w, C.c_void_p(loss_ptr), *p, out_mem,
                                            C.c_void_p(stream) if stream else None), self._h)

    def forward_mim(self, img, stream=None):
        """One call: (loss, pred [b, num_masked, patch_dim], masked_patches [b, num_masked, patch_dim], indices [b, n]).  indices
        is each image's noise permutation with the masked patch ids first; masked_patches are the image's patches at those ids, so
        mean((pred - masked_patches) ** 2) is the MSE the MAE paper trains with."""
        x = self._img(img)
        b, h, w, _ = x.shape
        n, nm, pd = self._shapes(h, w)
        loss = np.zeros(1, np.float32)
        pred, patches = np.empty((b, nm, pd), np.float32), np.empty((b, nm, pd), np.float32)
        idx = np.empty((b, n), np.int32)
        self.forward_raw(x.ctypes.data, _lib.MEM_HOST, b, h, w, loss.ctypes.data, _lib.MEM_HOST, stream, pred.ctypes.data,
                         patches.ctypes.data, idx.ctypes.data)
        return _as_tensor(loss.reshape(())), _as_tensor(pred), _as_tensor(patches), idx

    def __call__(self, img, training=True, **kwargs):
        """The reference's call: the reconstruction loss as a float32 0-d array (answers `.numpy()`)."""
        self._check_training(training)
        x = self._img(img)
        b, h, w, _ = x.shape
        self._shapes(h, w)
        loss = np.zeros(1, np.float32)
        self.forward_raw(x.ctypes.data, _lib.MEM_HOST, b, h, w, loss.ctypes.data, _lib.MEM_HOST)
        return _as_tensor(loss.reshape(()))


class MAE(_MaskedImageModel):
    """mae.py:17-92 (masked autoencoder): the encoder ViT over a random quarter (1 - masking_ratio) of the patches, the decoder
    over those and mask tokens, pixels predicted for the masked patches.  The call returns what the reference returns,
    mean(pred^2): its tf.square(pred, masked_patches) passes the patches as tf.square's `name` (SURVEY.md App. D); forward_mim
    also returns the masked patches.  The masks come from the engine's Philox noise (set_seed); precision and device are the
    encoder's, and the encoder's weights are read at every call that follows a change."""
    _kind = "mae"

    def __init__(self, image_size, encoder, decoder_dim, masking_ratio=0.75, decoder_depth=1, decoder_heads=8, decoder_dim_head=64, *,
                 seed=None):
        assert masking_ratio > 0 and masking_ratio < 1, 'masking ratio must be kept between 0 and 1'
        self.decoder_dim = decoder_dim
        self._build(image_size, encoder, masking_ratio, seed, (decoder_dim, decoder_depth, decoder_heads, decoder_dim_head))


class SimMIM(_MaskedImageModel):
    """simmim.py:72-129: the encoder ViT over all patches with the masked ones replaced by the mask token, a linear head on the
    masked rows, loss mean(|pred - masked_patches|) / num_masked (the reference's extra division kept).  Masks, precision, device
    and encoder weights as for MAE."""
    _kind = "simmim"

    def __init__(self, image_size, encoder, masking_ratio=0.5, *, seed=None):
        assert masking_ratio > 0 and masking_ratio < 1, 'masking ratio must be kept between 0 and 1'
        self._build(image_size, encoder, masking_ratio, seed)


class MPP(_MaskedImageModel):
    """mpp.py:133-218 (masked patch prediction): ceil(mask_prob * n) patches per image masked by the top_k of the engine's Philox
    noise, each masked patch replaced by the original patch at a random id (random-patch coin) and then by the pixel-space
    mask_token (replace coin), the encoder ViT (cls row included) over the corrupted image, to_bits on the masked rows.  The call
    returns the loss TF computes from mpp.py:128 as written: ln(K) times the mean over the masked rows of the sum of their logits
    (include/vitb200.h states every reading).  Draws, precision, device and encoder weights as for MAE."""
    _kind = "mpp"

    def __init__(self, image_size, transformer, patch_size, output_channel_bits=3, channels=3, max_pixel_val=1.0, mask_prob=0.15,
                 replace_prob=0.5, random_patch_prob=0.5, mean=None, std=None, *, seed=None):
        if isinstance(transformer, ViT) and not (isinstance(patch_size, int) and
                                                 (transformer._cfg.patch_h, transformer._cfg.patch_w) == (patch_size, patch_size)):
            raise ValueError(f"MPP: patch_size must be one int equal to both of the encoder's patch sides "
                             f"({transformer._cfg.patch_h} x {transformer._cfg.patch_w}); got {patch_size!r}")
        if channels != 3:
            raise ValueError(f"MPP: images of 3 channels (the encoder's patch Dense reads 3); got channels={channels!r}")
        if output_channel_bits * channels > 16:
            raise ValueError(f"MPP: to_bits would have 2^{output_channel_bits * channels} classes; at most 2^16 are supported")
        self.patch_size, self.output_channel_bits, self.channels = patch_size, output_channel_bits, channels
        self.max_pixel_val = max_pixel_val                               # no effect on the loss (see include/vitb200.h)
        self.mask_prob, self.replace_prob, self.random_patch_prob = mask_prob, replace_prob, random_patch_prob
        self.mean, self.std = mean, std
        mc = _lib.VbMppConfig()
        mc.mask_prob, mc.replace_prob, mc.random_patch_prob = float(mask_prob), float(replace_prob), float(random_patch_prob)
        mc.output_channel_bits = int(output_channel_bits)
        self._build(image_size, transformer, mask_prob, seed, mc=mc)
        self.transformer = self.encoder

    def _shapes(self, h, w):
        p = self.patch_size
        if h % p or w % p:
            raise ValueError("Image dimensions must be divisible by the patch size.")
        if self.random_patch_prob > 0:
            self.random_patch_prob / (1 - self.replace_prob)              # mpp.py:185: ZeroDivisionError when replace_prob == 1
        if self.mean and self.std:                                       # mpp.py:105-106,113-114: [c, 1, 1] against NHWC
            for v in (self.mean, self.std):
                c = int(np.size(v))
                if not (h == c or h == 1 or c == 1):
                    raise ValueError(f"MPP: mean / std of {c} values reshaped to [{c}, 1, 1] do not broadcast against images of "
                                     f"height {h} (mpp.py:114)")
        n = (h // p) * (w // p)
        return n, math.ceil(self.mask_prob * n), 2 ** (self.output_channel_bits * self.channels)

    def forward_raw(self, img_ptr, img_mem, batch, h, w, loss_ptr, out_mem, stream=None, logits_ptr=None, mask_ids_ptr=None,
                    source_ptr=None):
        """Pointer-level call (vb_forward_mpp): host or device buffers, optional cudaStream_t; logits [batch, k, K], mask_ids
        [batch, k] and source [batch, n] are written when their pointers are given."""
        self._finalize()
        p = [C.c_void_p(v) if v else None for v in (logits_ptr, mask_ids_ptr, source_ptr)]
        _lib.check(self._lib.vb_forward_mpp(self._h, C.c_void_p(img_ptr), img_mem, batch, h, w, C.c_void_p(loss_ptr), *p, out_mem,
                                            C.c_void_p(stream) if stream else None), self._h)

    def forward_mpp(self, img, stream=None):
        """One call: (loss, logits [b, k, K] of the masked rows, mask_ids [b, k] ascending, source [b, n]).  source[b, j] is j
        for an unchanged position, the random patch id whose pixels it took, or -1 where it took the mask token."""
        x = self._img(img)
        b, h, w, _ = x.shape
        n, k, K = self._shapes(h, w)
        loss = np.zeros(1, np.float32)
        logits, ids, src = np.empty((b, k, K), np.float32), np.empty((b, k), np.int32), np.empty((b, n), np.int32)
        self.forward_raw(x.ctypes.data, _lib.MEM_HOST, b, h, w, loss.ctypes.data, _lib.MEM_HOST, stream, logits.ctypes.data,
                         ids.ctypes.data, src.ctypes.data)
        return _as_tensor(loss.reshape(())), _as_tensor(logits), ids, src

    def __call__(self, inputs, training=True, **kwargs):
        """The reference's call: the loss as a float32 0-d array (answers `.numpy()`)."""
        self._check_training(training)
        x = self._img(inputs)
        b, h, w, _ = x.shape
        self._shapes(h, w)
        loss = np.zeros(1, np.float32)
        self.forward_raw(x.ctypes.data, _lib.MEM_HOST, b, h, w, loss.ctypes.data, _lib.MEM_HOST)
        return _as_tensor(loss.reshape(()))


def _spt_patch_size(patch_size):
    """SPT's Rearrange gets p1 = p2 = patch_size as given (vit_for_small_dataset.py:147): a tuple passes pair() and then fails
    inside einops in the reference, so it is refused here when the model is built."""
    if isinstance(patch_size, tuple):
        raise ValueError("the small-dataset ViT's SPT takes one integer patch_size (its Rearrange uses it for both sides); "
                         f"got {patch_size!r}")
    return int(patch_size)


class SmallDatasetViT(_EngineModel):
    """vit_for_small_dataset.py:159-215 (`vit_for_small_dataset.ViT`, "Vision Transformer for Small Datasets"): ViT with shifted
    patch tokens (SPT: the image and its four one-pixel shifts, LayerNorm, Dense) and locality self-attention (LSA: each token's
    own key masked, the scale exp(temperature) a learned scalar per layer).  to_out is always present.  Weights are ViT's names
    (SURVEY.md App. B) plus patch_norm.gamma / .beta, patch.kernel / .bias over p^2 * 15 inputs and layers.L.temperature, a
    scalar.  Runs as a whole forward only.  Images must have 3 channels."""
    _kind = "small_dataset_vit"

    def __init__(self, image_size, patch_size, num_classes, dim, depth, heads, mlp_dim, pool='cls', dim_head=64, dropout=0.0,
                 emb_dropout=0.0, *, precision="bf16", device=0, seed=None):
        image_height, image_width = pair(image_size)
        patch_height, patch_width = pair(patch_size)
        assert image_height % patch_height == 0 and image_width % patch_width == 0, 'Image dimensions must be divisible by the patch size.'
        assert pool in {'cls', 'mean'}, 'pool type must be either cls (cls token) or mean (mean pooling)'
        p = _spt_patch_size(patch_size)
        self.num_classes, self.pool, self.dim, self.dim_head = num_classes, pool, dim, dim_head
        self._dropout_rates = (dropout, emb_dropout)
        self._create(precision, device, image_h=image_height, image_w=image_width, patch_h=p, patch_w=p, num_classes=num_classes,
                     dim=dim, depth=depth, heads=heads, dim_head=dim_head, mlp_dim=mlp_dim, pool=0 if pool == 'cls' else 1)
        self.init_weights(seed)

    def _initial_value(self, name, shape, rng):
        a = super()._initial_value(name, shape, rng)          # a temperature's N(0, 1) draw is made, so later weights keep theirs
        if name.endswith(".temperature"):                     # log(dim_head^-0.5) in float32 (:94)
            a = np.full(shape, np.log(np.float32(self.dim_head ** -0.5)))
        return a


class SPT:
    """vit_for_small_dataset.py:142-157 on its own: `SPT(dim, patch_size)(img)` -> tokens [b, (H / p) (W / p), dim] of NHWC images
    with 3 channels.  Weights: patch_norm.gamma / .beta [p^2 * 15] and patch.kernel [p^2 * 15, dim] / .bias (Keras' initial values
    at construction; set_weights_dict replaces them).  Runs the engine's SPT kernel and the LayerNorm-folded GEMM (vb_op_spt)."""

    def __init__(self, dim, patch_size, *, precision="bf16", seed=None):
        self.dim, self.patch_size, self.precision = int(dim), _spt_patch_size(patch_size), precision
        k = self.patch_size ** 2 * 15
        lim = np.sqrt(6.0 / (k + self.dim))
        rng = np.random.default_rng(seed)
        self._specs = collections.OrderedDict([("patch_norm.gamma", (k,)), ("patch_norm.beta", (k,)), ("patch.kernel", (k, self.dim)),
                                               ("patch.bias", (self.dim,))])
        self._weights = collections.OrderedDict([
            ("patch_norm.gamma", np.ones(k, np.float32)), ("patch_norm.beta", np.zeros(k, np.float32)),
            ("patch.kernel", rng.uniform(-lim, lim, size=(k, self.dim)).astype(np.float32)), ("patch.bias", np.zeros(self.dim, np.float32))])

    def weight_specs(self):
        return collections.OrderedDict(self._specs)

    def set_weights_dict(self, weights):
        for name, arr in weights.items():
            if name not in self._specs:
                raise KeyError(f"SPT has no weight named {name!r}")
            a = np.ascontiguousarray(arr, dtype=np.float32)
            if tuple(a.shape) != self._specs[name]:
                raise ValueError(f"weight {name!r}: expected shape {self._specs[name]}, got {tuple(a.shape)}")
            self._weights[name] = a

    def get_weights_dict(self):
        return collections.OrderedDict((k, v.copy()) for k, v in self._weights.items())

    def __call__(self, x, training=True):
        img = np.ascontiguousarray(x, dtype=np.float32)
        if img.ndim != 4 or img.shape[3] != 3:
            raise ValueError("img must be NHWC float [b, H, W, 3]")
        if img.shape[1] % self.patch_size or img.shape[2] % self.patch_size:
            raise ValueError("Image dimensions must be divisible by the patch size.")
        w = self._weights
        out = _lib.op_spt(img, self.patch_size, w["patch_norm.gamma"], w["patch_norm.beta"], w["patch.kernel"], w["patch.bias"],
                          precision=self.precision)
        return _as_tensor(out[:, 1:])

    call = __call__


SMALL_DATASET_VIT_CTOR_KEYS = ("image_size", "patch_size", "num_classes", "dim", "depth", "heads", "mlp_dim", "pool", "dim_head",
                               "dropout", "emb_dropout")


ATS_CTOR_KEYS = ("image_size", "patch_size", "num_classes", "dim", "depth", "max_tokens_per_depth", "heads", "mlp_dim", "dim_head",
                 "dropout", "emb_dropout")


REGIONVIT_CTOR_KEYS = ("dim", "depth", "window_size", "num_classes", "tokenize_local_3_conv", "local_patch_size", "use_peg",
                       "attn_dropout", "ff_dropout")


def mobilevit_size_error(h, w, ph, pw):
    """The reference's regrouping rule (mobile_vit.py:196, enforced there by einops) for an h x w image: None, or what the first
    trunk stage that breaks it says.  conv1 and the second stem block halve the map (SAME: ceil), each trunk stage halves it again."""
    h, w = -(-h // 4), -(-w // 4)
    for s in range(3):
        h, w = -(-h // 2), -(-w // 2)
        if h % ph or w % pw:
            return (f"MobileViT stage {s + 1}: the {h} x {w} map is not divisible by patch_size ({ph}, {pw}); every trunk map (1/8, 1/16 "
                    "and 1/32 of the image, rounded up) must be")
    return None


def mobilevit_blocks(channels, expansion):
    """The seven MV2 blocks as mobile_vit.py:233-252 builds them: (attribute path, actual input width, hidden, output width, stride,
    expand, residual).  Keras infers input widths, so the reference's dim_in sets only hidden = int(dim_in * expansion) and the
    residual test; the fourth stem block is built as MV2Block(channels[2], channels[3]) but reads channels[3] channels."""
    c = channels
    spec = [("stem.0", c[0], c[0], c[1], 1), ("stem.1", c[1], c[1], c[2], 2), ("stem.2", c[2], c[2], c[3], 1), ("stem.3", c[2], c[3], c[3], 1),
            ("trunk.0.0", c[3], c[3], c[4], 2), ("trunk.1.0", c[5], c[5], c[6], 2), ("trunk.2.0", c[7], c[7], c[8], 2)]
    out = []
    for path, dim_in, cin, cout, stride in spec:
        hidden = int(dim_in * expansion)
        if expansion == 1 and hidden != cin:
            raise ValueError(f"MobileViT {path}: with expansion 1 the block is MV2Block({dim_in}, {cout}) whose depthwise convolution has "
                             f"{hidden} filters with groups={hidden}, but its input has {cin} channels (channels[2] != channels[3]); "
                             "the reference builds a grouped convolution or fails there")
        out.append((path, cin, hidden, cout, stride, expansion != 1, stride == 1 and dim_in == cout))
    return out


class MobileViT(_EngineModel):
    """mobile_vit.py:209-271: a stride-2 Conv_NxN_BN, four MobileNetV2 blocks (1x1 expand, 3x3 depthwise, 1x1 project, BatchNorm and
    SiLU), three trunk stages of a stride-2 MV2 block and a MobileViTBlock (k x k and 1x1 convolutions, a Transformer of 4 heads of 8
    within each of the ph * pw patch positions, a 1x1 convolution back, the concat with the block's input and a k x k convolution),
    then a 1x1 Conv_NxN_BN, the mean over pixels and a bias-free Dense.

    Inference only: the reference's call defaults to training=True, which makes every BatchNormalization use the batch's statistics;
    a call without training=False raises NotImplementedError here.  Every trunk map (1/8, 1/16 and 1/32 of the image, rounded up)
    must be divisible by patch_size: other image sizes raise ValueError naming the stage, at construction and at call time.  With
    expansion 1 and channels[2] != channels[3] the fourth stem block is refused (ValueError).
    Weights (SURVEY.md App. B) keep the reference's attribute paths: conv1.layers.{0,1} (Conv2D, BatchNormalization),
    stem.{i}.conv.{j} and trunk.{s}.0.conv.{j} (MV2 blocks: j = 0, 1, 3, 4, 6, 7 with the expand convolution, 0, 1, 3, 4 without),
    trunk.{s}.1.conv{1,2,3,4}.layers.{0,1}, trunk.{s}.1.transformer.layers.{l}.0.{norm, fn.to_qkv, fn.to_out.0},
    trunk.{s}.1.transformer.layers.{l}.1.{norm, fn.net.0, fn.net.3}, to_logits.0.layers.{0,1}, to_logits.2 (the Dense head)."""
    _kind = "mobilevit"
    _inference_only = ("MobileViT runs inference only: with training=True (the reference's default, mobile_vit.py:260) every "
                       "BatchNormalization normalises with the batch's own statistics; pass training=False")

    def __init__(self, image_size, dims, channels, num_classes, expansion=4, kernel_size=3, patch_size=(2, 2), depths=(2, 4, 3),
                 *, precision="bf16", device=0, seed=None):
        assert len(dims) == 3, 'dims must be a tuple of 3'
        assert len(depths) == 3, 'depths must be a tuple of 3'
        ih, iw = image_size
        ph, pw = patch_size
        assert ih % ph == 0 and iw % pw == 0
        init_dim, *_, last_dim = channels
        err = mobilevit_size_error(ih, iw, ph, pw)
        if err is not None:
            raise ValueError(err + " (the reference fails at its first call)")
        self.num_classes, self.image_size, self.patch_size = num_classes, (ih, iw), (ph, pw)
        self.blocks = mobilevit_blocks(channels, expansion)
        mc = _lib.VbMobilevitConfig()
        for i in range(10):
            mc.channels[i] = int(channels[i])
        mc.last_dim = int(last_dim)
        for i in range(3):
            mc.dims[i], mc.depths[i] = int(dims[i]), int(depths[i])
        mc.kernel_size, mc.ph, mc.pw = int(kernel_size), int(ph), int(pw)
        for i, (_, cin, hidden, cout, stride, expand, residual) in enumerate(self.blocks):
            mc.mv2_in[i], mc.mv2_hidden[i], mc.mv2_out[i], mc.mv2_stride[i] = cin, hidden, cout, stride
            mc.mv2_expand[i], mc.mv2_residual[i] = int(expand), int(residual)
        self._mc = mc
        self._create(precision, device, ext=mc, create="vb_create_mobilevit", image_h=ih, image_w=iw, num_classes=num_classes,
                     dim=last_dim)
        self.init_weights(seed)

    def __call__(self, img, training=True, **kwargs):
        """mobile_vit.py:260-271: NHWC float images -> logits [b, num_classes].  training must be False."""
        self._check_training(training)
        x = np.asarray(img)
        if x.ndim == 4:
            err = mobilevit_size_error(x.shape[1], x.shape[2], *self.patch_size)
            if err is not None:
                raise ValueError(err)
        return super().__call__(img, training=False)


MOBILEVIT_CTOR_KEYS = ("image_size", "dims", "channels", "num_classes", "expansion", "kernel_size", "patch_size", "depths")


SCALABLE_VIT_STAGE_KEYS = ("heads", "ssa_dim_key", "ssa_dim_value", "reduction_factor", "iwsa_dim_key", "iwsa_dim_value", "window_size")


def scalable_vit_size_error(stages, h, w):
    """The reference's shape rules for an h x w image: None, or (exception type, message) of the first stage that breaks one, in the
    order the reference meets them.  to_patches (SAME, stride 4) and each Downsample (SAME, stride 2) round up; in every stage with
    blocks the SSA's r x r stride-r VALID convolution needs a map of at least r on each side (TensorFlow refuses a negative output
    size), and IWSA asserts that its window divides the map (scalable_vit.py:171; None is the whole map)."""
    h, w = -(-h // 4), -(-w // 4)
    for i, st in enumerate(stages, 1):
        if i > 1:
            h, w = -(-h // 2), -(-w // 2)
        if st["depth"] == 0:
            continue
        r = st["reduction_factor"]
        if h < r or w < r:
            return ValueError, f"ScalableViT stage {i}: the {h} x {w} map is smaller than reduction_factor {r} (a VALID convolution)"
        wh, ww = st["window_size"] or h, st["window_size"] or w
        if h % wh or w % ww:
            return AssertionError, (f"ScalableViT stage {i}: height ({h}) or width ({w}) of feature map is not divisible by the window size "
                                    f"({wh}, {ww})")
    return None


class ScalableViT(_EngineModel):
    """scalable_vit.py:250-319: to_patches (Conv2D(dim, 7, stride 4, SAME)), then per stage s a Transformer on dim * 2^s channels and,
    between stages, Downsample (Conv2D(2 dim_s, 3, stride 2, SAME)); then the mean over the map, LayerNormalization and Dense.  Each
    block is built [SSA, MLP, PEG (first block only), MLP, IWSA] but unpacked as ssa, ff1, peg, iwsa, ff2 (:236), so it runs SSA,
    MLP, PEG, MLP, IWSA, each but the PEG pre-norm and residual; every Transformer ends with its own LayerNorm.  SSA: q from every
    pixel against keys and values of an r x r stride-r VALID convolution, scale ssa_dim_key^-0.5.  IWSA: attention within
    window_size windows (None: the whole map), plus a full 3x3 convolution (the LIM) of v, then to_out.

    There is no image_size: any image whose stage maps (ceil(H / 4), halved and rounded up per stage) are at least reduction_factor
    on each side and divisible by their window_size runs; a map smaller than reduction_factor raises ValueError naming the stage,
    a window that does not divide its map the reference's AssertionError.  There is no BatchNormalization: with dropout = 0
    training=True computes what training=False does.  At most 4 stages.
    Weights (SURVEY.md App. B) keep the reference's attribute paths: to_patches, scalable_layers.{s}.0.layers.{l}.{j} with j the
    construction index (0 SSA: .norm, .fn.to_q / to_k / to_v / to_out.0; 1 and 3 MLP: .norm, .fn.net.0 / net.3; 2 PEG: .proj;
    4 IWSA: .norm, .fn.local_interactive_module / to_q / to_k / to_v / to_out.0), scalable_layers.{s}.0.norm,
    scalable_layers.{s}.1.conv (Downsample), mlp_head.1 (LayerNormalization), mlp_head.2 (Dense)."""
    _kind = "scalable_vit"

    def __init__(self, num_classes, dim, depth, heads, reduction_factor, window_size=None, iwsa_dim_key=32, iwsa_dim_value=32,
                 ssa_dim_key=32, ssa_dim_value=32, ff_expansion_factor=4, channels=3, dropout=0.0, *, precision="bf16", device=0,
                 seed=None):
        assert isinstance(depth, tuple), 'depth needs to be tuple if integers indicating number of transformer blocks at that stage'
        num_stages = len(depth)
        per_stage = [_cast_tuple(v, num_stages) for v in (heads, ssa_dim_key, ssa_dim_value, reduction_factor, iwsa_dim_key,
                                                          iwsa_dim_value, window_size)]
        assert all(len(a) == num_stages for a in per_stage)
        if not 1 <= num_stages <= _lib.SCALABLE_VIT_STAGES:
            raise NotImplementedError(f"ScalableViT: the engine runs 1 to {_lib.SCALABLE_VIT_STAGES} stages; depth has {num_stages} entries")
        self.num_classes, self.channels = num_classes, channels
        self.stages = tuple(dict(depth=depth[i], **{k: per_stage[j][i] for j, k in enumerate(SCALABLE_VIT_STAGE_KEYS)})
                            for i in range(num_stages))
        self._dropout_rates = (dropout,)
        sc = _lib.VbScalableVitConfig()
        sc.num_stages = num_stages
        sc.ff_expansion_factor = int(ff_expansion_factor)
        for i, st in enumerate(self.stages):
            sc.dim[i], sc.depth[i] = int(dim) << i, int(st["depth"])
            for k in SCALABLE_VIT_STAGE_KEYS[:-1]:
                getattr(sc, k)[i] = int(st[k])
            sc.window[i] = 0 if st["window_size"] is None else int(st["window_size"])
            if st["window_size"] is not None and sc.window[i] <= 0:
                raise ValueError(f"ScalableViT stage {i + 1}: window_size must be positive or None")
        self._sc = sc
        self._create(precision, device, ext=sc, create="vb_create_scalable_vit", channels=channels, num_classes=num_classes,
                     dim=int(dim) << (num_stages - 1))
        self.init_weights(seed)

    def __call__(self, img, training=True, **kwargs):
        """scalable_vit.py:308-319: NHWC float images [b, H, W, channels] -> logits [b, num_classes]; extra kwargs are accepted and
        ignored, as there."""
        self._check_training(training)
        x = np.ascontiguousarray(img, dtype=np.float32)
        if x.ndim != 4 or x.shape[3] != self.channels:
            raise ValueError(f"ScalableViT: img must be NHWC float [b, H, W, {self.channels}] (channels={self.channels}), got shape "
                             f"{tuple(x.shape)}")
        err = scalable_vit_size_error(self.stages, x.shape[1], x.shape[2])
        if err is not None:
            raise err[0](err[1])
        b, h, w, _ = x.shape
        out = np.empty((b, self.num_classes), np.float32)
        self.forward_raw(x.ctypes.data, _lib.MEM_HOST, b, h, w, out.ctypes.data, _lib.MEM_HOST, None)
        return _as_tensor(out)


SCALABLE_VIT_CTOR_KEYS = ("num_classes", "dim", "depth", "heads", "reduction_factor", "window_size", "iwsa_dim_key", "iwsa_dim_value",
                          "ssa_dim_key", "ssa_dim_value", "ff_expansion_factor", "channels", "dropout")


def pit_stages(depth, heads):
    """pit.py:177,193: heads = cast_tuple(heads, len(depth)), then zip(depth, heads) -- a heads tuple shorter than depth drops the
    trailing stages, a longer one is cut.  The (depth, heads) pairs that run."""
    if isinstance(heads, tuple):
        if not all(isinstance(h, (int, np.integer)) and not isinstance(h, bool) for h in heads):
            raise TypeError(f"PiT: heads must be an int or a tuple of ints, got {heads!r}")
    elif isinstance(heads, (int, np.integer)) and not isinstance(heads, bool):
        heads = (heads,) * len(depth)
    else:
        raise TypeError(f"PiT: heads must be an int or a tuple of ints, got {heads!r}")
    return tuple((int(d), int(h)) for d, h in zip(depth, heads))


def pit_num_patches(side, patch_size):
    """Patches along one side: conv_output_size(side, p, p // 2) (pit.py:16-17), which for side >= p is extract_patches' VALID
    count floor((side - p) / (p // 2)) + 1."""
    return int(((side - patch_size) / (patch_size // 2)) + 1)


class PiT(_EngineModel):
    """pit.py:158-219 as the reference runs it.  `not_last = ind < (len(depth) < 1)` (:194) is `ind < 0`, never true, so no Pool is
    ever built and dim never doubles: the model is tf.image.extract_patches(patch_size, stride patch_size // 2, VALID) + Dense(dim),
    the cls row and positions, then one ViT Transformer(dim, depth[s], heads[s], dim_head, mlp_dim) per (depth, heads) pair of
    zip(depth, cast_tuple(heads)), then LayerNormalization + Dense on the cls row.  to_out is absent in a stage whose heads == 1
    and dim_head == dim (:59).
    Weights are ViT's names (SURVEY.md App. B) with layers.L counted across the stages in order.  There is no `transformer`
    attribute (the reference has none), so this runs as a whole forward only.
    A call-time image may be rectangular and give fewer patches than image_size (the first n + 1 rows of pos_embedding are used,
    :213); more patches than that raise ValueError (the reference fails to broadcast there), and so does an image smaller than one
    patch, where the reference's behaviour (extract_patches with no window) is not verifiable without TensorFlow.
    Limits the reference does not have: at most 8 stages after the zip and 1 to 32 heads per stage (NotImplementedError), and heads
    must be an int or a tuple of ints (TypeError; a bool, which cast_tuple would repeat as one head, is refused too)."""
    _kind = "pit"

    def __init__(self, image_size, patch_size, num_classes, dim, depth, heads, mlp_dim, dim_head=64, dropout=0.0, emb_dropout=0.0,
                 *, precision="bf16", device=0, seed=None):
        assert image_size % patch_size == 0, 'Image dimensions must be divisible by the patch size.'
        assert isinstance(depth, tuple), 'depth must be a tuple of integers, specifying the number of blocks before each downsizing'
        stages = pit_stages(depth, heads)
        side = pit_num_patches(image_size, patch_size)            # ZeroDivisionError for patch_size 1, as conv_output_size raises
        if len(stages) > _lib.PIT_MAX_STAGES:
            raise NotImplementedError(f"PiT: the engine runs at most {_lib.PIT_MAX_STAGES} stages; zip(depth, heads) gives {len(stages)}")
        if any(not 1 <= h <= 32 for _, h in stages):
            raise NotImplementedError(f"PiT: the engine runs 1 to 32 heads per stage; got {tuple(h for _, h in stages)}")
        self.num_classes, self.dim, self.dim_head, self.patch_size = num_classes, dim, dim_head, int(patch_size)
        self.stages, self.num_patches = stages, side * side
        self._dropout_rates = (dropout, emb_dropout)
        pc = _lib.VbPitConfig()
        pc.stages = len(stages)
        for s, (d, h) in enumerate(stages):
            pc.depth[s], pc.heads[s] = d, h
        self._pc = pc
        self._create(precision, device, ext=pc, create="vb_create_pit", image_h=image_size, image_w=image_size, patch_h=patch_size,
                     patch_w=patch_size, num_classes=num_classes, dim=dim, dim_head=dim_head, mlp_dim=mlp_dim)
        self.init_weights(seed)

    def __call__(self, img, training=True, **kwargs):
        """pit.py:207-219: NHWC float images [b, H, W, 3] -> logits [b, num_classes]; extra kwargs are accepted and ignored, as there."""
        self._check_training(training)
        x = np.ascontiguousarray(img, dtype=np.float32)
        if x.ndim != 4 or x.shape[3] != 3:
            raise ValueError(f"PiT: img must be NHWC float [b, H, W, 3], got shape {tuple(x.shape)}")
        b, h, w, _ = x.shape
        p = self.patch_size
        if h < p or w < p:
            raise ValueError(f"PiT: a {h} x {w} image is smaller than one {p} x {p} patch")
        n = pit_num_patches(h, p) * pit_num_patches(w, p)
        if n > self.num_patches:
            raise ValueError(f"PiT: the {h} x {w} image gives {n} patches but pos_embedding has rows for {self.num_patches}")
        out = np.empty((b, self.num_classes), np.float32)
        self.forward_raw(x.ctypes.data, _lib.MEM_HOST, b, h, w, out.ctypes.data, _lib.MEM_HOST, None)
        return _as_tensor(out)


PIT_CTOR_KEYS = ("image_size", "patch_size", "num_classes", "dim", "depth", "heads", "mlp_dim", "dim_head", "dropout", "emb_dropout")


class DistillWrapper(_WrapperModel):
    """distill.py:87-134: the teacher, the student over the wrapper's distillation token, distill_mlp (LayerNormalization + Dense)
    on the token's row and the soft-distillation loss, with the student, distill_mlp and the loss on the engine.  `wrapper([img,
    labels])` returns what the reference returns, a float32 loss vector [b], read as include/vitb200.h states: Keras'
    KLDivergence clips the log-probabilities to 1e-7, so the distillation term reads the teacher only.  An engine classifier on
    the student's device (_ENGINE_TEACHERS) runs as the teacher through its own handle, with no host copy of its logits; any
    other teacher is called on the host as `teacher(img, training=training)`.  hard=True constructs, and every call raises the
    reference's ValueError.  Precision and device are the student's; the student's weights are read at every call that follows
    a change."""
    _wrapped_name = "student"

    def __init__(self, teacher, student, temperature=1.0, alpha=0.5, hard=False, *, seed=None):
        assert (isinstance(student, (DistillableViT, DistillableT2TViT, DistillableEfficientViT))), 'student must be a vision transformer'
        if isinstance(student, DistillableT2TViT) and student._injected is not None:
            raise NotImplementedError("DistillWrapper: a DistillableT2TViT built around an injected transformer= runs its distillation "
                                      "call on the host around that transformer, so the wrapper has no device path for it")
        self.teacher, self.student = teacher, student
        self.dim, self.num_classes = student.dim, student.num_classes              # distill.py:96-97
        self.temperature, self.alpha, self.hard = temperature, alpha, hard
        self._dropout_rates = student._dropout_rates
        self.precision, self.device = student.precision, student.device
        self._cfg = _lib.VbConfig.from_buffer_copy(student._cfg)
        self._open(self._cfg, "vb_create_distill")
        self._share_weights()
        self.init_weights(seed)                        # distillation_token N(0, 1) and distill_mlp's Keras defaults

    @property
    def distillation_token(self):
        return self._weight_view("distillation_token")

    def _engine_teacher(self):
        """Whether the teacher runs through its own handle: one of _ENGINE_TEACHERS (exactly), open, on the student's device, and
        in a configuration whose call is vb_forward's logits."""
        t = self.teacher
        if type(t) not in _ENGINE_TEACHERS or getattr(t, "_h", None) is None or t.device != self.device:
            return False
        return not (isinstance(t, T2TViT) and t._injected is not None) and not (isinstance(t, LeViT) and t.num_distill_classes is not None)

    def forward_raw(self, img_ptr, img_mem, batch, h, w, labels_ptr, in_mem, temperature, alpha, loss_ptr, out_mem, stream=None,
                    teacher=None, teacher_logits_ptr=None, student_logits_ptr=None, distill_logits_ptr=None, teacher_logits_out_ptr=None):
        """Pointer-level call (vb_forward_distill_loss): host or device buffers, optional cudaStream_t.  Pass exactly one of
        `teacher` (an engine model) and `teacher_logits_ptr` ([batch, num_classes] in in_mem memory, as the labels); loss [batch]
        and the optional [batch, num_classes] outputs go to out_mem memory."""
        self._finalize()
        th = None
        if teacher is not None:
            teacher._finalize()
            th = teacher._h
        p = [C.c_void_p(v) if v else None for v in (teacher_logits_ptr, loss_ptr, student_logits_ptr, distill_logits_ptr,
                                                    teacher_logits_out_ptr)]
        _lib.check(self._lib.vb_forward_distill_loss(self._h, C.c_void_p(img_ptr), img_mem, batch, h, w, C.c_void_p(labels_ptr), th, p[0],
                                                     in_mem, float(temperature), float(alpha), *p[1:], out_mem,
                                                     C.c_void_p(stream) if stream else None), self._h)

    def _call(self, inputs, temperature, alpha, training, outputs):
        img, labels = inputs                                                      # distill.py:109
        alpha = alpha if alpha is not None else self.alpha
        T = temperature if temperature is not None else self.temperature
        if isinstance(self.student, DistillableEfficientViT):
            self.student(img, distill_token=self.distillation_token, training=training)   # raises, as distill.py:83 does
        on_engine = self._engine_teacher()
        if on_engine:
            self.teacher._check_training(training)
        self._check_training(training)
        if T == 0:
            raise ValueError("DistillWrapper: temperature 0 divides the logits by zero (inf / NaN in the reference)")
        x = self._img(img)
        b, h, w, _ = x.shape
        K = self.num_classes
        y = np.ascontiguousarray(labels, dtype=np.float32)
        if y.shape != (b, K):                                                     # categorical_crossentropy's shape check (:119)
            raise ValueError(f"Shapes {y.shape} and {(b, K)} are incompatible")
        if self.hard:                                                             # :131-132: argmax labels [b] against [b, K]
            raise ValueError(f"Shapes {(b,)} and {(b, K)} are incompatible")
        tl = None
        if not on_engine:
            t = self.teacher(img, training=training)                               # :114, with the caller's img object
            tl = np.ascontiguousarray(t.numpy() if hasattr(t, "numpy") else t, dtype=np.float32)
            if tl.shape != (b, K):
                raise ValueError(f"DistillWrapper: the teacher returned logits of shape {tl.shape}; expected [b, num_classes] = {(b, K)}")
        loss = np.empty(b, np.float32)
        rows = [np.empty((b, K), np.float32) for _ in range(3)] if outputs else [None] * 3
        ptr = lambda a: a.ctypes.data if a is not None else None
        self.forward_raw(x.ctypes.data, _lib.MEM_HOST, b, h, w, y.ctypes.data, _lib.MEM_HOST, T, alpha, loss.ctypes.data, _lib.MEM_HOST,
                         teacher=self.teacher if on_engine else None, teacher_logits_ptr=ptr(tl), student_logits_ptr=ptr(rows[0]),
                         distill_logits_ptr=ptr(rows[1]), teacher_logits_out_ptr=ptr(rows[2]))
        return (_as_tensor(loss),) + tuple(_as_tensor(r) for r in rows if r is not None)

    def __call__(self, inputs, temperature=None, alpha=None, training=True, **kwargs):
        """distill.py:108-134: inputs = [img, labels [b, num_classes]] -> the loss, float32 [b] (answers `.numpy()`)."""
        return self._call(inputs, temperature, alpha, training, False)[0]

    def forward_distill_loss(self, inputs, temperature=None, alpha=None):
        """One call with training=False: (loss [b], student_logits, distill_logits, teacher_logits), each [b, num_classes]."""
        return self._call(inputs, temperature, alpha, False, True)


# the engine classes whose `__call__(img, training=)` is exactly their vb_forward logits (T2TViT without an injected transformer,
# LeViT without a distillation head): DistillWrapper runs such a teacher through its handle
_ENGINE_TEACHERS = (ViT, DeepViT, CaiT, CrossViT, ParallelViT, PatchMergerViT, T2TViT, DistillableViT, DistillableT2TViT, CCT, LeViT, CvT,
                    SmallDatasetViT)


_FAMILY_CTORS = {"pit": (PiT, PIT_CTOR_KEYS), "scalable_vit": (ScalableViT, SCALABLE_VIT_CTOR_KEYS),
                 "mobilevit": (MobileViT, MOBILEVIT_CTOR_KEYS), "small_dataset_vit": (SmallDatasetViT, SMALL_DATASET_VIT_CTOR_KEYS),
                 "ats_vit": (ATSViT, ATS_CTOR_KEYS), "regionvit": (RegionViT, REGIONVIT_CTOR_KEYS), "nest": (NesT, NEST_CTOR_KEYS),
                 "crossformer": (CrossFormer, CROSSFORMER_CTOR_KEYS), "twins_svt": (TwinsSVT, TWINS_CTOR_KEYS),
                 "cvt": (CvT, CVT_CTOR_KEYS), "levit": (LeViT, LEVIT_CTOR_KEYS), "cct": (CCT, CCT_CTOR_KEYS)}


def from_config(cfg: dict, precision="bf16", device=0, seed=None):
    """Build a model from an oracle-style config dict (kind + reference kwargs)."""
    if cfg["kind"] in _FAMILY_CTORS:
        cls, keys = _FAMILY_CTORS[cfg["kind"]]
        return cls(**{k: v for k, v in cfg.items() if k in keys}, precision=precision, device=device, seed=seed)
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

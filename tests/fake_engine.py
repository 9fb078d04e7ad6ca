"""CPU double of libvitb200's C-ABI, for tests of the HOST logic only.

Constructing a `vit_tensorflow_b200.ViT` needs an H100 (`vb_create` refuses without one, and there is no CPU fallback in the
product).  What sits between the user and the C-ABI -- kwargs, ctypes marshalling, the attribute surface the reference's wrappers
poke at (`patch_embedding.layers[:2]`, `.weights`, `pos_embedding[:, 1:n]`, `transformer(tokens)`, `.numpy()` on results) -- is
plain Python, though, and can be exercised on a CPU box by handing the host classes an object that answers the same `vb_*`
calls on the same pointers, computing with the oracle.  `installed()` swaps it in for `_lib.load()`; nothing outside tests/ ever
imports this module.
"""
import contextlib
import ctypes as C

import numpy as np
from einops import rearrange

import oracle
from oracle import spec_numpy

_KINDS = {0: "vit", 1: "deepvit", 2: "cait", 3: "crossvit", 4: "parallel_vit", 5: "patch_merger_vit", 6: "t2t_vit"}


def _f32(ptr, shape):
    """float32 array over caller memory at `ptr` (a ctypes c_void_p)."""
    n = int(np.prod(shape))
    return np.ctypeslib.as_array(C.cast(ptr, C.POINTER(C.c_float)), shape=(n,)).reshape(shape)


class FakeLib:
    def __init__(self):
        self.handles = {}
        self.next_key = 0
        self.calls = []                # (entry, detail) log: the tests assert on what the host classes asked the engine for
        self.err = b""

    # ---- lifecycle -------------------------------------------------------------------------------------
    def vb_abi_version(self):
        return 4

    @staticmethod
    def _decode(c):
        """VbConfig (include/vitb200.h) -> oracle config: the inverse of what the host classes' `_create` calls encode."""
        kind = _KINDS[c.kind]
        pool = "mean" if c.pool else "cls"
        common = dict(num_classes=c.num_classes, dim=c.dim, depth=c.depth, heads=c.heads, mlp_dim=c.mlp_dim, dim_head=c.dim_head)
        if kind in ("vit", "parallel_vit"):
            extra = dict(num_parallel_branches=c.parallel_branches) if kind == "parallel_vit" else {}
            return oracle.make_config(kind, image_size=(c.image_h, c.image_w), patch_size=(c.patch_h, c.patch_w), pool=pool, **common, **extra)
        if kind == "deepvit":
            return oracle.make_config(kind, image_size=c.image_h, patch_size=c.patch_h, pool=pool, **common)
        if kind == "cait":
            return oracle.make_config(kind, image_size=c.image_h, patch_size=c.patch_h, cls_depth=c.cls_depth, **common)
        if kind == "patch_merger_vit":
            return oracle.make_config(kind, image_size=(c.image_h, c.image_w), patch_size=(c.patch_h, c.patch_w),
                                      patch_merge_layer=c.patch_merge_layer_index + 1, patch_merge_num_tokens=c.patch_merge_num_tokens, **common)
        if kind == "t2t_vit":
            layers = tuple((getattr(c, f"t2t_k{i}"), getattr(c, f"t2t_s{i}")) for i in range(c.t2t_num_layers))
            return oracle.make_config(kind, image_size=c.image_h, pool=pool, t2t_layers=layers, **common)
        if kind == "crossvit":
            names = ("sm_dim", "lg_dim", "sm_patch_size", "sm_enc_depth", "sm_enc_heads", "sm_enc_mlp_dim", "sm_enc_dim_head", "lg_patch_size",
                     "lg_enc_depth", "lg_enc_heads", "lg_enc_mlp_dim", "lg_enc_dim_head", "cross_attn_depth", "cross_attn_heads", "cross_attn_dim_head")
            return oracle.make_config(kind, image_size=c.image_h, num_classes=c.num_classes, depth=c.cross_depth, **{n: getattr(c, n) for n in names})
        raise ValueError(kind)

    def vb_create(self, cfg_ref, device, handle_ref):
        c = cfg_ref._obj
        if c.kind not in _KINDS or c.struct_size != C.sizeof(type(c)):
            self.err = b"fake engine: bad config"
            return 1
        cfg = self._decode(c)
        specs = list(oracle.weight_specs(cfg).items())
        if c.depth == 0 and cfg["kind"] == "vit":          # efficient.ViT shell: embed + head only (engine.cu does the same for depth 0)
            specs = [(n, s) for n, s in specs if not n.startswith("layers.")]
        self.next_key += 1
        key = self.next_key
        self.handles[key] = dict(cfg=cfg, specs=specs, w={}, finalized=False, keep=[])
        handle_ref._obj.value = key
        self.calls.append(("vb_create", cfg["kind"]))
        return 0

    def _h(self, h):
        return self.handles[h.value if hasattr(h, "value") else h]

    def vb_destroy(self, h):
        self.handles.pop(getattr(h, "value", h), None)

    def vb_last_error(self, h):
        return self.err

    def vb_last_launch_count(self, h):
        return 0

    # ---- weights ---------------------------------------------------------------------------------------
    def vb_num_weights(self, h):
        return len(self._h(h)["specs"])

    def vb_weight_info(self, h, i, name_ref, shape, ndim_ref):
        st = self._h(h)
        name, (shp, _) = st["specs"][i]
        b = name.encode()
        st["keep"].append(b)
        name_ref._obj.value = b
        for j, d in enumerate(shp):
            shape[j] = d
        ndim_ref._obj.value = len(shp)
        return 0

    def vb_set_weight(self, h, name, ptr, shape, ndim):
        st = self._h(h)
        shp = tuple(int(shape[j]) for j in range(ndim))
        st["w"][name.decode()] = _f32(ptr, shp).copy()
        st["finalized"] = False
        return 0

    def vb_finalize(self, h):
        st = self._h(h)
        missing = [n for n, _ in st["specs"] if n not in st["w"]]
        if missing:
            self.err = f"fake engine: weights not set: {missing[:3]}".encode()
            return 2
        st["finalized"] = True
        self.calls.append(("vb_finalize", None))
        return 0

    # ---- forward entries (host buffers only) -------------------------------------------------------------
    def _ready(self, h):
        st = self._h(h)
        assert st["finalized"], "host class called a forward entry before vb_finalize"
        return st

    def vb_forward(self, h, img, mem_in, b, hh, ww, out, mem_out, stream):
        st = self._ready(h)
        x = _f32(img, (b, hh, ww, 3))
        _f32(out, (b, st["cfg"]["num_classes"]))[:] = oracle.forward_numpy(x, st["w"], st["cfg"])
        self.calls.append(("vb_forward", (b, hh, ww)))
        return 0

    def vb_forward_distill(self, h, img, mem_in, b, hh, ww, tok, logits, dist, mem_out, stream):
        st = self._ready(h)
        d = st["cfg"]["dim"]
        lo, di = spec_numpy.forward_distill(_f32(img, (b, hh, ww, 3)), _f32(tok, (d,)).reshape(1, 1, d), st["w"], st["cfg"])
        _f32(logits, lo.shape)[:] = lo
        _f32(dist, di.shape)[:] = di
        self.calls.append(("vb_forward_distill", (b, hh, ww)))
        return 0

    def vb_forward_tokens(self, h, x, mem_in, b, n, out, mem_out, stream):
        st = self._ready(h)
        d = st["cfg"]["dim"]
        _f32(out, (b, n, d))[:] = spec_numpy.transformer_tokens(_f32(x, (b, n, d)), st["w"], st["cfg"])
        self.calls.append(("vb_forward_tokens", (b, n)))
        return 0

    def vb_embed_rows(self, h, hh, ww):
        cfg = self._h(h)["cfg"]
        if cfg["kind"] == "t2t_vit":
            gh, gw = oracle.t2t_token_grid(cfg, hh, ww)[-1]
            return gh * gw + 1
        n = (hh // cfg["patch_h"]) * (ww // cfg["patch_w"])
        return n + (0 if cfg["kind"] in ("cait", "patch_merger_vit") else 1)

    def vb_forward_embed(self, h, img, mem_in, b, hh, ww, out, mem_out, stream):
        st = self._ready(h)
        t = spec_numpy.embed_tokens(_f32(img, (b, hh, ww, 3)), st["w"], st["cfg"])
        _f32(out, t.shape)[:] = t
        self.calls.append(("vb_forward_embed", (b, hh, ww)))
        return 0

    def vb_forward_head(self, h, x, mem_in, b, n, out, mem_out, stream):
        st = self._ready(h)
        d = st["cfg"]["dim"]
        _f32(out, (b, st["cfg"]["num_classes"]))[:] = spec_numpy.head_logits(_f32(x, (b, n, d)), st["w"], st["cfg"])
        self.calls.append(("vb_forward_head", (b, n)))
        return 0

    def vb_to_patch(self, h, img, mem_in, b, hh, ww, out, mem_out, stream):
        cfg = self._h(h)["cfg"]
        p = rearrange(_f32(img, (b, hh, ww, 3)), 'b (h p1) (w p2) c -> b (h w) (p1 p2 c)', p1=cfg["patch_h"], p2=cfg["patch_w"])
        _f32(out, p.shape)[:] = p
        self.calls.append(("vb_to_patch", (b, hh, ww)))
        return 0

    def vb_patch_to_emb(self, h, x, mem_in, rows, out, mem_out, stream):
        st = self._ready(h)
        k, bias = st["w"]["patch.kernel"].astype(np.float64), st["w"]["patch.bias"].astype(np.float64)
        _f32(out, (rows, k.shape[1]))[:] = _f32(x, (rows, k.shape[0])).astype(np.float64) @ k + bias
        self.calls.append(("vb_patch_to_emb", rows))
        return 0


@contextlib.contextmanager
def installed():
    """`vit_tensorflow_b200._lib.load()` returns a FakeLib inside the block (and the real loader again afterwards)."""
    from vit_tensorflow_b200 import _lib
    fake = FakeLib()
    saved_load, saved_cached = _lib.load, _lib._lib
    _lib.load = lambda: fake
    try:
        yield fake
    finally:
        _lib.load, _lib._lib = saved_load, saved_cached

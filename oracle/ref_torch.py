"""torch-CPU float32 restatement of the reference forward pass.

TEST INFRASTRUCTURE (see oracle/__init__.py); doubles as the timed CPU baseline
("restated reference (torch CPU); TF unavailable").
PARITY UNPINNED at the TensorFlow boundary.

Written independently of oracle/spec_numpy.py (explicit reshape/permute instead of einops,
torch.nn.functional primitives instead of hand-rolled ones) so that the two restatements
cross-check each other.  Reference lines are cited per function.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

LN_EPS = 1e-3  # Keras LayerNormalization default


class _W:
    """Weight dict -> torch float32 tensors, fetched by name."""

    def __init__(self, weights, dtype=torch.float32):
        self.t = {k: torch.as_tensor(v).to(dtype) for k, v in weights.items()}

    def __getitem__(self, k):
        return self.t[k]

    def __contains__(self, k):
        return k in self.t


def _linear(x, w, name, bias=True):
    # Keras Dense: kernel [in, out]
    y = torch.matmul(x, w[name + ".kernel"])
    return y + w[name + ".bias"] if bias else y


def _ln(x, w, name):
    return F.layer_norm(x, (x.shape[-1],), w[name + ".gamma"], w[name + ".beta"], LN_EPS)


def _mlp(x, w, pre):
    return _linear(F.gelu(_linear(x, w, pre + "fc1")), w, pre + "fc2")  # exact erf GELU (vit.py:34)


def _im2col(img, ph, pw):
    # 'b (h p1) (w p2) c -> b (h w) (p1 p2 c)'  (vit.py:142), via reshape/permute
    b, H, W, c = img.shape
    gh, gw = H // ph, W // pw
    x = img.reshape(b, gh, ph, gw, pw, c).permute(0, 1, 3, 2, 4, 5)
    return x.reshape(b, gh * gw, ph * pw * c)


def _heads(t, h):
    b, n, hd = t.shape
    return t.reshape(b, n, h, hd // h).permute(0, 2, 1, 3)


def _merge(t):
    b, h, n, d = t.shape
    return t.permute(0, 2, 1, 3).reshape(b, n, h * d)


def _attn_vit(x, w, pre, heads, dim_head, deepvit):
    # vit.py:71-85, deepvit.py:73-91
    qkv = _linear(x, w, pre + "to_qkv", bias=False)
    inner = heads * dim_head
    q, k, v = (_heads(qkv[..., i * inner:(i + 1) * inner], heads) for i in range(3))
    attn = torch.softmax(torch.matmul(q, k.transpose(-1, -2)) * dim_head ** -0.5, dim=-1)
    if deepvit:
        # attn[b,g,i,j] = sum_h attn[b,h,i,j] W[h,g]; then LN over the head axis (deepvit.py:83-84)
        a = torch.matmul(attn.permute(0, 2, 3, 1), w[pre + "reattn_weights"])     # [b,i,j,g]
        a = _ln(a, w, pre + "reattn_norm")
        attn = a.permute(0, 3, 1, 2)
    out = _merge(torch.matmul(attn, v))
    if (pre + "to_out.kernel") in w:
        out = _linear(out, w, pre + "to_out")
    return out


def _attn_qkv(x, w, pre, heads, dim_head, context=None, talking=False):
    # cait.py:107-131, cross_vit.py:69-93
    ctx = x if context is None else torch.cat([x, context], dim=1)
    inner = heads * dim_head
    q = _heads(_linear(x, w, pre + "to_q", bias=False), heads)
    kv = _linear(ctx, w, pre + "to_kv", bias=False)
    k, v = _heads(kv[..., :inner], heads), _heads(kv[..., inner:], heads)
    dots = torch.matmul(q, k.transpose(-1, -2)) * dim_head ** -0.5
    if talking:
        dots = torch.matmul(dots.permute(0, 2, 3, 1), w[pre + "mix_pre"]).permute(0, 3, 1, 2)
    attn = torch.softmax(dots, dim=-1)
    if talking:
        attn = torch.matmul(attn.permute(0, 2, 3, 1), w[pre + "mix_post"]).permute(0, 3, 1, 2)
    return _linear(_merge(torch.matmul(attn, v)), w, pre + "to_out")


def _transformer_vit(x, w, cfg):
    deep = cfg["kind"] == "deepvit"
    for L in range(cfg["depth"]):
        pre = f"layers.{L}."
        x = _attn_vit(_ln(x, w, pre + "attn_norm"), w, pre, cfg["heads"], cfg["dim_head"], deep) + x
        x = _mlp(_ln(x, w, pre + "ff_norm"), w, pre) + x
    return x


def _transformer_parallel(x, w, cfg):
    # parallel_vit.py:114-117, Parallel :41-42
    for L in range(cfg["depth"]):
        pres = [f"layers.{L}.branch{i}." for i in range(cfg["num_parallel_branches"])]
        a = None
        for p in pres:
            y = _attn_vit(_ln(x, w, p + "attn_norm"), w, p, cfg["heads"], cfg["dim_head"], False)
            a = y if a is None else a + y
        x = a + x
        f = None
        for p in pres:
            y = _mlp(_ln(x, w, p + "ff_norm"), w, p)
            f = y if f is None else f + y
        x = f + x
    return x


def _forward_vit(img, w, cfg):
    # vit.py:159-177 / parallel_vit.py:167-185
    x = _linear(_im2col(img, cfg["patch_h"], cfg["patch_w"]), w, "patch")
    b, n, d = x.shape
    x = torch.cat([w["cls_token"].expand(b, 1, d), x], dim=1) + w["pos_embedding"][:, :n + 1]
    x = _transformer_parallel(x, w, cfg) if cfg["kind"] == "parallel_vit" else _transformer_vit(x, w, cfg)
    x = x.mean(dim=1) if cfg["pool"] == "mean" else x[:, 0]
    return _linear(_ln(x, w, "head_norm"), w, "head")


def _transformer_cait(x, w, cfg, stack, depth, context=None):
    for L in range(depth):
        pre = f"{stack}.layers.{L}."
        a = _attn_qkv(_ln(x, w, pre + "attn_norm"), w, pre, cfg["heads"], cfg["dim_head"], context, True)
        x = a * w[pre + "attn_scale"] + x
        x = _mlp(_ln(x, w, pre + "ff_norm"), w, pre) * w[pre + "ff_scale"] + x
    return x


def _forward_cait(img, w, cfg):
    # cait.py:180-194
    x = _linear(_im2col(img, cfg["patch_h"], cfg["patch_w"]), w, "patch")
    b, n, d = x.shape
    x = x + w["pos_embedding"][:, :n]
    x = _transformer_cait(x, w, cfg, "patch_transformer", cfg["depth"])
    cls = w["cls_token"].expand(b, 1, d)
    x = _transformer_cait(cls, w, cfg, "cls_transformer", cfg["cls_depth"], context=x)
    return _linear(_ln(x[:, 0], w, "head_norm"), w, "head")


def _forward_crossvit(img, w, cfg):
    # cross_vit.py:290-303
    tok = {}
    for br in ("sm", "lg"):
        p = cfg[f"{br}_patch_size"]
        x = _linear(_im2col(img, p, p), w, f"{br}_embed.patch")
        b, n, d = x.shape
        tok[br] = torch.cat([w[f"{br}_embed.cls_token"].expand(b, 1, d), x], dim=1) + w[f"{br}_embed.pos_embedding"][:, :n + 1]

    def enc(x, pre, br):
        for L in range(cfg[f"{br}_enc_depth"]):
            p = f"{pre}layers.{L}."
            x = _attn_qkv(_ln(x, w, p + "attn_norm"), w, p, cfg[f"{br}_enc_heads"], cfg[f"{br}_enc_dim_head"]) + x
            x = _mlp(_ln(x, w, p + "ff_norm"), w, p) + x
        return _ln(x, w, pre + "final_norm")

    def cross(cls, ctx, pre):
        x = cls
        proj = (pre + "project_in.kernel") in w
        if proj:
            x = _linear(x, w, pre + "project_in")
        x = _attn_qkv(_ln(x, w, pre + "norm"), w, pre, cfg["cross_attn_heads"], cfg["cross_attn_dim_head"], context=ctx)
        if proj:
            x = _linear(x, w, pre + "project_out")
        return x + cls

    sm, lg = tok["sm"], tok["lg"]
    for D in range(cfg["depth"]):
        sm, lg = enc(sm, f"blocks.{D}.sm_enc.", "sm"), enc(lg, f"blocks.{D}.lg_enc.", "lg")
        sm_cls, sm_p, lg_cls, lg_p = sm[:, :1], sm[:, 1:], lg[:, :1], lg[:, 1:]
        for R in range(cfg["cross_attn_depth"]):
            sm_cls = cross(sm_cls, lg_p, f"blocks.{D}.cross.{R}.sm_attend_lg.")
            lg_cls = cross(lg_cls, sm_p, f"blocks.{D}.cross.{R}.lg_attend_sm.")
        sm, lg = torch.cat([sm_cls, sm_p], dim=1), torch.cat([lg_cls, lg_p], dim=1)
    return (_linear(_ln(sm[:, 0], w, "sm_head_norm"), w, "sm_head")
            + _linear(_ln(lg[:, 0], w, "lg_head_norm"), w, "lg_head"))


def _patch_merger(x, w, pre="patch_merger."):
    # vit_with_patch_merger.py:49-55
    x = _ln(x, w, pre + "norm")
    sim = torch.matmul(w[pre + "queries"], x.transpose(1, 2) * x.shape[-1] ** -0.5)
    return torch.matmul(torch.softmax(sim, dim=-1), x)


def _forward_patch_merger_vit(img, w, cfg):
    # vit_with_patch_merger.py:174-185, Transformer.call :118-126
    x = _linear(_im2col(img, cfg["patch_h"], cfg["patch_w"]), w, "patch")
    x = x + w["pos_embedding"][:, :x.shape[1]]
    for L in range(cfg["depth"]):
        pre = f"layers.{L}."
        x = _attn_vit(_ln(x, w, pre + "attn_norm"), w, pre, cfg["heads"], cfg["dim_head"], False) + x
        x = _mlp(_ln(x, w, pre + "ff_norm"), w, pre) + x
        if L == cfg["patch_merge_layer_index"]:
            x = _patch_merger(x, w)
    return _linear(_ln(x.mean(dim=1), w, "head_norm"), w, "head")


def _unfold_same(x, k, stride):
    # tf.image.extract_patches(..., padding='SAME') (t2t.py:43) through F.pad + F.unfold; unfold orders the patch vector
    # (channel, k_row, k_col), TensorFlow (k_row, k_col, channel) -> permute.  x [b, H, W, C] -> [b, oh*ow, k*k*C]
    b, H, W, C = x.shape
    oh, ow = (H + stride - 1) // stride, (W + stride - 1) // stride
    ph, pw = max((oh - 1) * stride + k - H, 0), max((ow - 1) * stride + k - W, 0)
    xp = F.pad(x.permute(0, 3, 1, 2), (pw // 2, pw - pw // 2, ph // 2, ph - ph // 2))
    cols = F.unfold(xp, kernel_size=k, stride=stride)                       # [b, C*k*k, L]
    L = cols.shape[-1]
    assert L == oh * ow
    return cols.reshape(b, C, k, k, L).permute(0, 4, 2, 3, 1).reshape(b, L, k * k * C)


def _t2t_tokens(img, w, cfg):
    # t2t.py:58-74 with RearrangeUnfoldTransformer.call :39-48
    x = img
    last = len(cfg["t2t_layers"]) - 1
    for i, (k, st) in enumerate(cfg["t2t_layers"]):
        if i > 0:
            b, n, c = x.shape
            hh = int(n ** 0.5)
            x = x.reshape(b, hh, n // hh, c)
        x = _unfold_same(x, k, st)
        if i != last:
            d = x.shape[-1]
            pre = f"t2t.{i}.layers.0."
            x = _attn_vit(_ln(x, w, pre + "attn_norm"), w, pre, 1, d, False) + x
            x = _mlp(_ln(x, w, pre + "ff_norm"), w, pre) + x
    return _linear(x, w, "patch")


def _forward_t2t_vit(img, w, cfg):
    # t2t.py:96-116
    x = _t2t_tokens(img, w, cfg)
    b, n, d = x.shape
    x = torch.cat([w["cls_token"].expand(b, 1, d), x], dim=1) + w["pos_embedding"][:, :n + 1]
    x = _transformer_vit(x, w, cfg)
    x = x.mean(dim=1) if cfg["pool"] == "mean" else x[:, 0]
    return _linear(_ln(x, w, "head_norm"), w, "head")


class TorchReference:
    """Holds the weights as torch tensors once; `__call__(img)` -> logits (numpy float32)."""

    def __init__(self, weights, cfg, dtype=torch.float32):
        self.cfg = cfg
        self.w = _W(weights, dtype)
        self.dtype = dtype

    @torch.no_grad()
    def __call__(self, img):
        x = torch.as_tensor(img).to(self.dtype)
        kind = self.cfg["kind"]
        if kind in ("vit", "deepvit", "parallel_vit"):
            y = _forward_vit(x, self.w, self.cfg)
        elif kind == "cait":
            y = _forward_cait(x, self.w, self.cfg)
        elif kind == "crossvit":
            y = _forward_crossvit(x, self.w, self.cfg)
        elif kind == "patch_merger_vit":
            y = _forward_patch_merger_vit(x, self.w, self.cfg)
        elif kind == "t2t_vit":
            y = _forward_t2t_vit(x, self.w, self.cfg)
        else:
            raise ValueError(kind)
        return y.float().numpy()

    @torch.no_grad()
    def transformer(self, tokens):
        return _transformer_vit(torch.as_tensor(tokens).to(self.dtype), self.w, self.cfg).float().numpy()


def forward(img, weights, cfg):
    return TorchReference(weights, cfg)(img)

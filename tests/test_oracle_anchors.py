"""Second, independent anchors for the oracle's building blocks (VERDICT r1 item 9): the numpy-float64 spec against PyTorch's own
implementations of the same published operators, on random inputs.  None of this is TensorFlow (absent from this image: the reference's own
code is pinned by tests/test_reference_shim.py, the TensorFlow primitives under it stay assumed, SURVEY.md Appendix A), but it is
third-party code the spec did not come from:

  attention core (vit.py:77-82)            F.scaled_dot_product_attention
  fused-QKV multi-head attention            torch.nn.MultiheadAttention with mapped weights (vit.py:59,63,72-84)
  extract_patches SAME (t2t.py:43)          F.pad with TF's documented SAME split + F.unfold (window extraction, stride handling)
  LayerNormalization eps 1e-3 (vit.py:18)   F.layer_norm
  exact-erf GELU (vit.py:29-34)             F.gelu(approximate='none')
  Rearrange patches (vit.py:142)            F.unfold with kernel = stride = patch (window order) -- besides einops itself
  talking heads / re-attention (cait.py:114-127, deepvit.py:79-87)   plain-loop restatements without einsum / einops: which axis of the
                                            [h, g] mix matrices is contracted, LayerNorm over the head axis, head-major column order
"""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import spec_numpy as S


def test_attention_core_vs_torch_sdpa():
    rng = np.random.default_rng(0)
    b, h, n, d = 2, 3, 37, 16
    x = rng.standard_normal((b, n, h * d))
    w = {"l.to_qkv.kernel": rng.standard_normal((h * d, 3 * h * d)) / np.sqrt(h * d)}
    got = S.attention_vit(x, w, "l.", h, d)                          # no to_out in w: the attention core, heads merged
    qkv = torch.from_numpy(x @ w["l.to_qkv.kernel"])
    q, k, v = (t.reshape(b, n, h, d).transpose(1, 2) for t in qkv.chunk(3, dim=-1))
    ref = F.scaled_dot_product_attention(q, k, v).transpose(1, 2).reshape(b, n, h * d).numpy()
    np.testing.assert_allclose(got, ref, rtol=1e-10, atol=1e-12)


def test_fused_qkv_attention_vs_torch_multihead_attention():
    rng = np.random.default_rng(1)
    b, h, n, d = 2, 4, 19, 8
    e = h * d
    x = rng.standard_normal((b, n, e))
    w = {"l.to_qkv.kernel": rng.standard_normal((e, 3 * e)) / np.sqrt(e), "l.to_out.kernel": rng.standard_normal((e, e)) / np.sqrt(e),
         "l.to_out.bias": rng.standard_normal(e)}
    got = S.attention_vit(x, w, "l.", h, d)
    mha = torch.nn.MultiheadAttention(e, h, bias=True, batch_first=True, dtype=torch.float64)
    with torch.no_grad():
        mha.in_proj_weight.copy_(torch.from_numpy(w["l.to_qkv.kernel"].T))      # rows [q | k | v] = tf.split(qkv, 3, -1) (vit.py:73)
        mha.in_proj_bias.zero_()
        mha.out_proj.weight.copy_(torch.from_numpy(w["l.to_out.kernel"].T))
        mha.out_proj.bias.copy_(torch.from_numpy(w["l.to_out.bias"]))
        xt = torch.from_numpy(x)
        ref, _ = mha(xt, xt, xt, need_weights=False)
    np.testing.assert_allclose(got, ref.numpy(), rtol=1e-9, atol=1e-11)


@pytest.mark.parametrize("H,W,k,s", [(224, 224, 7, 4), (56, 56, 3, 2), (28, 28, 3, 2), (9, 11, 3, 2), (10, 7, 5, 3), (8, 8, 2, 2)])
def test_extract_patches_same_vs_torch_unfold(H, W, k, s):
    rng = np.random.default_rng(H + k)
    b, C = 2, 3
    x = rng.standard_normal((b, H, W, C))
    got = S.extract_patches_same(x, k, s)                                        # [b, oh, ow, (k_row, k_col, c)]
    oh, ow = -(-H // s), -(-W // s)
    ph, pw = max((oh - 1) * s + k - H, 0), max((ow - 1) * s + k - W, 0)          # TF SAME: smaller half first
    xt = F.pad(torch.from_numpy(x).permute(0, 3, 1, 2), (pw // 2, pw - pw // 2, ph // 2, ph - ph // 2))
    u = F.unfold(xt, kernel_size=k, stride=s)                                    # [b, C*k*k, L], rows ordered (c, k_row, k_col)
    assert u.shape[-1] == oh * ow
    ref = u.reshape(b, C, k, k, oh, ow).permute(0, 4, 5, 2, 3, 1).reshape(b, oh, ow, k * k * C).numpy()
    np.testing.assert_array_equal(got, ref)


def test_patch_rearrange_vs_torch_unfold():
    rng = np.random.default_rng(2)
    b, H, W, C, p1, p2 = 2, 24, 32, 3, 8, 16
    img = rng.standard_normal((b, H, W, C))
    w = {"patch.kernel": np.eye(p1 * p2 * C), "patch.bias": np.zeros(p1 * p2 * C)}
    got = S.patch_embed(img, w, "patch", p1, p2)                                 # identity Dense: the Rearrange alone
    u = F.unfold(torch.from_numpy(img).permute(0, 3, 1, 2), kernel_size=(p1, p2), stride=(p1, p2))      # rows (c, p1, p2)
    ref = u.reshape(b, C, p1, p2, -1).permute(0, 4, 2, 3, 1).reshape(b, -1, p1 * p2 * C).numpy()        # -> (p1 p2 c)
    np.testing.assert_array_equal(got, ref)


def test_layernorm_and_gelu_vs_torch():
    rng = np.random.default_rng(3)
    x = rng.standard_normal((5, 7, 48)) * 3 + 1
    w = {"n.gamma": rng.uniform(0.5, 1.5, 48), "n.beta": rng.standard_normal(48)}
    ref = F.layer_norm(torch.from_numpy(x), (48,), torch.from_numpy(w["n.gamma"]), torch.from_numpy(w["n.beta"]), eps=1e-3).numpy()
    np.testing.assert_allclose(S.layer_norm(x, w, "n"), ref, rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(S.gelu(x), F.gelu(torch.from_numpy(x), approximate="none").numpy(), rtol=1e-12, atol=1e-14)


def _explicit_head_mix(t, W):
    """out[b, g, i, j] = sum_h t[b, h, i, j] * W[h, g] written as plain loops: the meaning TensorFlow documents for
    einsum('b h i j, h g -> b g i j') (deepvit.py:83, cait.py:123,125; SURVEY.md App. A item 6)."""
    b, h, n, m = t.shape
    out = np.zeros((b, W.shape[1], n, m))
    for bb in range(b):
        for g in range(W.shape[1]):
            for hh in range(h):
                out[bb, g] += t[bb, hh] * W[hh, g]
    return out


def test_cait_talking_heads_vs_explicit_loops():
    """cait.py:114-127 restated without einsum / einops: projections, per-head scores, pre-softmax mix over the IN-head axis,
    softmax over keys, post-softmax mix, P V, heads merged head-major."""
    rng = np.random.default_rng(5)
    b, h, n, d, dim = 2, 3, 7, 4, 10
    x = rng.standard_normal((b, n, dim))
    w = {"l.to_q.kernel": rng.standard_normal((dim, h * d)), "l.to_kv.kernel": rng.standard_normal((dim, 2 * h * d)),
         "l.mix_pre": rng.standard_normal((h, h)), "l.mix_post": rng.standard_normal((h, h)),
         "l.to_out.kernel": rng.standard_normal((h * d, dim)), "l.to_out.bias": rng.standard_normal(dim)}
    got = S.attention_qkv(x, w, "l.", h, d, talking_heads=True)
    q = x @ w["l.to_q.kernel"]
    kv = x @ w["l.to_kv.kernel"]
    k, v = kv[..., :h * d], kv[..., h * d:]                                    # tf.split(kv, 2): [k | v]
    dots = np.zeros((b, h, n, n))
    for hh in range(h):                                                        # 'b n (h d) -> b h n d': column = h * d + d'
        qs, ks = q[..., hh * d:(hh + 1) * d], k[..., hh * d:(hh + 1) * d]
        for bb in range(b):
            dots[bb, hh] = qs[bb] @ ks[bb].T * d ** -0.5
    dots = _explicit_head_mix(dots, w["l.mix_pre"])
    e = np.exp(dots - dots.max(-1, keepdims=True))
    attn = _explicit_head_mix(e / e.sum(-1, keepdims=True), w["l.mix_post"])
    out = np.zeros((b, n, h * d))
    for hh in range(h):
        for bb in range(b):
            out[bb, :, hh * d:(hh + 1) * d] = attn[bb, hh] @ v[bb, :, hh * d:(hh + 1) * d]
    ref = out @ w["l.to_out.kernel"] + w["l.to_out.bias"]
    np.testing.assert_allclose(got, ref, rtol=1e-10, atol=1e-10)


def test_deepvit_reattention_vs_explicit_loops():
    """deepvit.py:79-87 restated with loops: softmax, head mix, LayerNorm over the HEAD axis of every (query, key) pair
    (eps 1e-3, biased variance, gamma / beta indexed by head), then P V."""
    rng = np.random.default_rng(6)
    b, h, n, d = 2, 4, 6, 3
    dim = h * d
    x = rng.standard_normal((b, n, dim))
    w = {"l.to_qkv.kernel": rng.standard_normal((dim, 3 * dim)), "l.reattn_weights": rng.standard_normal((h, h)),
         "l.reattn_norm.gamma": rng.uniform(0.5, 1.5, h), "l.reattn_norm.beta": rng.standard_normal(h)}
    got = S.attention_vit(x, w, "l.", h, d, deepvit=True)
    qkv = x @ w["l.to_qkv.kernel"]
    q, k, v = qkv[..., :dim], qkv[..., dim:2 * dim], qkv[..., 2 * dim:]
    attn = np.zeros((b, h, n, n))
    for bb in range(b):
        for hh in range(h):
            s = q[bb, :, hh * d:(hh + 1) * d] @ k[bb, :, hh * d:(hh + 1) * d].T * d ** -0.5
            e = np.exp(s - s.max(-1, keepdims=True))
            attn[bb, hh] = e / e.sum(-1, keepdims=True)
    mixed = _explicit_head_mix(attn, w["l.reattn_weights"])
    normed = np.zeros_like(mixed)
    for bb in range(b):
        for i in range(n):
            for j in range(n):
                col = mixed[bb, :, i, j]
                mu, var = col.mean(), ((col - col.mean()) ** 2).mean()
                normed[bb, :, i, j] = (col - mu) / np.sqrt(var + 1e-3) * w["l.reattn_norm.gamma"] + w["l.reattn_norm.beta"]
    ref = np.zeros((b, n, dim))
    for bb in range(b):
        for hh in range(h):
            ref[bb, :, hh * d:(hh + 1) * d] = normed[bb, hh] @ v[bb, :, hh * d:(hh + 1) * d]
    np.testing.assert_allclose(got, ref, rtol=1e-10, atol=1e-10)


def test_crossvit_cross_attention_vs_explicit_loops():
    """cross_vit.py:128-138 + 69-93 + 159-160 restated with loops: project_in -> LayerNorm of the query token only -> keys /
    values over [normed query ; raw context] (kv_include_self) -> per-head softmax attention -> to_out -> project_out -> + cls."""
    rng = np.random.default_rng(7)
    b, m, d_q, d_c, h, dh = 2, 5, 6, 10, 2, 4                                  # query branch width 6, context branch width 10
    cls, ctx = rng.standard_normal((b, 1, d_q)), rng.standard_normal((b, m, d_c))
    cfg = dict(cross_attn_heads=h, cross_attn_dim_head=dh)
    w = {"x.project_in.kernel": rng.standard_normal((d_q, d_c)), "x.project_in.bias": rng.standard_normal(d_c),
         "x.project_out.kernel": rng.standard_normal((d_c, d_q)), "x.project_out.bias": rng.standard_normal(d_q),
         "x.norm.gamma": rng.uniform(0.5, 1.5, d_c), "x.norm.beta": rng.standard_normal(d_c),
         "x.to_q.kernel": rng.standard_normal((d_c, h * dh)), "x.to_kv.kernel": rng.standard_normal((d_c, 2 * h * dh)),
         "x.to_out.kernel": rng.standard_normal((h * dh, d_c)), "x.to_out.bias": rng.standard_normal(d_c)}
    got = S._cross_attend(cls, ctx, w, cfg, "x.")
    ref = np.zeros_like(cls)
    for bb in range(b):
        x = cls[bb, 0] @ w["x.project_in.kernel"] + w["x.project_in.bias"]
        xn = (x - x.mean()) / np.sqrt(((x - x.mean()) ** 2).mean() + 1e-3) * w["x.norm.gamma"] + w["x.norm.beta"]
        rows = np.vstack([xn[None, :], ctx[bb]])                               # the normed query token is key / value row 0
        q = xn @ w["x.to_q.kernel"]
        kv = rows @ w["x.to_kv.kernel"]
        k, v = kv[:, :h * dh], kv[:, h * dh:]
        o = np.zeros(h * dh)
        for hh in range(h):
            s = k[:, hh * dh:(hh + 1) * dh] @ q[hh * dh:(hh + 1) * dh] * dh ** -0.5
            p = np.exp(s - s.max())
            o[hh * dh:(hh + 1) * dh] = (p / p.sum()) @ v[:, hh * dh:(hh + 1) * dh]
        y = o @ w["x.to_out.kernel"] + w["x.to_out.bias"]
        ref[bb, 0] = y @ w["x.project_out.kernel"] + w["x.project_out.bias"] + cls[bb, 0]
    np.testing.assert_allclose(got, ref, rtol=1e-10, atol=1e-10)


def test_patch_merger_vs_explicit_loops():
    """vit_with_patch_merger.py:49-55 with loops: LayerNorm, similarity of every learned query with every (scaled) token, softmax
    over the TOKENS, weighted sum of the normed tokens."""
    rng = np.random.default_rng(8)
    b, n, d, t = 2, 9, 6, 3
    x = rng.standard_normal((b, n, d))
    w = {"patch_merger.norm.gamma": rng.uniform(0.5, 1.5, d), "patch_merger.norm.beta": rng.standard_normal(d),
         "patch_merger.queries": rng.standard_normal((t, d))}
    got = S.patch_merger(x, w)
    ref = np.zeros((b, t, d))
    for bb in range(b):
        xn = np.stack([(r - r.mean()) / np.sqrt(((r - r.mean()) ** 2).mean() + 1e-3) * w["patch_merger.norm.gamma"]
                       + w["patch_merger.norm.beta"] for r in x[bb]])
        for tt in range(t):
            s = np.array([w["patch_merger.queries"][tt] @ (xn[i] * d ** -0.5) for i in range(n)])
            p = np.exp(s - s.max())
            ref[bb, tt] = (p / p.sum()) @ xn
    np.testing.assert_allclose(got, ref, rtol=1e-10, atol=1e-10)

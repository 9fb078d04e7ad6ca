"""ATS-ViT on the H100 (ats_vit.py): the fp32 engine against the float64 restatement with the same noise (identical draws and
returned ids), the bf16 engine teacher-forced to its own draws, a model that never samples against ViT, the captured-graph
replay of the noise counter, and the refusals."""
import ctypes as C
import os

import numpy as np
import pytest

import ats_oracle as o

pytestmark = pytest.mark.gpu

SMALL, BENCH = o.SMALL, o.BENCH
GOLDEN = os.path.join(os.path.dirname(__file__), "golden")


def build(cfg, precision, seed=0):
    from vit_tensorflow_b200 import ATSViT
    K = cfg["max_tokens_per_depth"]
    m = ATSViT(image_size=cfg["image"], patch_size=cfg["patch"], num_classes=5, dim=cfg["dim"], depth=len(K), max_tokens_per_depth=K,
               heads=cfg["heads"], mlp_dim=cfg["mlp_dim"], dim_head=cfg["dim_head"], precision=precision)
    w = o.weights(cfg, seed)
    m.set_weights_dict(w)
    return m, w


images = o.images


def can_sample(cfg, n0):
    """The layers whose input pitch lets them sample: P_0 = n0, P_{L+1} = 1 + min(P_L - 1, K_L)."""
    out, p = [], n0
    for L, k in enumerate(cfg["max_tokens_per_depth"]):
        if p - 1 > k:
            out.append(L)
        p = 1 + min(p - 1, k)
    return out


def engine_draws(m, cfg, n0):
    """{layer: draws} of every layer the engine sampled in its last forward."""
    got = {}
    for L in can_sample(cfg, n0):
        draws, _, sampled = m.last_draws(L)
        if sampled:
            got[L] = draws
    return got


@pytest.mark.parametrize("name", sorted(SMALL))
def test_fp32_matches_spec_and_reference_draw_for_draw(name):
    cfg = SMALL[name]
    m, w = build(cfg, "fp32")
    img = images(cfg, o.BATCH)
    ref = o.forward(w, img, cfg, seed=o.SEED)
    z = np.load(os.path.join(GOLDEN, f"ats_{name}__refshim.npz"))      # the reference's own ats_vit.py, same noise
    assert float(z["margin"]) >= 1e-3
    logits, ids = m(img, True, training=False)
    assert np.array_equal(np.asarray(ids), ref["token_ids"]) and np.array_equal(np.asarray(ids), z["token_ids_f32"])
    n0 = (cfg["image"][0] // cfg["patch"][0]) * (cfg["image"][1] // cfg["patch"][1]) + 1
    got = engine_draws(m, cfg, n0)
    assert sorted(got) == ref["sampled"]
    for L in ref["sampled"]:
        assert np.array_equal(got[L], ref["draws"][L])
    scale = max(np.abs(ref["logits"]).max(), 1.0)
    np.testing.assert_allclose(np.asarray(logits), ref["logits"], rtol=0, atol=2e-4 * scale)
    np.testing.assert_allclose(np.asarray(logits), z["logits_ref_f32"], rtol=0, atol=2e-4 * scale)


def test_fp32_smaller_image():
    cfg = SMALL["dh16_rect"]
    m, w = build(cfg, "fp32")
    img = images(cfg, 2, size=(12, 24))                  # pos_embedding[:, :n + 1]
    ref = o.forward(w, img, dict(cfg, image=(12, 24)), seed=0)
    logits, ids = m(img, True, training=False)
    assert np.array_equal(np.asarray(ids), ref["token_ids"])
    np.testing.assert_allclose(np.asarray(logits), ref["logits"], rtol=0, atol=2e-4 * max(np.abs(ref["logits"]).max(), 1.0))


def _bf16_forced(cfg, b):
    """The bf16 engine's draws, checked one by one: each must lie within delta of that draw's maximum under the oracle's perturbed
    pseudo-logits (the oracle forced to the engine's earlier draws, so that both hold the same tokens), delta derived from how far
    bf16 storage alone (forward_bf16_storage) moves those perturbed logits.  Then the logits of the oracle forced to all of them."""
    m, w = build(cfg, "bf16")
    img = images(cfg, b)
    logits, ids = m(img, True, training=False)
    n0 = (cfg["image"][0] // cfg["patch"][0]) * (cfg["image"][1] // cfg["patch"][1]) + 1
    forced = engine_draws(m, cfg, n0)
    ref = o.forward(w, img, cfg, seed=0, forced=forced)
    low = o.forward(w, img, cfg, seed=0, forced=forced, bf16_storage=True)
    assert sorted(forced) == ref["sampled"]
    for L, draws in forced.items():
        pert, pb = ref["pert"][L], low["pert"][L]
        live = pert > -1e300
        delta = 4.0 * np.abs(pert - pb)[live].max() + 1e-3
        chosen = np.take_along_axis(pert, draws[:, :, None].astype(np.int64) - 1, 2)[..., 0]
        assert (chosen >= pert.max(-1) - delta).all(), (L, delta, (pert.max(-1) - chosen).max())
    assert np.array_equal(np.asarray(ids), ref["token_ids"])
    err = np.linalg.norm(np.asarray(logits) - ref["logits"]) / np.linalg.norm(ref["logits"])
    assert err < 3e-2, err
    assert np.isfinite(np.asarray(logits)).all()


@pytest.mark.parametrize("name", sorted(SMALL))
def test_bf16_teacher_forced_small(name):
    _bf16_forced(SMALL[name], 3)


@pytest.mark.parametrize("name", sorted(BENCH))
def test_bf16_teacher_forced_bench(name):
    _bf16_forced(BENCH[name], 2)


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_no_sampling_is_vit(precision):
    from vit_tensorflow_b200 import ViT
    cfg = dict(SMALL["dh64"], max_tokens_per_depth=(200, 144, 144))
    m, w = build(cfg, precision)
    v = ViT(image_size=cfg["image"], patch_size=cfg["patch"], num_classes=5, dim=cfg["dim"], depth=3, heads=cfg["heads"],
            mlp_dim=cfg["mlp_dim"], dim_head=cfg["dim_head"], precision=precision)
    v.set_weights_dict(w)
    img = images(cfg, 4)
    logits, ids = m(img, True, training=False)
    assert np.array_equal(np.asarray(logits), np.asarray(v(img, training=False)))
    assert np.array_equal(np.asarray(ids), np.broadcast_to(np.arange(144), (4, 144)))


def test_graph_replay_and_seed():
    import torch
    cfg = SMALL["dh64"]
    m, w = build(cfg, "bf16")
    img = images(cfg, 4)
    stream = torch.cuda.Stream()
    m.set_sampling_seed(123)
    first = m.forward_ats(img, stream=stream.cuda_stream)          # eager
    second = m.forward_ats(img, stream=stream.cuda_stream)         # captured, then launched
    assert not np.array_equal(first[1], second[1])                  # the counter advanced: fresh draws
    m.set_sampling_seed(123)
    third = m.forward_ats(img, stream=stream.cuda_stream)           # replayed
    assert m.graph_stats()["replays"] >= 1 and m.graph_stats()["failures"] == 0
    assert np.array_equal(third[0], first[0]) and np.array_equal(third[1], first[1])
    fourth = m.forward_ats(img, stream=stream.cuda_stream)
    assert np.array_equal(fourth[0], second[0]) and np.array_equal(fourth[1], second[1])


def test_refusals_and_training_rule():
    from vit_tensorflow_b200 import ATSViT, _lib
    cfg = SMALL["dh32"]
    m, _ = build(cfg, "bf16")
    img = images(cfg, 1)
    with pytest.raises(_lib.VbError, match="whole forward only"):
        m.forward_tokens(np.zeros((1, 5, cfg["dim"]), np.float32))
    with pytest.raises(_lib.VbError, match="whole forward only"):
        m.forward_head(np.zeros((1, 5, cfg["dim"]), np.float32))
    d = ATSViT(image_size=32, patch_size=4, num_classes=5, dim=64, depth=1, max_tokens_per_depth=(8,), heads=2, mlp_dim=64, dropout=0.1)
    with pytest.raises(NotImplementedError):
        d(img)
    assert d(img, training=False).shape == (1, 5)
    cfgc = _lib.VbConfig()
    cfgc.struct_size = C.sizeof(_lib.VbConfig)
    cfgc.kind = _lib.KIND["ats_vit"]
    h = C.c_void_p()
    lib = _lib.load()
    assert lib.vb_create(C.byref(cfgc), 0, C.byref(h)) != 0


def test_profile_has_no_simt_gemm_in_bf16():
    """Every GEMM of the bf16 forward on the wgmma kernel (a GEMM off it would be profiled as 'other'): 'other' holds exactly the
    ATS kernels (ats_init, ats_sample + ats_gather per layer that can sample, the token-id output)."""
    cfg = BENCH["p16_384"]
    m, _ = build(cfg, "bf16")
    img = images(cfg, 2)
    m(img, training=False)
    m.profile(True)
    m.profile_read(reset=True)
    m(img, training=False)
    prof = m.profile_read()
    m.profile(False)
    depth = len(cfg["max_tokens_per_depth"])
    gemms = sum(prof[c]["launches"] for c in ("gemm_wgmma", "gemm_wgmma_gelu", "gemm_wgmma_residual"))
    assert gemms == 1 + 4 * depth                                 # patch embedding, then to_qkv, to_out, fc1, fc2 per layer
    assert prof["other"]["launches"] == 2 + 2 * len(can_sample(cfg, 577))
    assert prof["attention"]["launches"] == depth


def _numpy_sample(qkv, B, P, heads, dh, scale, rows, K, seed, counter):
    """ats_sample in float64 from the same (rounded) q|k|v: returns (perturbed logits [B][K, c_b], offsets)."""
    HD, C = heads * dh, max(rows) - 1
    out = []
    for b in range(B):
        c = rows[b] - 1
        x = qkv[b * P:b * P + c + 1].astype(np.float64)
        acc = np.zeros(c)
        for h in range(heads):
            q, k, v = x[0, h * dh:(h + 1) * dh], x[:, HD + h * dh:HD + (h + 1) * dh], x[:, 2 * HD + h * dh:2 * HD + (h + 1) * dh]
            s = k @ q * scale
            p = np.exp(s - s.max())
            p /= p.sum()
            acc += p[1:] * np.linalg.norm(v[1:], axis=1)
        lg = np.log(acc / (acc.sum() + 1e-6) + 1e-6)
        u = o.uniform((B, K, C), seed, counter)[b][:, C - c:]
        out.append(lg[None, :] - np.log(-np.log(u + 1e-6) + 1e-6))
    return out, [C - (r - 1) for r in rows]


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_op_ats_sample_against_numpy(precision):
    from vit_tensorflow_b200 import _lib
    B, P, heads, dh, K = 5, 97, 3, 64, 40
    rows = [97, 60, 41, 97, 2]
    rng = np.random.default_rng(5)
    qkv = rng.standard_normal((B * P, 3 * heads * dh)).astype(np.float32)
    if precision == "bf16":
        qkv = o.bf16_round(qkv).astype(np.float32)
    scale = 48 ** -0.5                                                # a widened head's model scale
    sel, rows_new, draws = _lib.op_ats_sample(qkv, B, P, heads, dh, scale, rows, K, seed=99, counter=7, precision=precision)
    pert, off = _numpy_sample(qkv, B, P, heads, dh, scale, rows, K, 99, 7)
    for b in range(B):
        best = pert[b].argmax(-1) + 1                                 # compact index
        top2 = np.sort(pert[b], -1)[:, -2:] if pert[b].shape[1] > 1 else np.zeros((K, 2)) + [0, 1]
        clear = top2[:, 1] - top2[:, 0] > (1e-4 if precision == "fp32" else 1e-3)
        chosen = draws[b] - off[b]
        assert (chosen >= 1).all() and (chosen <= rows[b] - 1).all()
        assert np.array_equal(chosen[clear], best[clear])
        assert (pert[b][np.arange(K), chosen - 1] >= pert[b].max(-1) - 1e-3).all()
        kept = np.unique(chosen)
        assert rows_new[b] == len(kept) + 1 and sel[b, 0] == 0 and np.array_equal(sel[b, 1:1 + len(kept)], kept)
    # C <= K: nothing drawn, every row kept
    sel, rows_new, draws = _lib.op_ats_sample(qkv, B, P, heads, dh, scale, [30, 20, 41, 2, 9], K, precision=precision)
    assert (draws == -1).all() and list(rows_new) == [30, 20, 41, 2, 9]
    assert np.array_equal(sel[2, :41], np.arange(41))


COUNTS = [1, 15, 16, 17, 63, 64, 65, 200, 256]


@pytest.mark.parametrize("n", [256, 401, 577])
def test_op_masked_flash_against_numpy(n):
    """Per-image key counts around the 16-key and 64-key block boundaries on the resident kernel (pitch <= 256) and the streaming
    one (pitch 401, 577)."""
    from vit_tensorflow_b200 import _lib
    B, heads, dh = len(COUNTS), 2, 64
    HD = heads * dh
    rng = np.random.default_rng(n)
    qkv = o.bf16_round(rng.standard_normal((B * n, 3 * HD))).astype(np.float32)
    _lib.last_attention_path()
    out, _ = _lib.op_masked_attention(qkv, B, n, heads, dh, COUNTS)
    assert _lib.last_attention_path() == "flash"
    assert np.isfinite(out).all()
    for b, c in enumerate(COUNTS):
        x = qkv[b * n:(b + 1) * n].astype(np.float64)
        for h in range(heads):
            q, k, v = x[:c, h * dh:(h + 1) * dh], x[:c, HD + h * dh:HD + (h + 1) * dh], x[:c, 2 * HD + h * dh:2 * HD + (h + 1) * dh]
            s = q @ k.T / 8.0
            p = np.exp(s - s.max(1, keepdims=True))
            p /= p.sum(1, keepdims=True)
            np.testing.assert_allclose(out[b * n:b * n + c, h * dh:(h + 1) * dh], p @ v, rtol=0, atol=3e-2)


def test_op_masked_fp32_path():
    from vit_tensorflow_b200 import _lib
    B, n, heads, dh = 3, 70, 2, 80
    HD = heads * dh
    nk = [1, 64, 70]
    qkv = np.random.default_rng(3).standard_normal((B * n, 3 * HD)).astype(np.float32)
    out, _ = _lib.op_masked_attention(qkv, B, n, heads, dh, nk, precision="fp32")
    assert np.isfinite(out).all()
    for b, c in enumerate(nk):
        x = qkv[b * n:(b + 1) * n].astype(np.float64)
        for h in range(heads):
            q, k, v = x[:, h * dh:(h + 1) * dh], x[:c, HD + h * dh:HD + (h + 1) * dh], x[:c, 2 * HD + h * dh:2 * HD + (h + 1) * dh]
            s = q @ k.T * dh ** -0.5
            p = np.exp(s - s.max(1, keepdims=True))
            p /= p.sum(1, keepdims=True)
            np.testing.assert_allclose(out[b * n:(b + 1) * n, h * dh:(h + 1) * dh], p @ v, rtol=0, atol=1e-4)

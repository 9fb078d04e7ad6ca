"""The small-dataset ViT on the H100 (vit_for_small_dataset.py): the fp32 and bf16 engines against the float64 restatement and
the reference's fixtures, locality self-attention's diagonal mask on both flash kernels and the materialised path
(vb_op_lsa_attention), SPT with its cls row (vb_op_spt), graph replay, and the refusals.

Tolerances are the ViT tests' (test_gpu_models.py): fp32 1e-4 + 1e-3 |ref|, bf16 6e-2 + 4e-2 |ref| per logit."""
import ctypes as C
import os

import numpy as np
import pytest

import small_vit_oracle as o

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
CASES = [(n, k) for n in sorted(o.SMALL) for k in o.WEIGHTS]


def fp32_tol(ref):
    return 1e-4 + 1e-3 * np.abs(ref)


def bf16_tol(ref):
    return 6e-2 + 4e-2 * np.abs(ref)


def build(cfg, precision, kind="init"):
    from vit_tensorflow_b200 import SmallDatasetViT
    m = SmallDatasetViT(image_size=cfg["image"], patch_size=cfg["patch"], num_classes=5, dim=cfg["dim"], depth=cfg["depth"],
                        heads=cfg["heads"], mlp_dim=cfg["mlp_dim"], pool=cfg["pool"], dim_head=cfg["dim_head"], precision=precision)
    w = o.weights(cfg, kind)
    m.set_weights_dict(w)
    return m, w


@pytest.mark.parametrize("name,kind", CASES)
def test_fp32_matches_reference_fixture_and_spec(name, kind):
    cfg = o.SMALL[name]
    m, w = build(cfg, "fp32", kind)
    img = o.images(cfg, o.BATCH)
    got = np.asarray(m(img, training=False))
    ref = o.forward(w, img, cfg)
    z = np.load(os.path.join(GOLDEN, f"small_vit_{name}__{kind}__refshim.npz"))
    assert (np.abs(got - ref) <= fp32_tol(ref)).all(), np.abs(got - ref).max()
    assert (np.abs(got - z["logits_ref_f32"]) <= fp32_tol(ref)).all()


@pytest.mark.parametrize("name,kind", CASES)
def test_bf16_matches_spec(name, kind):
    cfg = o.SMALL[name]
    m, w = build(cfg, "bf16", kind)
    img = o.images(cfg, o.BATCH)
    got = np.asarray(m(img, training=False))
    ref = o.forward(w, img, cfg)
    assert (np.abs(got - ref) <= bf16_tol(ref)).all(), np.abs(got - ref).max()


@pytest.mark.parametrize("name", sorted(o.BENCH))
def test_bf16_matches_spec_bench(name):
    cfg = o.BENCH[name]
    m, w = build(cfg, "bf16")
    img = o.images(cfg, 2)
    got = np.asarray(m(img, training=False))
    ref = o.forward(w, img, cfg)
    assert (np.abs(got - ref) <= bf16_tol(ref)).all(), np.abs(got - ref).max()


def _bf16(a):
    a = np.asarray(a, np.float32)
    u = a.view(np.uint32).astype(np.uint64)
    return (((u + 0x7FFF + ((u >> 16) & 1)) >> 16) << 16).astype(np.uint32).view(np.float32).astype(np.float64)


@pytest.mark.parametrize("dh", [32, 48, 64, 80])
@pytest.mark.parametrize("n", [2, 15, 16, 17, 63, 64, 65, 255, 256, 257, 577])
def test_lsa_attention_op(n, dh):
    """q = k and scale 4 / sqrt(dh): an unmasked diagonal would hold nearly all the weight (logit 4 sqrt(dh) against others of
    spread 4), so a missing mask shows as out ~ v_i.  bf16 runs the resident flash kernel up to 256 keys and the streaming one
    above, heads narrower than 64 widened; dh 80 and fp32 the materialised-scores path."""
    from vit_tensorflow_b200 import _lib
    B, heads = 2, 2
    HD = heads * dh
    rng = np.random.default_rng(n * 100 + dh)
    q = rng.standard_normal((B * n, HD)).astype(np.float32)
    v = rng.standard_normal((B * n, HD)).astype(np.float32)
    qkv = np.concatenate([q, q, v], 1)
    scale = 4.0 / np.sqrt(dh)
    for precision in ("bf16", "fp32") if n in (2, 65, 257) else ("bf16",):
        rnd = _bf16 if precision == "bf16" else (lambda a: np.asarray(a, np.float64))
        _lib.last_attention_path()
        out, _ = _lib.op_lsa_attention(qkv, B, n, heads, dh, scale, precision=precision)
        path = _lib.last_attention_path()
        assert path == ("flash" if precision == "bf16" and dh <= 64 else "simt"), path
        for b in range(B):
            for h in range(heads):
                qh = rnd(q[b * n:(b + 1) * n, h * dh:(h + 1) * dh])
                vh = rnd(v[b * n:(b + 1) * n, h * dh:(h + 1) * dh])
                want = o.lsa(qh, qh, vh, scale)
                got = out[b * n:(b + 1) * n, h * dh:(h + 1) * dh]
                np.testing.assert_allclose(got, want, rtol=0, atol=2e-2 if precision == "bf16" else 1e-4)
                if n > 2:
                    assert np.abs(want - vh).max() > 0.5          # the inputs do tell a missing mask apart


def test_lsa_attention_op_refuses_one_token():
    from vit_tensorflow_b200 import _lib
    with pytest.raises(_lib.VbError, match="n >= 2"):
        _lib.op_lsa_attention(np.zeros((2, 3 * 64), np.float32), 2, 1, 1, 64, 1.0)


@pytest.mark.parametrize("dim", [64, 96])
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_spt_op(precision, dim):
    """SPT with nonzero beta and bias plus cls and positions: row 0 must be exactly cls + pos[0] up to rounding, although the
    folded GEMM yields beta . W + bias on the zero cls row.  dim 64 folds the LayerNorm into the bf16 GEMM, dim 96 does not."""
    from vit_tensorflow_b200 import _lib
    cfg = dict(o.SMALL["rect_p4_dh80_mean"], dim=dim)
    w = o.weights(cfg, "stress")
    img = o.images(cfg, 3)
    rows = 1 + (16 // 4) * (32 // 4)
    cls, pos = w["cls_token"].reshape(dim), w["pos_embedding"].reshape(rows, dim)
    got = _lib.op_spt(img, 4, w["patch_norm.gamma"], w["patch_norm.beta"], w["patch.kernel"], w["patch.bias"], cls, pos, precision=precision)
    ref = o.embed(w, img, 4)
    tol = fp32_tol(ref) if precision == "fp32" else bf16_tol(ref)
    assert (np.abs(got - ref) <= tol).all(), np.abs(got - ref).max()
    assert (np.abs(got[:, 0] - (cls + pos[0])) <= tol[:, 0]).all()
    assert np.abs(w["patch_norm.beta"] @ w["patch.kernel"] + w["patch.bias"]).max() > 0.5   # the trap is armed
    from vit_tensorflow_b200 import SPT
    s = SPT(dim, 4, precision=precision)
    s.set_weights_dict({k: w[k] for k in s.weight_specs()})
    tok = np.asarray(s(img))
    no_pos = ref[:, 1:] - w["pos_embedding"][:, 1:]
    assert tok.shape == (3, rows - 1, dim) and (np.abs(tok - no_pos) <= tol[:, 1:]).all()


def test_graph_replay_bit_identical():
    import torch
    from vit_tensorflow_b200 import _lib
    cfg = o.SMALL["sq_p4_dh64"]
    m, _ = build(cfg, "bf16", "stress")
    img = torch.from_numpy(o.images(cfg, 8)).cuda()
    out = torch.empty(8, 5, device="cuda")
    s = torch.cuda.Stream()
    eager = np.asarray(m(img.cpu().numpy(), training=False))
    got = []
    for _ in range(3):                                   # eager, captured, replayed
        out.zero_()
        m.forward_raw(img.data_ptr(), _lib.MEM_DEVICE, 8, 32, 32, out.data_ptr(), _lib.MEM_DEVICE, s.cuda_stream)
        s.synchronize()
        got.append(out.cpu().numpy().copy())
    assert m.graph_stats()["replays"] >= 1
    for g in got:
        assert np.array_equal(g, eager)


def test_refusals():
    from vit_tensorflow_b200 import SmallDatasetViT, _lib
    cfg = o.SMALL["sq_p4_dh16"]
    m, _ = build(cfg, "fp32")
    img = o.images(cfg, 2)
    msg = "small-dataset ViT runs as a whole forward only"
    for call in (lambda: m.forward_embed(img), lambda: m.forward_tokens(np.zeros((2, 17, 32), np.float32)),
                 lambda: m.forward_head(np.zeros((2, 17, 32), np.float32)), lambda: m.to_patch(img),
                 lambda: m.patch_to_emb(np.zeros((2, 240), np.float32))):
        with pytest.raises(_lib.VbError, match=msg):
            call()
    buf = np.zeros(64, np.float32)
    rc = m._lib.vb_forward_distill(m._h, img.ctypes.data_as(C.c_void_p), _lib.MEM_HOST, 2, 16, 16, buf.ctypes.data_as(C.c_void_p),
                                   buf.ctypes.data_as(C.c_void_p), buf.ctypes.data_as(C.c_void_p), _lib.MEM_HOST, None)
    assert rc != 0 and msg in m._lib.vb_last_error(m._h).decode()
    with pytest.raises(ValueError):
        m(np.zeros((1, 16, 16, 4), np.float32), training=False)
    d = SmallDatasetViT(image_size=16, patch_size=4, num_classes=5, dim=32, depth=1, heads=2, mlp_dim=32, dropout=0.1, precision="fp32")
    with pytest.raises(NotImplementedError):
        d(img)
    assert np.asarray(d(img, training=False)).shape == (2, 5)

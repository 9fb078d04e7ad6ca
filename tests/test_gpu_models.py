"""GPU end-to-end parity: `Model(...)(img)` through the Python host classes -> C-ABI -> CUDA, against the oracle
on identical seeded weights/inputs.

fp32 engine path: BASELINE.json's gate, rtol=1e-3 / atol=1e-4 against the numpy-float64 spec.
bf16 engine path (wgmma / mma.sync): stated tolerance |err| <= 6e-2 + 4e-2*|ref| on O(1) logits (bf16 operands and bf16
activations with fp32 accumulation)."""
import json
import os

import numpy as np
import pytest

import oracle
from cases import MID, SMALL, cfg_of

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
BF16_RTOL, BF16_ATOL = 4e-2, 6e-2


def _model(cfg, precision):
    from vit_tensorflow_b200 import from_config
    return from_config(cfg, precision=precision)


@pytest.mark.parametrize("name", sorted(SMALL))
@pytest.mark.parametrize("gen", ["init_weights", "stress_weights"])
def test_fp32_gate_vs_oracle(lib, name, gen):
    cfg = cfg_of(name)
    w = getattr(oracle, gen)(cfg, 11)
    img = oracle.make_image(cfg, 2, 12)
    m = _model(cfg, "fp32")
    m.set_weights_dict(w)
    got = m(img, training=False)
    ref = oracle.forward_numpy(img, w, cfg)
    assert got.shape == ref.shape and got.dtype == np.float32
    np.testing.assert_allclose(got, ref, rtol=1e-3, atol=1e-4)
    assert m.last_launch_count > 0
    # committed golden fixture of the same case
    z = np.load(os.path.join(GOLDEN, f"{name}__{gen}.npz"))
    np.testing.assert_allclose(got, z["logits_f64"], rtol=1e-3, atol=1e-4)
    # ... and the logits the REFERENCE'S OWN CODE gave for it (unmodified vit_tensorflow modules over the numpy TensorFlow
    # stand-in, tests/golden/make_ref_golden.py): the CUDA path against the reference, not against our restatement
    zr = np.load(os.path.join(GOLDEN, f"{name}__{gen}__refshim.npz"))
    np.testing.assert_allclose(got, zr["logits_ref_f64"], rtol=1e-3, atol=1e-4)


@pytest.mark.parametrize("name", sorted(SMALL) + sorted(MID))
def test_bf16_vs_oracle(lib, name):
    cfg = cfg_of(name)
    w = oracle.stress_weights(cfg, 11)
    img = oracle.make_image(cfg, 3, 12)
    m = _model(cfg, "bf16")
    m.set_weights_dict(w)
    got = m(img, training=False)
    ref = oracle.forward_numpy(img, w, cfg)
    err = np.abs(got - ref)
    assert np.isfinite(got).all()
    assert (err <= BF16_ATOL + BF16_RTOL * np.abs(ref)).all(), f"max err {err.max():.4f} (|ref| mean {np.abs(ref).mean():.3f})"


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_smaller_image_truncates_pos_embedding(lib, precision):
    # vit.py:165: pos_embedding[:, :n+1]
    cfg = cfg_of("vit_small")
    w = oracle.stress_weights(cfg, 1)
    img = oracle.make_image(cfg, 2, 3, h=32, w=48)
    m = _model(cfg, precision)
    m.set_weights_dict(w)
    got = m(img, training=False)
    ref = oracle.forward_numpy(img, w, cfg)
    if precision == "fp32":
        np.testing.assert_allclose(got, ref, rtol=1e-3, atol=1e-4)
    else:
        assert (np.abs(got - ref) <= BF16_ATOL + BF16_RTOL * np.abs(ref)).all()


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_transformer_tokens_entry(lib, precision):
    # model.transformer(tokens) with arbitrary n (mae.py:69)
    from oracle import spec_numpy
    cfg = cfg_of("vit_small")
    w = oracle.stress_weights(cfg, 2)
    m = _model(cfg, precision)
    m.set_weights_dict(w)
    x = np.random.default_rng(0).standard_normal((3, 9, cfg["dim"])).astype(np.float32)
    got = m.transformer(x)
    ref = spec_numpy.transformer_tokens(x, w, cfg)
    if precision == "fp32":
        np.testing.assert_allclose(got, ref, rtol=1e-3, atol=1e-4)
    else:
        assert (np.abs(got - ref) <= 5e-2 + 3e-2 * np.abs(ref)).all()


@pytest.mark.parametrize("pool", ["cls", "mean"])
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_distillable_vit_forward(lib, precision, pool):
    # DistillMixin.call (distill.py:16-45): token appended as the last row, (logits, distill_tokens) returned
    from oracle import spec_numpy
    from vit_tensorflow_b200 import DistillableViT
    cfg = dict(cfg_of("vit_small"))
    cfg["pool"] = pool
    w = oracle.stress_weights(cfg, 4)
    kw = dict(image_size=(cfg["image_h"], cfg["image_w"]), patch_size=(cfg["patch_h"], cfg["patch_w"]), num_classes=cfg["num_classes"],
              dim=cfg["dim"], depth=cfg["depth"], heads=cfg["heads"], mlp_dim=cfg["mlp_dim"], pool=pool, dim_head=cfg["dim_head"])
    m = DistillableViT(precision=precision, **kw)
    m.set_weights_dict(w)
    img = oracle.make_image(cfg, 3, 8)
    tok = np.random.default_rng(3).standard_normal((1, 1, cfg["dim"])).astype(np.float32)
    logits, dist = m(img, tok, training=False)
    ref_l, ref_d = spec_numpy.forward_distill(img, tok, w, cfg)
    assert logits.shape == (3, cfg["num_classes"]) and dist.shape == (3, cfg["dim"])
    if precision == "fp32":
        np.testing.assert_allclose(logits, ref_l, rtol=1e-3, atol=1e-4)
        np.testing.assert_allclose(dist, ref_d, rtol=1e-3, atol=1e-4)
    else:
        assert (np.abs(logits - ref_l) <= BF16_ATOL + BF16_RTOL * np.abs(ref_l)).all()
        assert (np.abs(dist - ref_d) <= BF16_ATOL + BF16_RTOL * np.abs(ref_d)).all()
    # without a token the call is the plain ViT forward
    plain = m(img, training=False)
    refp = oracle.forward_numpy(img, w, cfg)
    tol = (1e-4 + 1e-3 * np.abs(refp)) if precision == "fp32" else (BF16_ATOL + BF16_RTOL * np.abs(refp))
    assert (np.abs(plain - refp) <= tol).all()


@pytest.mark.parametrize("name", ["vit_small", "vit_mean_rect", "cait_small", "merger_small", "t2t_small"])
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_stage_entries_embed_and_head(lib, name, precision):
    """vb_forward_embed / vb_forward_head: `call` before and after `self.transformer` (vit.py:160-166,170-175), the two stages the
    injected-transformer shell (efficient.py) and the wrappers' attribute surface are made of."""
    from oracle import spec_numpy
    cfg = cfg_of(name)
    w = oracle.stress_weights(cfg, 21)
    img = oracle.make_image(cfg, 3, 22)
    m = _model(cfg, precision)
    m.set_weights_dict(w)
    tol = (lambda r: 1e-4 + 1e-3 * np.abs(r)) if precision == "fp32" else (lambda r: BF16_ATOL + BF16_RTOL * np.abs(r))
    tok = m.forward_embed(img)
    ref_tok = spec_numpy.embed_tokens(img, w, cfg)
    assert tok.shape == ref_tok.shape
    assert (np.abs(tok - ref_tok) <= tol(ref_tok)).all()
    x = np.random.default_rng(5).standard_normal((3, 6, cfg["dim"])).astype(np.float32)
    got = m.forward_head(x)
    ref = spec_numpy.head_logits(x, w, cfg)
    assert (np.abs(got - ref) <= tol(ref)).all()
    np.testing.assert_array_equal(m.mlp_head(x[:, 0]), m.forward_head(x[:, :1]))   # model.mlp_head(x [b, dim])


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_patch_embedding_layers(lib, precision):
    """`patch_embedding.layers[:2]` = (Rearrange, Dense) as mae.py:37 / simmim.py:79 take them apart; `.layers[-1]` mpp.py:200."""
    from einops import rearrange
    cfg = cfg_of("vit_mean_rect")
    w = oracle.stress_weights(cfg, 2)
    img = oracle.make_image(cfg, 2, 3)
    m = _model(cfg, precision)
    m.set_weights_dict(w)
    to_patch, patch_to_emb = m.patch_embedding.layers[:2]
    patches = to_patch(img)
    np.testing.assert_array_equal(patches, rearrange(img, 'b (h p1) (w p2) c -> b (h w) (p1 p2 c)', p1=cfg["patch_h"], p2=cfg["patch_w"]))
    emb = patch_to_emb(patches)
    ref = patches.astype(np.float64) @ w["patch.kernel"].astype(np.float64) + w["patch.bias"]
    tol = (1e-4 + 1e-3 * np.abs(ref)) if precision == "fp32" else (BF16_ATOL + BF16_RTOL * np.abs(ref))
    assert emb.shape == ref.shape and (np.abs(emb - ref) <= tol).all()
    np.testing.assert_array_equal(m.patch_embedding(img), emb)
    assert m.pos_embedding.shape == (1, cfg["num_patches"] + 1, cfg["dim"]) and m.cls_token.shape == (1, 1, cfg["dim"])
    # mae.py:38 / simmim.py:80: `pixel_values_per_patch = self.patch_to_emb.weights[0].shape[0]`
    assert patch_to_emb.weights[0].shape[0] == cfg["patch_h"] * cfg["patch_w"] * 3 and len(patch_to_emb.weights) == 2
    np.testing.assert_array_equal(patch_to_emb.weights[0], w["patch.kernel"])
    np.testing.assert_array_equal(patch_to_emb.get_weights()[1], w["patch.bias"])


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_efficient_vit_shell(lib, precision):
    """efficient.ViT (efficient.py:12-55): embed -> injected transformer -> head.  With another engine model's `.transformer`
    injected and the same weights it must reproduce the plain ViT; with a Python callable the oracle composition."""
    from oracle import spec_numpy
    from vit_tensorflow_b200 import EfficientViT, ViT
    cfg = cfg_of("vit_small")
    w = oracle.stress_weights(cfg, 9)
    img = oracle.make_image(cfg, 3, 10)
    kw = dict(image_size=cfg["image_size"], patch_size=cfg["patch_size"], num_classes=cfg["num_classes"], dim=cfg["dim"])
    vit = ViT(depth=cfg["depth"], heads=cfg["heads"], mlp_dim=cfg["mlp_dim"], dim_head=cfg["dim_head"], precision=precision, **kw)
    vit.set_weights_dict(w)
    shell_w = {k: v for k, v in w.items() if not k.startswith("layers.")}
    eff = EfficientViT(transformer=vit.transformer, precision=precision, **kw)
    assert sorted(eff.weight_specs()) == sorted(shell_w)
    eff.set_weights_dict(shell_w)
    got = eff(img)
    ref = oracle.forward_numpy(img, w, cfg)
    tol = (1e-4 + 1e-3 * np.abs(ref)) if precision == "fp32" else (BF16_ATOL + BF16_RTOL * np.abs(ref))
    assert (np.abs(got - ref) <= tol).all()
    # an arbitrary callable: tokens -> 0.5 * tokens reversed along n
    eff2 = EfficientViT(transformer=lambda x, training=True: 0.5 * x[:, ::-1], pool="mean", precision=precision, **kw)
    eff2.set_weights_dict(shell_w)
    cfg2 = dict(cfg, pool="mean")
    ref2 = spec_numpy.head_logits(0.5 * spec_numpy.embed_tokens(img, w, cfg2)[:, ::-1], w, cfg2)
    got2 = eff2(img)
    tol2 = (1e-4 + 1e-3 * np.abs(ref2)) if precision == "fp32" else (BF16_ATOL + BF16_RTOL * np.abs(ref2))
    assert (np.abs(got2 - ref2) <= tol2).all()


def test_t2t_injected_transformer_and_smaller_image(lib):
    """T2TViT(transformer=...) (t2t.py:82-86) and a smaller image than configured (pos_embedding[:, :n+1], t2t.py:102)."""
    from oracle import spec_numpy
    from vit_tensorflow_b200 import T2TViT
    cfg = cfg_of("t2t_small")
    w = oracle.stress_weights(cfg, 13)
    m = _model(cfg, "fp32")
    m.set_weights_dict(w)
    img = oracle.make_image(cfg, 2, 14, h=24, w=24)
    np.testing.assert_allclose(m(img), oracle.forward_numpy(img, w, cfg), rtol=1e-3, atol=1e-4)
    inj = T2TViT(image_size=cfg["image_size"], num_classes=cfg["num_classes"], dim=cfg["dim"], t2t_layers=cfg["t2t_layers"],
                 transformer=m.transformer, precision="fp32")
    inj.set_weights_dict({k: v for k, v in w.items() if not k.startswith("layers.")})
    img = oracle.make_image(cfg, 2, 15)
    np.testing.assert_allclose(inj(img), oracle.forward_numpy(img, w, cfg), rtol=1e-3, atol=1e-4)


def test_patch_merger_never_merges_when_index_out_of_range(lib):
    # depth = 1 -> default(patch_merge_layer, depth // 2) - 1 = -1: the merger is never applied (vit_with_patch_merger.py:108,123)
    cfg = oracle.make_config("patch_merger_vit", image_size=32, patch_size=8, num_classes=4, dim=64, depth=1, heads=2, mlp_dim=64, dim_head=32)
    assert cfg["patch_merge_layer_index"] == -1
    w = oracle.stress_weights(cfg, 1)
    img = oracle.make_image(cfg, 2, 2)
    m = _model(cfg, "fp32")
    m.set_weights_dict(w)
    np.testing.assert_allclose(m(img), oracle.forward_numpy(img, w, cfg), rtol=1e-3, atol=1e-4)


@pytest.mark.parametrize("batch", [1, 7])
@pytest.mark.parametrize("name", ["vit_small", "vit_mid", "cait_small"])
def test_ragged_batches(lib, name, batch):
    """Batch sizes that do not fill a 128-row GEMM tile (1 image) or leave a ragged last tile (7 images x 197 rows)."""
    cfg = cfg_of(name)
    w = oracle.stress_weights(cfg, 31)
    img = oracle.make_image(cfg, batch, 32)
    m = _model(cfg, "bf16")
    m.set_weights_dict(w)
    got = m(img, training=False)
    ref = oracle.forward_numpy(img, w, cfg)
    assert got.shape == (batch, cfg["num_classes"])
    assert (np.abs(got - ref) <= BF16_ATOL + BF16_RTOL * np.abs(ref)).all()


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_deepvit_batch_times_heads_beyond_65535(lib, precision):
    """DeepViT with 16 heads at batch 4100 on a one-patch image (n = 2 tokens): the re-attention runs over 65 600 (image,
    head) items, more than a grid's y / z dimension holds (attn_generic_mma.cu rows path in bf16, kernels.cu SIMT path in fp32)."""
    cfg = oracle.make_config("deepvit", image_size=16, patch_size=16, num_classes=10, dim=64, depth=2, heads=16, mlp_dim=64,
                             dim_head=16)
    w = oracle.stress_weights(cfg, 41) if precision == "bf16" else oracle.init_weights(cfg, 41)
    img = oracle.make_image(cfg, 4100, 42)
    m = _model(cfg, precision)
    m.set_weights_dict(w)
    got = m(img, training=False)
    ref = oracle.forward_numpy(img, w, cfg)
    assert got.shape == (4100, 10)
    if precision == "fp32":
        np.testing.assert_allclose(got, ref, rtol=1e-3, atol=1e-4)
    else:
        assert (np.abs(got - ref) <= BF16_ATOL + BF16_RTOL * np.abs(ref)).all()


def test_batch_independence_and_determinism(lib):
    """Images are independent (no cross-sample op): logits of a batch equal logits of its halves, bit for bit,
    and repeated calls are bit-identical (what the data-parallel sharding relies on)."""
    cfg = cfg_of("vit_mid")
    w = oracle.init_weights(cfg, 5)
    img = oracle.make_image(cfg, 4, 6)
    m = _model(cfg, "bf16")
    m.set_weights_dict(w)
    full = m(img, training=False)
    again = m(img, training=False)
    np.testing.assert_array_equal(full, again)
    halves = np.concatenate([m(img[:2], training=False), m(img[2:], training=False)])
    np.testing.assert_array_equal(full, halves)


def test_full_size_batch_permutation_equivariance(lib):
    """BASELINE.json configs[1] at full size (ViT-B/16 224^2, batch 256 -- far beyond what the CPU oracle finishes in seconds),
    through a size-independent property of the path: images are independent, so permuting the batch permutes the logits, bit
    for bit (M = 50 432 token rows = 394 full GEMM tiles whose boundaries fall inside images; every (image, head) attention
    item lands on a different CTA).  Plus finiteness and a non-degenerate spread of the logits."""
    cfg = oracle.make_config("vit", image_size=224, patch_size=16, num_classes=1000, dim=768, depth=12, heads=12, mlp_dim=3072)
    m = _model(cfg, "bf16")                       # random init from the reference's distributions (host class, seed None)
    rng = np.random.default_rng(7)
    img = rng.standard_normal((256, 224, 224, 3), dtype=np.float32)
    perm = rng.permutation(256)
    a = m(img, training=False)
    b = m(img[perm], training=False)
    assert a.shape == (256, 1000) and np.isfinite(a).all() and a.std() > 1e-3
    np.testing.assert_array_equal(a[perm], b)


def test_native_dp_single_rank_allgather(lib, tmp_path):
    """vb_dp_init / vb_forward_allgather (SURVEY.md 8e through the C-ABI itself) with a world of one rank: the in-place
    ncclAllGather must leave exactly vb_forward's logits in the gather buffer.  Three calls under a torch side stream: eager,
    graph capture and graph replay of the forward in front of the collective (checked through graph_stats).  Runs in a child
    process (its own NCCL communicator, with a time limit); any failure fails the test.  The 2-GPU form of the same check is
    tools/dp_check.py, run on two or more GPUs."""
    import subprocess
    import sys
    code = r"""
import sys, numpy as np, torch
sys.path.insert(0, %r)
import oracle
from vit_tensorflow_b200 import from_config
from vit_tensorflow_b200.runtime import NativeDataParallel
cfg = oracle.make_config("vit", image_size=64, patch_size=16, num_classes=10, dim=64, depth=2, heads=4, mlp_dim=128, dim_head=16)
m = from_config(cfg, precision="bf16", seed=3)
img = oracle.make_image(cfg, 4, 5)
ref = m(img, training=False)
dp = NativeDataParallel(m, 4, (64, 64), rank=0, world=1, id_bytes=None)
x = torch.from_numpy(img).cuda()
s = torch.cuda.Stream()
torch.cuda.synchronize()
st0 = m.graph_stats()
for _ in range(3):
    with torch.cuda.stream(s):
        out = dp.forward_device(x)
    s.synchronize()
    np.testing.assert_array_equal(out.cpu().numpy(), ref)
st = m.graph_stats()
delta = (st["captures"] - st0["captures"], st["replays"] - st0["replays"], st["failures"] - st0["failures"])
assert delta == (1, 1, 0), (delta, st["last_failure"])
print("native dp ok")
""" % os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "native dp ok" in r.stdout, "native NCCL data-parallel path failed:\n" + r.stdout[-400:] + r.stderr[-1200:]


def test_dropout_training_semantics(lib):
    from vit_tensorflow_b200 import ViT
    m = ViT(image_size=32, patch_size=16, num_classes=4, dim=64, depth=1, heads=2, mlp_dim=64, dim_head=32, dropout=0.1,
            precision="fp32")
    img = np.zeros((1, 32, 32, 3), np.float32)
    with pytest.raises(NotImplementedError):
        m(img)                     # training=True default + dropout > 0 (vit.py:159)
    assert m(img, training=False).shape == (1, 4)

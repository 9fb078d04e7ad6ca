"""GPU: the captured-graph forward, and the serving wrappers that run it, give the same bits as the eager forward.

On any stream but the NULL / legacy one, `vb_forward` runs a (image pointer, logits pointer, batch, h, w, stream) key eagerly on
its first call, captures the whole forward into a CUDA graph on its second and replays that graph from the third on
(engine.cu, vb_forward).  The replay is what `runtime.HostPipeline`, `DataParallel` / `NativeDataParallel` under a side stream
and any caller of `forward_raw` with a stream are served by.  It is right only if the host-side state captured on call 2
(workspace pointers, TMA descriptors, cached patch-embedding residuals, staging buffers, packed weights, side streams, head-mix
parameters) is still valid on call N.

"Eager" is the same model called on the NULL stream (`model(img)`).  Results are compared bit for bit: the kernels are
deterministic (test_gpu_models.py::test_batch_independence_and_determinism).  Every case asserts the `graph_stats()` deltas it
expects, so a capture that silently fell back to eager fails the test instead of passing on eager results."""
import numpy as np
import pytest
import torch

import oracle
from cases import MID, SMALL

pytestmark = pytest.mark.gpu

BF16_RTOL, BF16_ATOL = 4e-2, 6e-2          # the bf16 bound of test_gpu_models.py

# DeepViT / CaiT with 8 and 16 heads over 65 tokens: the head-mixing attention runs on attn_generic_mma.cu's rows path, which
# reads the mix weights back once per weight set and passes them as kernel parameters (attention_mix_params)
ROWS = {
    "deepvit_h8": dict(kind="deepvit", image_size=64, patch_size=8, num_classes=10, dim=128, depth=2, heads=8, mlp_dim=128, dim_head=16),
    "deepvit_h16": dict(kind="deepvit", image_size=64, patch_size=8, num_classes=10, dim=128, depth=2, heads=16, mlp_dim=128,
                        dim_head=16),
    "cait_h8": dict(kind="cait", image_size=64, patch_size=8, num_classes=10, dim=128, depth=2, cls_depth=1, heads=8, mlp_dim=128,
                    dim_head=16),
    "cait_h16": dict(kind="cait", image_size=64, patch_size=8, num_classes=10, dim=128, depth=2, cls_depth=1, heads=16, mlp_dim=128,
                     dim_head=16),
}
# patch 14: a patch row segment is pw * C = 42 floats, not a multiple of 4, so im2col takes its scalar form
PATCH14 = dict(kind="vit", image_size=56, patch_size=14, num_classes=10, dim=64, depth=2, heads=4, mlp_dim=128, dim_head=16)


def _cfg(name):
    d = dict({**SMALL, **MID, **ROWS, "vit_patch14": PATCH14}[name])
    return oracle.make_config(d.pop("kind"), **d)


def _model(cfg, precision, w):
    from vit_tensorflow_b200 import from_config
    m = from_config(cfg, precision=precision)
    m.set_weights_dict(w)
    m.build()
    return m


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _launch(m, x, out, s):
    """The forward of device image `x` ([b, h, w, 3], any contiguous view) into device logits `out` on stream `s`."""
    from vit_tensorflow_b200 import _lib
    assert x.is_contiguous() and out.is_contiguous()
    b, h, w, _ = x.shape
    m.forward_raw(x.data_ptr(), _lib.MEM_DEVICE, b, h, w, out.data_ptr(), _lib.MEM_DEVICE, s.cuda_stream)


def _fwd(m, x, out, s):
    """_launch, then wait for it and return the logits.  The wait also orders this call before the next one on any stream: the
    calls of one handle share its workspace."""
    _launch(m, x, out, s)
    s.synchronize()
    return out.cpu().numpy()


def _fwd_host(m, img, out, s):
    from vit_tensorflow_b200 import _lib
    b, h, w, _ = img.shape
    m.forward_raw(img.ctypes.data, _lib.MEM_HOST, b, h, w, out.ctypes.data, _lib.MEM_HOST, s.cuda_stream)
    return out.copy()


def _expect(m, before, captures, replays):
    st = m.graph_stats()
    got = (st["captures"] - before["captures"], st["replays"] - before["replays"], st["failures"] - before["failures"])
    assert got == (captures, replays, 0), f"(captures, replays, failures) deltas {got}; last capture failure: {st['last_failure']!r}"


def _eq(got, ref):
    np.testing.assert_array_equal(got, ref)


# ---------------------------------------------------------------------------------------------------------- every model kind
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("name", sorted(SMALL) + sorted(ROWS) + ["t2t_mid"])
def test_capture_and_replay_equal_eager(lib, name, precision):
    """Calls 1-4 of one key (eager, capture, replay, replay) equal the eager forward; a replay after the image buffer was
    overwritten in place computes the new image.  Once with device buffers, once with host image and host logits (the engine's
    staging buffers are then the key)."""
    cfg = _cfg(name)
    m = _model(cfg, precision, oracle.stress_weights(cfg, 11))
    B, nc = 2, cfg["num_classes"]
    img1, img2 = oracle.make_image(cfg, B, 12), oracle.make_image(cfg, B, 13)
    e1, e2 = m(img1, training=False), m(img2, training=False)
    assert np.isfinite(e1).all() and np.isfinite(e2).all() and not np.array_equal(e1, e2)
    s = torch.cuda.Stream()

    x, x2, out = _dev(img1), _dev(img2), torch.full((B, nc), float("nan"), device="cuda")
    torch.cuda.synchronize()
    st = m.graph_stats()
    for cap, rep in ((0, 0), (1, 0), (1, 1), (1, 2)):
        _eq(_fwd(m, x, out, s), e1)
        _expect(m, st, cap, rep)
    with torch.cuda.stream(s):
        x.copy_(x2)                                   # same pointer, new image
    _eq(_fwd(m, x, out, s), e2)
    _expect(m, st, 1, 3)

    himg, hout = img1.copy(), np.full((B, nc), np.nan, np.float32)
    st = m.graph_stats()
    for cap, rep in ((0, 0), (1, 0), (1, 1), (1, 2)):
        _eq(_fwd_host(m, himg, hout, s), e1)
        _expect(m, st, cap, rep)
    himg[...] = img2
    _eq(_fwd_host(m, himg, hout, s), e2)
    _expect(m, st, 1, 3)


# ------------------------------------------------------------------------------------------------- keys that change in between
@pytest.mark.parametrize("name,precision,small_hw", [
    ("vit_small", "fp32", 48), ("vit_small", "bf16", 48), ("deepvit_h8", "bf16", 48), ("cait_h16", "bf16", 48),
    ("t2t_small", "bf16", 24), ("crossvit_small", "bf16", 48),
])
def test_interleaved_keys(lib, name, precision, small_hw):
    """Batch 2, 5, 2 on one buffer, a smaller image (pos_embedding truncation) and the first key again on a second stream,
    round-robin three times: every call equals the eager forward of what it was given."""
    cfg = _cfg(name)
    m = _model(cfg, precision, oracle.stress_weights(cfg, 21))
    nc = cfg["num_classes"]
    big = oracle.make_image(cfg, 5, 22)
    small = oracle.make_image(cfg, 2, 23, h=small_hw, w=small_hw)
    ref2, ref5, refs = m(big[:2], training=False), m(big, training=False), m(small, training=False)
    xb, xs, out = _dev(big), _dev(small), torch.empty((5, nc), device="cuda")
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    torch.cuda.synchronize()
    st = m.graph_stats()
    calls = [(xb[:2], s1, ref2), (xb, s1, ref5), (xb[:2], s1, ref2), (xs, s1, refs), (xb[:2], s2, ref2)]
    for _ in range(3):
        for x, s, ref in calls:
            _eq(_fwd(m, x, out[:x.shape[0]], s), ref)
    # keys: (2, s1) six calls -> 1 capture + 4 replays; (5, s1), (small, s1), (2, s2) three calls each -> 1 + 1
    _expect(m, st, 4, 7)


# ------------------------------------------------------------------------------------------------------------- invalidation
@pytest.mark.parametrize("name", ["vit_small", "cait_h8"])
def test_residual_cache_eviction_recaptures(lib, name):
    """Seven batch sizes overflow the per-handle cache of patch-embedding residuals (6 entries), which drops every graph: the
    key captured before must run eagerly, capture again and replay, all equal to eager."""
    cfg = _cfg(name)
    m = _model(cfg, "bf16", oracle.stress_weights(cfg, 31))
    img = oracle.make_image(cfg, 7, 32)
    refs = {b: m(img[:b], training=False) for b in range(1, 8)}
    x, out = _dev(img), torch.empty((7, cfg["num_classes"]), device="cuda")
    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    st = m.graph_stats()
    for _ in range(2):
        _eq(_fwd(m, x[:1], out[:1], s), refs[1])
    _expect(m, st, 1, 0)
    for b in range(2, 8):
        _eq(_fwd(m, x[:b], out[:b], s), refs[b])
    _expect(m, st, 1, 0)
    for _ in range(3):                                # dropped: eager, capture, replay -- not a replay of the old graph
        _eq(_fwd(m, x[:1], out[:1], s), refs[1])
    _expect(m, st, 2, 1)


def test_more_keys_than_the_graph_map_holds(lib):
    """70 batch-1 keys (image-aligned views of one device buffer, one logits row each), three calls per key: the map of graphs
    is dropped when a call finds more than 64 keys in it, and every result stays equal to eager.  That happens on the second
    call of key 64 (the 65th), which then runs eagerly again and captures on its third call: 70 captures, 69 replays.  The
    first key, dropped, captures again."""
    cfg = _cfg("vit_small")
    m = _model(cfg, "bf16", oracle.stress_weights(cfg, 41))
    n = 70
    img = oracle.make_image(cfg, n, 42)
    refs = [m(img[i:i + 1], training=False) for i in range(n)]
    x, out = _dev(img), torch.empty((n, cfg["num_classes"]), device="cuda")
    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    st = m.graph_stats()
    for i in range(n):
        for _ in range(3):
            _eq(_fwd(m, x[i:i + 1], out[i:i + 1], s), refs[i])
    _expect(m, st, n, n - 1)
    for _ in range(3):
        _eq(_fwd(m, x[:1], out[:1], s), refs[0])
    _expect(m, st, n + 1, n)


@pytest.mark.parametrize("name,changed", [
    ("deepvit_h8", None), ("deepvit_h8", "layers.1.reattn_weights"),
    ("cait_h8", None), ("cait_h8", "patch_transformer.layers.0.mix_post"),
])
def test_weights_reloaded_after_replays(lib, name, changed):
    """set_weights_dict after replays: the whole dict, or one head-mix matrix only (same device pointer, new values).  The next
    eager, capture and replay calls equal a fresh model built with the new weights."""
    cfg = _cfg(name)
    w1 = oracle.stress_weights(cfg, 51)
    if changed is None:
        w2 = oracle.stress_weights(cfg, 52)
    else:
        w2 = dict(w1)
        w2[changed] = np.random.default_rng(53).standard_normal(w1[changed].shape).astype(np.float32)
    img = oracle.make_image(cfg, 2, 54)
    m = _model(cfg, "bf16", w1)
    ref1 = m(img, training=False)
    fresh = _model(cfg, "bf16", w2)
    ref2 = fresh(img, training=False)
    fresh.close()
    assert not np.array_equal(ref1, ref2)
    x, out = _dev(img), torch.empty((2, cfg["num_classes"]), device="cuda")
    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    st = m.graph_stats()
    for _ in range(3):
        _eq(_fwd(m, x, out, s), ref1)
    _expect(m, st, 1, 1)
    m.set_weights_dict(w2 if changed is None else {changed: w2[changed]})
    for _ in range(3):
        _eq(_fwd(m, x, out, s), ref2)
    _expect(m, st, 2, 2)


@pytest.mark.parametrize("name", ["cait_h8", "t2t_small", "crossvit_small"])
def test_profiling_toggled_around_replays(lib, name):
    """Profiled calls run eagerly (one stream: T2T and CrossViT do not fork while profiling) and give the same bits; replays
    resume once profiling is off."""
    cfg = _cfg(name)
    m = _model(cfg, "bf16", oracle.stress_weights(cfg, 61))
    img = oracle.make_image(cfg, 2, 62)
    ref = m(img, training=False)
    x, out = _dev(img), torch.empty((2, cfg["num_classes"]), device="cuda")
    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    st = m.graph_stats()
    for _ in range(3):
        _eq(_fwd(m, x, out, s), ref)
    _expect(m, st, 1, 1)
    m.profile(True)
    for _ in range(2):
        _eq(_fwd(m, x, out, s), ref)
    _expect(m, st, 1, 1)
    m.profile(False)
    assert sum(v["launches"] for v in m.profile_read().values()) > 0
    for _ in range(2):
        _eq(_fwd(m, x, out, s), ref)
    _expect(m, st, 1, 3)


# ------------------------------------------------------------------------------------------------------------- two handles
def test_other_handles_do_not_break_a_capture(lib):
    """Handle A (CaiT, 8 heads: head-mix parameters cached per weight set) runs its first call, then another handle is created
    and finalized, an op-level attention call runs, or a third handle is created and destroyed: A's second call must still
    capture, and A's replays equal A eager.  Then A and B interleaved on one stream and on two streams."""
    from vit_tensorflow_b200 import _lib
    ca, cb = _cfg("cait_h8"), _cfg("deepvit_h8")
    wa = oracle.stress_weights(ca, 71)
    A = _model(ca, "bf16", wa)
    ia, ib = oracle.make_image(ca, 2, 72), oracle.make_image(cb, 3, 73)
    ra = A(ia, training=False)
    xa = _dev(ia)
    outs = [torch.empty((2, ca["num_classes"]), device="cuda") for _ in range(3)]     # one key of A per disturbance
    s, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    torch.cuda.synchronize()
    st = A.graph_stats()

    _eq(_fwd(A, xa, outs[0], s), ra)
    B = _model(cb, "bf16", oracle.stress_weights(cb, 74))              # vb_create + vb_finalize of another handle
    rb = B(ib, training=False)
    _eq(_fwd(A, xa, outs[0], s), ra)
    _expect(A, st, 1, 0)
    for _ in range(2):
        _eq(_fwd(A, xa, outs[0], s), ra)
    _expect(A, st, 1, 2)

    rng = np.random.default_rng(75)
    q, k, v = (rng.standard_normal((2, 65, 128)).astype(np.float32) for _ in range(3))
    mix = [rng.standard_normal((8, 8)).astype(np.float32) for _ in range(2)]
    _eq(_fwd(A, xa, outs[1], s), ra)
    _lib.op_attention(q, k, v, 8, variant=2, mix_a=mix[0], mix_b=mix[1])    # op-level entry with head-mix weights of its own
    _eq(_fwd(A, xa, outs[1], s), ra)
    _expect(A, st, 2, 2)

    _eq(_fwd(A, xa, outs[2], s), ra)
    C = _model(cb, "bf16", oracle.stress_weights(cb, 76))
    C(ib, training=False)
    C.close()
    _eq(_fwd(A, xa, outs[2], s), ra)
    _eq(_fwd(A, xa, outs[2], s), ra)
    _expect(A, st, 3, 3)

    xb, ob = _dev(ib), torch.empty((3, cb["num_classes"]), device="cuda")
    torch.cuda.synchronize()
    stb = B.graph_stats()
    for _ in range(3):                                                # one stream
        _eq(_fwd(A, xa, outs[0], s), ra)
        _eq(_fwd(B, xb, ob, s), rb)
    for _ in range(3):                                                # two streams, A and B in flight together
        _launch(A, xa, outs[0], s)
        _launch(B, xb, ob, s2)
        s.synchronize()
        s2.synchronize()
        _eq(outs[0].cpu().numpy(), ra)
        _eq(ob.cpu().numpy(), rb)
    _expect(A, st, 3, 9)
    _expect(B, stb, 2, 2)                                             # (B, s): eager, capture, replay; (B, s2): the same


# ----------------------------------------------------------------------------------------------------------- serving wrappers
def test_host_pipeline_serves_replays(lib):
    """runtime.HostPipeline over DataParallel (world 1): six submits of different pinned images; every returned buffer equals
    the eager forward of the previous submit's image and flush() that of the last.  The two device input buffers are two
    keys: each is captured once, on its second use, and replayed on its third."""
    from vit_tensorflow_b200.runtime import DataParallel, HostPipeline
    cfg = _cfg("cait_h8")
    m = _model(cfg, "bf16", oracle.stress_weights(cfg, 81))
    B = 3
    imgs = [oracle.make_image(cfg, B, 82 + i) for i in range(6)]
    refs = [m(img, training=False) for img in imgs]
    pinned = [torch.from_numpy(img).pin_memory() for img in imgs]
    pipe = HostPipeline(DataParallel(m, B, (cfg["image_h"], cfg["image_w"]), rank=0, world=1))
    st = m.graph_stats()
    for i, img in enumerate(pinned):
        prev = pipe.submit(img)
        if i == 0:
            assert prev is None
        else:
            _eq(prev.numpy(), refs[i - 1])
    _eq(pipe.flush().numpy(), refs[-1])
    _expect(m, st, 2, 2)


# -------------------------------------------------------------------------------------------- device buffers as callers pass them
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_unaligned_device_image(lib, precision):
    """A device image at a storage offset of one float (not 16-byte aligned: the scalar im2col) gives the logits of an aligned
    copy, eagerly and replayed."""
    cfg = _cfg("vit_small")
    m = _model(cfg, precision, oracle.stress_weights(cfg, 91))
    img = oracle.make_image(cfg, 3, 92)
    ref = m(img, training=False)
    flat = torch.empty(img.size + 1, device="cuda")
    x = flat[1:].view(img.shape)
    x.copy_(_dev(img))
    assert x.data_ptr() % 16 != 0
    out = torch.empty((3, cfg["num_classes"]), device="cuda")
    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    st = m.graph_stats()
    for _ in range(3):
        _eq(_fwd(m, x, out, s), ref)
    _expect(m, st, 1, 1)


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_patch14_scalar_im2col_vs_oracle(lib, precision):
    """ViT with 14 x 14 patches (pw * C = 42: the scalar im2col on every call) against the float64 oracle, within the bounds of
    test_gpu_models.py; the captured forward equals the eager one."""
    cfg = _cfg("vit_patch14")
    w = oracle.stress_weights(cfg, 95)
    m = _model(cfg, precision, w)
    img = oracle.make_image(cfg, 3, 96)
    got = m(img, training=False)
    ref = oracle.forward_numpy(img, w, cfg)
    if precision == "fp32":
        np.testing.assert_allclose(got, ref, rtol=1e-3, atol=1e-4)
    else:
        err = np.abs(got - ref)
        assert (err <= BF16_ATOL + BF16_RTOL * np.abs(ref)).all(), f"max err {err.max():.4f}"
    x, out = _dev(img), torch.empty((3, cfg["num_classes"]), device="cuda")
    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    st = m.graph_stats()
    for _ in range(3):
        _eq(_fwd(m, x, out, s), got)
    _expect(m, st, 1, 1)


@pytest.mark.parametrize("name", ["vit_small", "crossvit_small"])
def test_logits_into_a_row_slice(lib, name):
    """Logits written into rows [3, 3 + B) of a larger device buffer (CrossViT accumulates its second head into them): the rows
    outside the slice keep their contents, eagerly and replayed."""
    cfg = _cfg(name)
    m = _model(cfg, "bf16", oracle.stress_weights(cfg, 97))
    B, nc = 2, cfg["num_classes"]
    img = oracle.make_image(cfg, B, 98)
    ref = m(img, training=False)
    big = torch.full((B + 6, nc), 7.25, device="cuda")
    out = big[3:3 + B]
    x = _dev(img)
    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    st = m.graph_stats()
    for _ in range(3):
        _eq(_fwd(m, x, out, s), ref)
        whole = big.cpu().numpy()
        assert (whole[:3] == 7.25).all() and (whole[3 + B:] == 7.25).all()
    _expect(m, st, 1, 1)

"""CPU checks of the float64 references in test_gpu_conv_ops.py, at every case shape it runs, against independent statements of
the same operations: the convolution against spec_numpy.extract_patches_same(...) @ W (SAME) and torch.nn.functional.conv2d in
float64 with the TF padding written out by F.pad (as cct_oracle.forward_torch does); the ReLU + max-pool against
cct_oracle.maxpool_same; the sequence pooling against its float64 torch restatement (cct_oracle.forward_torch's)."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import cct_oracle
from oracle import spec_numpy
from test_gpu_conv_ops import (CONV_CASES, PAD_SHAPES, POOL_CASES, SEQ_CASES, conv_operands, conv_ref, gelu, layer_norm,
                               maxpool_relu_ref, out_geometry, pool_operands, seq_operands, seq_pool_ref)


def _torch_conv(x, kernel, k, s, valid):
    """float64 torch: NCHW, the TF SAME padding (smaller half first) spelled out by F.pad."""
    t = torch.from_numpy(np.asarray(x, np.float64)).permute(0, 3, 1, 2)
    if not valid:
        H, W = t.shape[-2:]
        oh, ow = -(-H // s), -(-W // s)
        ph, pw = max((oh - 1) * s + k - H, 0), max((ow - 1) * s + k - W, 0)
        t = F.pad(t, (pw // 2, pw - pw // 2, ph // 2, ph - ph // 2))
    w = torch.from_numpy(np.asarray(kernel, np.float64)).permute(3, 2, 0, 1)
    return F.conv2d(t, w, stride=s).permute(0, 2, 3, 1).numpy()


def _check_conv(B, H, W, cin, N, k, s, valid, seed):
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((B, H, W, cin))
    kernel = rng.standard_normal((k, k, cin, N)) / np.sqrt(k * k * cin)
    got = conv_ref(x, kernel, s, valid)
    oh, ow = out_geometry(H, k, s, valid)[0], out_geometry(W, k, s, valid)[0]
    assert got.shape == (B, oh, ow, N)
    np.testing.assert_allclose(got, _torch_conv(x, kernel, k, s, valid), rtol=1e-12, atol=1e-12)
    if not valid:
        patches = spec_numpy.extract_patches_same(x, k, s)
        np.testing.assert_allclose(got, patches @ kernel.reshape(-1, N), rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("c", CONV_CASES, ids=[c["id"] for c in CONV_CASES])
def test_conv_reference(c):
    N = min(c["N"], 16)                                           # the output width does not change the geometry
    B = 1 if c["B"] * c["H"] * c["W"] > 10000 else c["B"]
    _check_conv(B, c["H"], c["W"], c["cin"], N, c["k"], c["s"], c["valid"], len(c["id"]))


@pytest.mark.parametrize("cin", [64, 20])
@pytest.mark.parametrize("H,W,s", PAD_SHAPES)
def test_conv_reference_padded_tap_shapes(H, W, s, cin):
    _check_conv(2, H, W, cin, 8, 3, s, False, H * W + s + cin)


@pytest.mark.parametrize("c", [c for c in CONV_CASES if c["ln"] is not None or c["gelu_in"]], ids=lambda c: c["id"])
def test_on_load_transform_reference(c):
    """The LayerNorm (biased variance, eps) and exact-erf GELU the conv reference applies before the convolution."""
    x, _, _, gamma, beta, _ = conv_operands(c)
    v = x[:, c["off"]:c["off"] + c["cin"]].astype(np.float64)
    t = torch.from_numpy(v)
    if c["ln"] is not None:
        got = layer_norm(v, gamma.astype(np.float64), beta.astype(np.float64), c["ln"])
        t = F.layer_norm(t, (c["cin"],), torch.from_numpy(gamma.astype(np.float64)), torch.from_numpy(beta.astype(np.float64)), eps=c["ln"])
        np.testing.assert_allclose(got, t.numpy(), rtol=1e-9, atol=1e-9)
        v = got
    if c["gelu_in"]:
        np.testing.assert_allclose(gelu(v), F.gelu(torch.from_numpy(v)).numpy(), rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("with_pos", [False, True])
@pytest.mark.parametrize("k,s,H,W,C", POOL_CASES)
def test_maxpool_reference(k, s, H, W, C, with_pos):
    x, pos, rows = pool_operands(k, s, H, W, C, with_pos)
    relu = np.maximum(x.astype(np.float64), 0)
    pooled = cct_oracle.maxpool_same(relu, k, s).reshape(2, -1, C)
    t = F.max_pool2d(F.pad(torch.from_numpy(relu).permute(0, 3, 1, 2), _same_pads(H, W, k, s), value=-math.inf), k, s)
    np.testing.assert_array_equal(pooled, t.permute(0, 2, 3, 1).reshape(2, -1, C).numpy())
    want = np.zeros((2, rows, C))
    want[:, :pooled.shape[1]] = pooled + (0 if pos is None else pos)
    np.testing.assert_array_equal(maxpool_relu_ref(x, k, s, pos, rows, np.float64), want)


def _same_pads(H, W, k, s):
    oh, ow = -(-H // s), -(-W // s)
    ph, pw = max((oh - 1) * s + k - H, 0), max((ow - 1) * s + k - W, 0)
    return (pw // 2, pw - pw // 2, ph // 2, ph - ph // 2)


@pytest.mark.parametrize("n,D,kind", SEQ_CASES)
def test_seq_pool_reference(n, D, kind):
    x, gamma, beta, pw, pb = seq_operands(n, D, kind)
    got = seq_pool_ref(x.astype(np.float64), gamma.astype(np.float64), beta.astype(np.float64), pw, pb)
    t = {k: torch.from_numpy(np.asarray(v, np.float64)) for k, v in dict(g=gamma, b=beta, pw=pw).items()}
    y = F.layer_norm(torch.from_numpy(x.astype(np.float64)), (D,), t["g"], t["b"], eps=1e-3)
    a = torch.softmax(y @ t["pw"][:, None] + pb, dim=1)
    np.testing.assert_allclose(got, (a * y).sum(1).numpy(), rtol=1e-10, atol=1e-10)

"""The boundary is a C ABI: tests/abi_client.c is compiled by gcc as strict C99 against include/vitb200.h (no C++, no
Python host code), linked to libvitb200.so, and
  * without a GPU it must stop at vb_create with the no-CPU-fallback error (CPU test),
  * on an H100 its logits (weights and image generated inside the C program) must match the oracle (GPU test)."""
import os
import subprocess
import zlib

import numpy as np
import pytest

import oracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIBDIR = os.path.join(ROOT, "vit_tensorflow_b200")


def _build_client(tmp_path, lib):
    exe = str(tmp_path / "abi_client")
    cmd = ["gcc", "-std=c99", "-Wall", "-Wextra", "-Werror", "-pedantic", "-I", os.path.join(ROOT, "include"),
           os.path.join(ROOT, "tests", "abi_client.c"), "-o", exe, "-L", LIBDIR, "-l:libvitb200.so", "-lm", f"-Wl,-rpath,{LIBDIR}"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return exe


def _has_gpu():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


def _fnv1a(name):
    h = 2166136261
    for ch in name.encode():
        h = ((h ^ ch) * 16777619) & 0xFFFFFFFF
    return h


def _hash_unit(seed, count):
    """abi_client.c: hash_unit() -- murmur3 finaliser on 32-bit integers"""
    x = (np.arange(count, dtype=np.uint64) * np.uint64(2654435761) + np.uint64(seed)) & np.uint64(0xFFFFFFFF)
    x ^= x >> np.uint64(16)
    x = (x * np.uint64(0x85ebca6b)) & np.uint64(0xFFFFFFFF)
    x ^= x >> np.uint64(13)
    x = (x * np.uint64(0xc2b2ae35)) & np.uint64(0xFFFFFFFF)
    x ^= x >> np.uint64(16)
    return x.astype(np.float64) / 4294967296.0 * 2.0 - 1.0


def _pattern(name, shape):
    """abi_client.c: pattern()"""
    v = _hash_unit(_fnv1a(name), int(np.prod(shape)))
    leaf = name.rsplit(".", 1)[-1]
    if leaf == "kernel" and len(shape) == 2:
        v = v * np.sqrt(6.0 / (shape[0] + shape[1]))
    elif leaf == "gamma":
        v = 1.0 + 0.2 * v
    elif leaf in ("bias", "beta"):
        v = 0.2 * v
    else:
        v = 1.7 * v
    return v.astype(np.float32).reshape(shape)


def _image():
    return (1.7 * _hash_unit(12345, 3 * 32 * 48 * 3)).astype(np.float32).reshape(3, 32, 48, 3)


@pytest.mark.skipif(_has_gpu(), reason="checks the no-GPU failure mode")
def test_c_client_compiles_as_c99_and_fails_loudly_without_gpu(lib, tmp_path):
    exe = _build_client(tmp_path, lib)
    r = subprocess.run([exe, str(tmp_path / "out.txt")], capture_output=True, text=True)
    assert r.returncode == 3, (r.returncode, r.stderr)
    assert "no CUDA device available" in r.stderr and "no CPU fallback" in r.stderr


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_c_client_matches_oracle(lib, tmp_path, precision):
    exe = _build_client(tmp_path, lib)
    out = tmp_path / "out.txt"
    r = subprocess.run([exe, str(out), precision], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    got = np.loadtxt(out).reshape(3, 7)
    cfg = oracle.make_config("vit", image_size=(32, 48), patch_size=(8, 16), num_classes=7, dim=64, depth=2, heads=2, mlp_dim=96,
                             dim_head=32)
    w = {name: _pattern(name, shape) for name, (shape, _) in oracle.weight_specs(cfg).items()}
    img = _image()
    ref = oracle.forward_numpy(img, w, cfg)
    if precision == "fp32":
        np.testing.assert_allclose(got, ref, rtol=1e-3, atol=1e-4)
    else:
        assert (np.abs(got - ref) <= 6e-2 + 4e-2 * np.abs(ref)).all()
    assert "kernel launches" in r.stdout and zlib.crc32(out.read_bytes()) != 0

"""Images per second of the RegionViT forward (bf16 engine) on two 224^2 ImageNet configurations, and RegionViT's stage-1
regional-to-local attention on its own.

    python tools/regionvit_bench.py [--batch 256] [--steps 20] [--warmup 5] [--out DIR]

  regionvit_readme  RegionViT(dim=(64, 128, 256, 512), depth=(2, 2, 8, 2), window_size=7, num_classes=1000)   (the README's)
  regionvit_s       RegionViT(dim=(96, 192, 384, 768), depth=(2, 2, 14, 2), window_size=7, num_classes=1000,
                              tokenize_local_3_conv=True)                                                  (RegionViT-S-like)

One JSON line per configuration: images/s over `steps` forwards on a CUDA stream (device-resident image and logits, so the
forward is captured into a CUDA graph and replayed, as a server calling forward_raw would run it), timed with CUDA events after
`warmup` untimed forwards; GFLOP per image computed from shapes (not measured); the per-kernel-class time split of one profiled
eager forward (vb_profile_read, events around every launch: a separate run); and the card name and power limit read in the same
run.  A last line times the stage-1 R2L attention shape (batch * 64 windows of 1 + 7 x 7 = 50 tokens, 4 heads of 32) through
vb_op_r2l_attention, on the R2L flash kernel and on the gather / materialised-scores / scatter path the engine takes off it.
Nothing is written to the tree; --out writes the lines to DIR/regionvit_bench.jsonl as well.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from cct_bench import card  # noqa: E402

CONFIGS = {
    "regionvit_readme": dict(dim=(64, 128, 256, 512), depth=(2, 2, 8, 2), window_size=7, num_classes=1000),
    "regionvit_s": dict(dim=(96, 192, 384, 768), depth=(2, 2, 14, 2), window_size=7, num_classes=1000, tokenize_local_3_conv=True),
}
IMAGE = 224
HEADS, INNER = 4, 128


def flops_per_image(m, image=IMAGE) -> dict:
    """2 * MACs at the model's shapes: the encoders, the Downsamples and PEGs, per layer the regional q|k|v, QK^T / PV and to_out,
    then over all tokens q|k|v, the R2L windows' QK^T / PV, to_out and the MLP, and the classifier.  LayerNorm, GELU, softmax and
    the mean are not counted."""
    from vit_tensorflow_b200.models import regionvit_maps
    d0 = m.dims[0]
    maps = regionvit_maps(image, image, m.local_patch_size, m.window_size)
    (lh, lw), (rh, rw) = maps[0]
    p = m.region_patch_size
    if m.tokenize_local_3_conv:
        h1 = -(-image // 2)
        local = 2.0 * h1 * h1 * 27 * d0 + 2 * 2.0 * lh * lw * 9 * d0 * d0
    else:
        local = 2.0 * lh * lw * 64 * 3 * d0
    parts = dict(encoders=local + 2.0 * rh * rw * 3 * p * p * d0, downsample=0.0, attention=0.0, gemm=0.0)
    for s, ((lh, lw), (rh, rw)) in enumerate(maps):
        d = m.dims[s]
        L, R = lh * lw, rh * rw
        if s:
            parts["downsample"] += 2.0 * (L + R) * 9 * m.dims[s - 1] * d + (2.0 * 9 * L * d if m.use_peg else 0.0)
        n = 1 + (lh // rh) * (lw // rw)
        per = 2.0 * R * d * 3 * INNER + 2.0 * R * INNER * d                          # regional q|k|v, to_out
        per += 2.0 * (L + R) * d * 3 * INNER + 2.0 * (L + R) * INNER * d + 2 * 2.0 * (L + R) * d * 4 * d
        parts["gemm"] += m.depths[s] * per
        parts["attention"] += m.depths[s] * (4.0 * R * R * INNER + 4.0 * R * n * n * INNER)
    head = 2.0 * m.dims[-1] * m.num_classes
    total = sum(parts.values()) + head
    return dict(gflop_per_image=total / 1e9, **{f"gflop_{k}": v / 1e9 for k, v in parts.items()})


def _forward_fn(m, batch):
    import torch
    from vit_tensorflow_b200 import _lib
    img = torch.randn(batch, IMAGE, IMAGE, 3, device="cuda")
    out = torch.empty(batch, m.num_classes, device="cuda")
    s = torch.cuda.Stream()
    torch.cuda.synchronize()

    def fwd():
        m.forward_raw(img.data_ptr(), _lib.MEM_DEVICE, batch, IMAGE, IMAGE, out.data_ptr(), _lib.MEM_DEVICE, s.cuda_stream)
    return fwd, s, out


def _profile(m, fwd):
    m.profile(True)                                  # one eager forward with events around every launch
    m.profile_read(reset=True)
    fwd()
    prof = m.profile_read(reset=True)
    m.profile(False)
    return prof


def run(name, batch, steps, warmup):
    import numpy as np
    import torch
    from vit_tensorflow_b200 import RegionViT
    kw = CONFIGS[name]
    m = RegionViT(**kw, precision="bf16", seed=0)
    fwd, s, out = _forward_fn(m, batch)
    for _ in range(warmup):
        fwd()
    s.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(s)
    for _ in range(steps):
        fwd()
    b.record(s)
    b.synchronize()
    ms = a.elapsed_time(b) / steps
    graphs = m.graph_stats()
    assert np.isfinite(out.cpu().numpy()).all()
    prof = _profile(m, fwd)
    f = flops_per_image(m)
    ips = batch / (ms / 1e3)
    return dict(config=name, model="RegionViT(" + ", ".join(f"{k}={v}" for k, v in kw.items()) + ")", image=IMAGE, precision="bf16",
                batch=batch, steps=steps, ms_per_forward=ms, images_per_s=ips, tflops_achieved=ips * f["gflop_per_image"] / 1e3,
                **f, graph_replays=graphs["replays"],
                profile_ms={k: round(v["ms"], 4) for k, v in prof.items() if v["launches"]},
                profile_launches={k: v["launches"] for k, v in prof.items() if v["launches"]})


def stage1_r2l_attention(batch, iters=20):
    """The stage-1 R2L attention at 224^2: a 56 x 56 local map over an 8 x 8 region map, batch * 64 windows of 7 x 7 local tokens
    plus their regional token, 4 heads of 32, fused q|k|v rows of pitch 384 as the engine packs them.  flash: vb_op_r2l_attention
    on the R2L flash kernel.  fallback: the same operands with one extra column (pitch 385, which the kernel's 16-byte loads
    refuse), so the op runs the path the engine takes off the kernel (window gather, materialised scores with the R2L bias,
    scatter); both must agree."""
    import numpy as np
    from vit_tensorflow_b200 import _lib
    lh = lw = 56
    rh = rw = 8
    ws, dh = 7, 32
    rng = np.random.default_rng(0)
    rows = batch * (lh * lw + rh * rw)
    qkv = rng.standard_normal((rows, 385)).astype(np.float32)
    table = rng.standard_normal(((2 * ws - 1) ** 2, HEADS)).astype(np.float32)
    _lib.last_attention_path()
    out, ms_flash = _lib.op_r2l_attention(np.ascontiguousarray(qkv[:, :384]), batch, lh, lw, rh, rw, HEADS, dh, table, ws, iters=iters)
    flash_path = _lib.last_attention_path()
    out_fb, ms_fallback = _lib.op_r2l_attention(qkv, batch, lh, lw, rh, rw, HEADS, dh, table, ws, iters=iters)
    fallback_path = _lib.last_attention_path()
    windows, n = batch * rh * rw, 1 + 49
    flops = 4.0 * windows * HEADS * n * n * dh
    return dict(config="stage1_r2l_attention", windows=windows, tokens_per_window=n, heads=HEADS, dim_head=dh,
                flash_ms=ms_flash, flash_path=flash_path, fallback_ms=ms_fallback, fallback_path=fallback_path,
                max_abs_diff=float(np.abs(out - out_fb).max()), speedup=ms_fallback / ms_flash,
                flash_tflops=flops / (ms_flash / 1e3) / 1e12)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--configs", default=",".join(CONFIGS))
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("tools/regionvit_bench.py measures on a CUDA device; none is visible")
    hw = card()
    lines = []
    for name in [c for c in args.configs.split(",") if c]:
        line = dict(run(name, args.batch, args.steps, args.warmup), **hw)
        print(json.dumps(line), flush=True)
        lines.append(line)
    line = dict(stage1_r2l_attention(args.batch), **hw)
    print(json.dumps(line), flush=True)
    lines.append(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "regionvit_bench.jsonl"), "a") as fh:
            for line in lines:
                fh.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()

"""Images per second of the NesT forward (bf16 engine) on two 224^2 ImageNet configurations, and NesT's level-0 block attention on
its own.

    python tools/nest_bench.py [--batch 256] [--steps 20] [--warmup 5] [--out DIR]

  nest_readme  NesT(image_size=224, patch_size=4, dim=96, heads=3, num_hierarchies=3, block_repeats=(2, 2, 8), num_classes=1000)
  nest_b       NesT(image_size=224, patch_size=4, dim=128, heads=4, num_hierarchies=3, block_repeats=(2, 2, 20), num_classes=1000)

One JSON line per configuration: images/s over `steps` forwards on a CUDA stream (device-resident image and logits, so the
forward is captured into a CUDA graph and replayed, as a server calling forward_raw would run it), timed with CUDA events after
`warmup` untimed forwards; GFLOP per image computed from shapes (not measured); the per-kernel-class time split of one profiled
eager forward (vb_profile_read, events around every launch: a separate run); and the card name and power limit read in the same
run.  A last line times the README model's level-0 attention shape (batch * 16 blocks of 14 x 14 = 196 tokens, 3 heads of 32)
through vb_op_block_attention, on the windowed flash kernel and on the materialised-scores path the engine takes off it.  Nothing is written to the tree; --out writes the lines to DIR/nest_bench.jsonl as well.
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
    "nest_readme": dict(image_size=224, patch_size=4, dim=96, heads=3, num_hierarchies=3, block_repeats=(2, 2, 8), num_classes=1000),
    "nest_b": dict(image_size=224, patch_size=4, dim=128, heads=4, num_hierarchies=3, block_repeats=(2, 2, 20), num_classes=1000),
}
IMAGE = 224


def flops_per_image(m, image=IMAGE) -> dict:
    """2 * MACs at the model's shapes: the patch embedding, per block q|k|v, QK^T and PV inside the blocks, to_out and the MLP, the
    aggregation convolutions and the classifier.  LayerNorm, softmax, the max-pool and the mean are not counted."""
    pl = m.plan
    p, dh, mult = pl["patch_size"], pl["dim"] // pl["heads"], m._nc.mlp_mult
    h = w = image // p
    total = 2.0 * h * w * p * p * 3 * pl["dim"]
    parts = dict(patch_embedding=total, attention=0.0, gemm=0.0, aggregate=0.0)
    n = len(pl["levels"])
    for i, lv in enumerate(pl["levels"]):
        d, inner, bs = lv["dim"], dh * lv["heads"], 2 ** (n - 1 - i)
        tokens, block = h * w, (h // bs) * (w // bs)
        per = 2.0 * tokens * d * 3 * inner + 2.0 * tokens * inner * d + 2 * 2.0 * tokens * d * mult * d
        parts["gemm"] += lv["depth"] * per
        parts["attention"] += lv["depth"] * 4.0 * tokens * block * inner
        if lv["aggregate"]:
            parts["aggregate"] += 2.0 * tokens * 9 * d * 2 * d
            h, w = -(-h // 2), -(-w // 2)
    head = 2.0 * pl["last_dim"] * m.num_classes
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
    from vit_tensorflow_b200 import NesT
    kw = CONFIGS[name]
    m = NesT(**kw, precision="bf16", seed=0)
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
    return dict(config=name, model="NesT(" + ", ".join(f"{k}={v}" for k, v in kw.items()) + ")", image=IMAGE, precision="bf16",
                batch=batch, steps=steps, ms_per_forward=ms, images_per_s=ips, tflops_achieved=ips * f["gflop_per_image"] / 1e3,
                **f, graph_replays=graphs["replays"],
                profile_ms={k: round(v["ms"], 4) for k, v in prof.items() if v["launches"]},
                profile_launches={k: v["launches"] for k, v in prof.items() if v["launches"]})


def level0_attention(batch, iters=20):
    """The README model's level-0 attention: batch * 16 blocks of 14 x 14 tokens on a 56 x 56 map, 3 heads of 32, fused q|k|v rows
    (pitch 320: 288 rounded up to 64, as the engine packs them).  flash: vb_op_block_attention on the windowed flash kernel.
    fallback: the same operands with one extra column (pitch 289, which the flash kernel's 16-byte loads refuse), so the op runs the
    path the engine takes off the flash kernel (row permutation, materialised scores, permutation back); both must agree."""
    import numpy as np
    from vit_tensorflow_b200 import _lib
    H = W = 56
    heads, dh = 3, 32
    rng = np.random.default_rng(0)
    qkv = rng.standard_normal((batch * H * W, 320)).astype(np.float32)
    _lib.last_attention_path()
    out, ms_flash = _lib.op_block_attention(qkv, H, W, 14, 14, heads, dh, iters=iters)
    flash_path = _lib.last_attention_path()
    out_fb, ms_fallback = _lib.op_block_attention(np.ascontiguousarray(qkv[:, :289]), H, W, 14, 14, heads, dh, iters=iters)
    fallback_path = _lib.last_attention_path()
    blocks = batch * 16
    flops = 4.0 * blocks * heads * 196 * 196 * dh
    return dict(config="level0_attention", blocks=blocks, tokens_per_block=196, heads=heads, dim_head=dh,
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
        raise SystemExit("tools/nest_bench.py measures on a CUDA device; none is visible")
    hw = card()
    lines = []
    for name in [c for c in args.configs.split(",") if c]:
        line = dict(run(name, args.batch, args.steps, args.warmup), **hw)
        print(json.dumps(line), flush=True)
        lines.append(line)
    line = dict(level0_attention(args.batch), **hw)
    print(json.dumps(line), flush=True)
    lines.append(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "nest_bench.jsonl"), "a") as fh:
            for line in lines:
                fh.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()

"""Images per second of the LeViT forward (bf16 engine) on two 224^2 ImageNet configurations.

    python tools/levit_bench.py [--batch 256] [--steps 20] [--warmup 5] [--out DIR]

  levit_readme  LeViT(image_size=224, dim=(256, 384, 512), depth=4, heads=(4, 6, 8), mlp_mult=2)   the reference README's model
  levit_128s    LeViT(image_size=224, dim=(128, 256, 384), depth=(2, 3, 4), heads=(4, 6, 8), mlp_mult=2, dim_key=16,
                dim_value=32)                                                                      shaped like the paper's LeViT-128S

One JSON line per configuration: images/s over `steps` forwards on a CUDA stream (device-resident image and logits, so the
forward is captured into a CUDA graph and replayed, as a server calling forward_raw would run it), timed with CUDA events after
`warmup` untimed forwards; algorithmic GFLOP per image computed from the model's true shapes (not the zero-padded head widths the
engine runs; not measured); the per-kernel-class time split of one profiled forward (vb_profile_read, events around every launch:
a separate eager run); and the card name and power limit read in the same run.  Nothing is written to the tree; --out writes the
lines to DIR/levit_bench.jsonl as well.
"""
from __future__ import annotations

import argparse
import json
import math
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from cct_bench import card  # noqa: E402

CONFIGS = {
    "levit_readme": dict(image_size=224, num_classes=1000, dim=(256, 384, 512), depth=4, heads=(4, 6, 8), mlp_mult=2, stages=3),
    "levit_128s": dict(image_size=224, num_classes=1000, dim=(128, 256, 384), depth=(2, 3, 4), heads=(4, 6, 8), mlp_mult=2, stages=3,
                       dim_key=16, dim_value=32),
}


def flops_per_image(m) -> dict:
    """2 * MACs of every matmul at the model's shapes: the stem convolutions (as GEMMs of the im2col rows), per block the q / k / v
    projections, QK^T, PV, to_out and the MLP, and the classifier.  BatchNorm (folded), softmax and pooling are not counted."""
    h, cin, stem = m.image_size, 3, []
    for cout in (32, 64, 128, m.dims[0]):
        h = -(-h // 2)
        stem.append(2.0 * h * h * 9 * cin * cout)
        cin = cout
    total, fmap, dk, dv = sum(stem), m.image_size // 16, m.dim_key, m.dim_value
    for ind in range(m.stages):
        plan = [(m.dims[ind], m.dims[ind], m.layer_heads[ind], m.mlp_mult, 1)] * m.depths[ind]
        if ind != m.stages - 1:
            plan.append((m.dims[ind], m.dims[ind + 1], 2 * m.layer_heads[ind], 2, 2))
        for d, dout, hh, mult, step in plan:
            nk, nq = fmap * fmap, math.ceil(fmap / step) ** 2
            total += 2.0 * (nq * d * hh * dk + nk * d * hh * (dk + dv) + nq * nk * hh * (dk + dv) + nq * hh * dv * dout
                            + 2 * nq * dout * dout * mult)
            if step == 2:
                fmap = math.ceil(fmap / 2)
    total += 2.0 * m.dims[-1] * m.num_classes
    return dict(gflop_per_image=total / 1e9, stem_gflop_per_image=sum(stem) / 1e9)


def run(name, batch, steps, warmup):
    import numpy as np
    import torch
    from vit_tensorflow_b200 import LeViT, _lib
    kw = CONFIGS[name]
    m = LeViT(**kw, precision="bf16", seed=0)
    img = torch.randn(batch, m.image_size, m.image_size, 3, device="cuda")
    out = torch.empty(batch, m.num_classes, device="cuda")
    s = torch.cuda.Stream()
    torch.cuda.synchronize()

    def fwd():
        m.forward_raw(img.data_ptr(), _lib.MEM_DEVICE, batch, m.image_size, m.image_size, out.data_ptr(), _lib.MEM_DEVICE, s.cuda_stream)

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
    m.profile(True)                                  # one eager forward with events around every launch
    m.profile_read(reset=True)
    fwd()
    prof = m.profile_read(reset=True)
    m.profile(False)
    f = flops_per_image(m)
    ips = batch / (ms / 1e3)
    return dict(config=name, model="LeViT(" + ", ".join(f"{k}={v}" for k, v in kw.items()) + ")", precision="bf16",
                batch=batch, steps=steps, ms_per_forward=ms, images_per_s=ips, tflops_achieved=ips * f["gflop_per_image"] / 1e3,
                **f, graph_replays=graphs["replays"],
                profile_ms={k: round(v["ms"], 4) for k, v in prof.items() if v["launches"]},
                profile_launches={k: v["launches"] for k, v in prof.items() if v["launches"]})


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
        raise SystemExit("tools/levit_bench.py measures on a CUDA device; none is visible")
    hw = card()
    lines = []
    for name in args.configs.split(","):
        line = dict(run(name, args.batch, args.steps, args.warmup), **hw)
        print(json.dumps(line), flush=True)
        lines.append(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "levit_bench.jsonl"), "a") as fh:
            for line in lines:
                fh.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()

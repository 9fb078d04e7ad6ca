"""Images per second of the MPP call (bf16 engine), against the plain ViT forward of the same encoder.

    python tools/mpp_bench.py [--batch 256] [--steps 20] [--warmup 5] [--out DIR]

  mpp_b16         MPP on ViT-B/16 at 224^2 (dim 768, depth 12, 12 heads of 64, mlp 3072), patch 16, the defaults (3 bits: 512
                  classes; mask 0.15, replace 0.5, random patch 0.5): the encoder over all 197 rows, to_bits on the 30 masked
  vit_b16         the plain ViT-B/16 forward of that encoder
  mpp_usage       mpp.py's usage block: ViT(256, 32, dim 1024, depth 6, heads 8, mlp 2048), mask 0.15, random patch 0.30,
                  replace 0.50
  vit_usage       the plain forward of that encoder

One JSON line per configuration: images/s over `steps` calls on a CUDA stream (device-resident image and loss, so the call is
captured into a CUDA graph and replayed), timed with CUDA events after `warmup` untimed calls; the per-kernel-class time split of
one profiled eager call (a separate run); and the card name and power limit read in the same run.  Nothing is written to the
tree; --out writes the lines to DIR/mpp_bench.jsonl as well.
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

B16 = dict(image_size=224, patch_size=16, num_classes=1000, dim=768, depth=12, heads=12, mlp_dim=3072)
README = dict(image_size=256, patch_size=32, num_classes=1000, dim=1024, depth=6, heads=8, mlp_dim=2048)
CONFIGS = {
    "mpp_b16": ("mpp", B16, {}),
    "vit_b16": ("vit", B16, {}),
    "mpp_usage": ("mpp", README, dict(mask_prob=0.15, random_patch_prob=0.30, replace_prob=0.50)),
    "vit_usage": ("vit", README, {}),
}


def run(name, batch, steps, warmup):
    import numpy as np
    import torch
    from vit_tensorflow_b200 import MPP, ViT, _lib
    kind, enc_kw, kw = CONFIGS[name]
    enc = ViT(**enc_kw, precision="bf16", seed=0)
    size = enc_kw["image_size"]
    m = enc if kind == "vit" else MPP(image_size=size, transformer=enc, patch_size=enc_kw["patch_size"], seed=1, **kw)
    img = torch.randn(batch, size, size, 3, device="cuda")
    out = torch.empty(batch if kind == "vit" else 1, 1000 if kind == "vit" else 1, device="cuda")
    s = torch.cuda.Stream()
    torch.cuda.synchronize()

    def fwd():                                            # logits (ViT) or the loss (MPP) in device memory
        m.forward_raw(img.data_ptr(), _lib.MEM_DEVICE, batch, size, size, out.data_ptr(), _lib.MEM_DEVICE, s.cuda_stream)
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
    m.profile(True)
    m.profile_read(reset=True)
    fwd()
    prof = m.profile_read(reset=True)
    m.profile(False)
    return dict(config=name, precision="bf16", batch=batch, steps=steps, ms_per_call=ms, images_per_s=batch / (ms / 1e3),
                graph_replays=graphs["replays"], profile_ms={k: round(v["ms"], 4) for k, v in prof.items() if v["launches"]},
                profile_launches={k: v["launches"] for k, v in prof.items() if v["launches"]})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("tools/mpp_bench.py measures on a CUDA device; none is visible")
    hw = card()
    lines = []
    for name in CONFIGS:
        line = dict(run(name, args.batch, args.steps, args.warmup), **hw)
        print(json.dumps(line), flush=True)
        lines.append(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "mpp_bench.jsonl"), "a") as fh:
            for line in lines:
                fh.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()

"""Images per second of the small-dataset ViT forward (bf16 engine) against a plain ViT of the same dimensions.

    python tools/small_vit_bench.py [--batch 256] [--steps 20] [--warmup 5] [--out DIR]

  sdvit_readme  vit_for_small_dataset.ViT(image_size=256, patch_size=16, num_classes=1000, dim=1024, depth=6, heads=16,
                                          mlp_dim=2048)   (the reference README's; 257 keys: the streaming flash kernel)
  sdvit_cifar   image_size=32, patch_size=4, num_classes=1000, dim=192, depth=9, heads=12, mlp_dim=384   (65 keys: the resident
                flash kernel)
  vit_readme / vit_cifar   vit.ViT with the same dimensions

One JSON line per model: images/s over `steps` forwards on a CUDA stream (device-resident image and logits, so the forward is
captured into a CUDA graph and replayed), timed with CUDA events after `warmup` untimed forwards; the per-kernel-class time
split of one profiled eager forward (a separate run: the SPT kernel is in "im2col", its LayerNorm statistics in "layernorm");
and the card name and power limit read in the same run.  Nothing is written to the tree; --out writes the lines to
DIR/small_vit_bench.jsonl as well.
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

MODELS = {
    "readme": dict(image_size=256, patch_size=16, num_classes=1000, dim=1024, depth=6, heads=16, mlp_dim=2048),
    "cifar": dict(image_size=32, patch_size=4, num_classes=1000, dim=192, depth=9, heads=12, mlp_dim=384),
}


def run(name, batch, steps, warmup):
    import numpy as np
    import torch
    from vit_tensorflow_b200 import SmallDatasetViT, ViT, _lib
    family, size = name.split("_")
    kw = MODELS[size]
    m = (SmallDatasetViT if family == "sdvit" else ViT)(**kw, precision="bf16", seed=0)
    s_img = kw["image_size"]
    img = torch.randn(batch, s_img, s_img, 3, device="cuda")
    out = torch.empty(batch, kw["num_classes"], device="cuda")
    s = torch.cuda.Stream()
    torch.cuda.synchronize()

    def fwd():
        m.forward_raw(img.data_ptr(), _lib.MEM_DEVICE, batch, s_img, s_img, out.data_ptr(), _lib.MEM_DEVICE, s.cuda_stream)
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
    total = sum(v["ms"] for v in prof.values())
    return dict(config=name, precision="bf16", batch=batch, steps=steps, ms_per_forward=ms, images_per_s=batch / (ms / 1e3),
                graph_replays=graphs["replays"], profile_ms={k: round(v["ms"], 4) for k, v in prof.items() if v["launches"]},
                profile_share={k: round(v["ms"] / total, 4) for k, v in prof.items() if v["launches"]},
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
        raise SystemExit("tools/small_vit_bench.py measures on a CUDA device; none is visible")
    hw = card()
    lines = []
    for name in ("sdvit_readme", "vit_readme", "sdvit_cifar", "vit_cifar"):
        line = dict(run(name, args.batch, args.steps, args.warmup), **hw)
        print(json.dumps(line), flush=True)
        lines.append(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "small_vit_bench.jsonl"), "a") as fh:
            for line in lines:
                fh.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()

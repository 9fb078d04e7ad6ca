"""Images per second of the ATS-ViT forward (bf16 engine) on the README model, against a plain ViT of the same dimensions.

    python tools/ats_vit_bench.py [--batch 256] [--steps 20] [--warmup 5] [--out DIR]

  ats_readme  ats_vit.ViT(image_size=256, patch_size=16, num_classes=1000, dim=1024, depth=6,
                          max_tokens_per_depth=(256, 128, 64, 32, 16, 8), heads=16, mlp_dim=2048)   (the README's)
  vit_same    vit.ViT with the same dimensions: every layer carries all 257 rows

One JSON line per model: images/s over `steps` forwards on a CUDA stream (device-resident image and logits, so the forward is
captured into a CUDA graph and replayed), timed with CUDA events after `warmup` untimed forwards; the per-kernel-class time
split of one profiled eager forward (a separate run); and the card name and power limit read in the same run.  The ATS rows
per layer are 257, 257, 129, 65, 33, 17 at most (layer 0 never samples: 256 tokens, K = 256).  Nothing is written to the tree;
--out writes the lines to DIR/ats_vit_bench.jsonl as well.
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

KW = dict(image_size=256, patch_size=16, num_classes=1000, dim=1024, depth=6, heads=16, mlp_dim=2048)
TOKENS = (256, 128, 64, 32, 16, 8)


def run(name, batch, steps, warmup):
    import numpy as np
    import torch
    from vit_tensorflow_b200 import ATSViT, ViT, _lib
    m = ATSViT(**KW, max_tokens_per_depth=TOKENS, precision="bf16", seed=0) if name == "ats_readme" else ViT(**KW, precision="bf16", seed=0)
    img = torch.randn(batch, 256, 256, 3, device="cuda")
    out = torch.empty(batch, 1000, device="cuda")
    s = torch.cuda.Stream()
    torch.cuda.synchronize()

    def fwd():
        m.forward_raw(img.data_ptr(), _lib.MEM_DEVICE, batch, 256, 256, out.data_ptr(), _lib.MEM_DEVICE, s.cuda_stream)
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
    return dict(config=name, precision="bf16", batch=batch, steps=steps, ms_per_forward=ms, images_per_s=batch / (ms / 1e3),
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
        raise SystemExit("tools/ats_vit_bench.py measures on a CUDA device; none is visible")
    hw = card()
    lines = []
    for name in ("ats_readme", "vit_same"):
        line = dict(run(name, args.batch, args.steps, args.warmup), **hw)
        print(json.dumps(line), flush=True)
        lines.append(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "ats_vit_bench.jsonl"), "a") as fh:
            for line in lines:
                fh.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()

"""Images per second of the MAE and SimMIM calls (bf16 engine), against the plain ViT forward of the same encoder.

    python tools/mim_bench.py [--batch 256] [--steps 20] [--warmup 5] [--out DIR]

  mae_b16         MAE on ViT-B/16 at 224^2 (dim 768, depth 12, 12 heads of 64, mlp 3072), decoder 512 x 8 with 16 heads of 32,
                  masking_ratio 0.75: the encoder runs on 49 of the 196 patches, the decoder on all 196
  vit_b16         the plain ViT-B/16 forward of that encoder (197 rows per layer)
  mae_readme      the README's MAE (README.md:685-735): encoder ViT(256, 32, dim 1024, depth 6, heads 8, mlp 2048), decoder 512 x 6
  simmim_readme   the README's SimMIM (README.md:745-775) over the same encoder, masking_ratio 0.5
  vit_readme      the plain forward of that encoder

One JSON line per configuration: images/s over `steps` calls on a CUDA stream (device-resident image and loss, so the call is
captured into a CUDA graph and replayed), timed with CUDA events after `warmup` untimed calls; the per-kernel-class time split of
one profiled eager call (a separate run); and the card name and power limit read in the same run.  Nothing is written to the
tree; --out writes the lines to DIR/mim_bench.jsonl as well.
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
    "mae_b16": ("mae", B16, dict(decoder_dim=512, decoder_depth=8, decoder_heads=16, decoder_dim_head=32, masking_ratio=0.75)),
    "vit_b16": ("vit", B16, {}),
    "mae_readme": ("mae", README, dict(decoder_dim=512, decoder_depth=6, masking_ratio=0.75)),
    "simmim_readme": ("simmim", README, dict(masking_ratio=0.5)),
    "vit_readme": ("vit", README, {}),
}


def run(name, batch, steps, warmup):
    import numpy as np
    import torch
    from vit_tensorflow_b200 import MAE, SimMIM, ViT, _lib
    kind, enc_kw, kw = CONFIGS[name]
    enc = ViT(**enc_kw, precision="bf16", seed=0)
    size = enc_kw["image_size"]
    m = enc if kind == "vit" else (MAE if kind == "mae" else SimMIM)(image_size=size, encoder=enc, seed=1, **kw)
    img = torch.randn(batch, size, size, 3, device="cuda")
    out = torch.empty(batch if kind == "vit" else 1, 1000 if kind == "vit" else 1, device="cuda")
    s = torch.cuda.Stream()
    torch.cuda.synchronize()

    def fwd():                                            # logits (ViT) or the loss (MAE / SimMIM) in device memory
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
        raise SystemExit("tools/mim_bench.py measures on a CUDA device; none is visible")
    hw = card()
    lines = []
    for name in CONFIGS:
        line = dict(run(name, args.batch, args.steps, args.warmup), **hw)
        print(json.dumps(line), flush=True)
        lines.append(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "mim_bench.jsonl"), "a") as fh:
            for line in lines:
                fh.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()

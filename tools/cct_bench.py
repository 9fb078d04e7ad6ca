"""Images per second of the CCT forward (bf16 engine) on the two configurations of the CCT paper.

    python tools/cct_bench.py [--batch 256] [--steps 20] [--warmup 5] [--out DIR]

  cct_14_7x2  cct_14(img_size=224, kernel_size=7, n_conv_layers=2)              ImageNet model: 196 tokens, dim 384
  cct_7_3x1   cct_7(img_size=32, kernel_size=3, n_conv_layers=1, num_classes=10)  CIFAR model: 256 tokens, dim 256

One JSON line per configuration: images/s over `steps` forwards on a CUDA stream (device-resident image and logits, so the
forward is captured into a CUDA graph and replayed, as a server calling forward_raw would run it), timed with CUDA events after
`warmup` untimed forwards; algorithmic GFLOP per image computed from the shapes (not measured); the per-kernel-class time split
of one profiled forward (vb_profile_read, events around every launch: a separate eager run); and the card name and power limit
read in the same run.  Nothing is written to the tree; --out writes the lines to DIR/cct_bench.jsonl as well.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CONFIGS = {
    "cct_14_7x2": ("cct_14", dict(img_size=224, kernel_size=7, n_conv_layers=2)),
    "cct_7_3x1": ("cct_7", dict(img_size=32, kernel_size=3, n_conv_layers=1, num_classes=10)),
}


def flops_per_image(m) -> dict:
    """2 * MACs of every matmul at the true shapes: the convolutions (as GEMMs of the im2col rows), the encoder layers, the
    sequence pooling and the classifier.  Max-pool, LayerNorm and softmax are not counted."""
    c = m._cfg
    h, w, cin, conv = c.image_h, c.image_w, 3, []
    for i in range(c.cct_conv_layers):
        h, w = -(-h // c.cct_stride), -(-w // c.cct_stride)
        cout = c.dim if i == c.cct_conv_layers - 1 else 64
        conv.append(2.0 * h * w * c.cct_kernel * c.cct_kernel * cin * cout)
        h, w = -(-h // c.cct_pool_stride), -(-w // c.cct_pool_stride)
        cin = cout
    n, d = m.sequence_length, c.dim
    layer = 2.0 * n * d * 3 * d + 4.0 * n * n * d + 2.0 * n * d * d + 4.0 * n * d * c.mlp_dim
    total = sum(conv) + c.depth * layer + 2.0 * n * d + 2.0 * d * c.num_classes
    return dict(gflop_per_image=total / 1e9, conv_gflop_per_image=[f / 1e9 for f in conv], tokens=n)


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=30)
        limit, sm_max = (float(v) for v in r.stdout.strip().split(","))
    except Exception:
        limit = sm_max = None
    return dict(gpu=name, power_limit_w=limit, sm_max_mhz=sm_max)


def run(name, batch, steps, warmup):
    import numpy as np
    import torch
    import vit_tensorflow_b200 as vb
    from vit_tensorflow_b200 import _lib
    factory, kw = CONFIGS[name]
    m = getattr(vb, factory)(**kw, precision="bf16", seed=0)
    c = m._cfg
    img = torch.randn(batch, c.image_h, c.image_w, 3, device="cuda")
    out = torch.empty(batch, c.num_classes, device="cuda")
    s = torch.cuda.Stream()
    torch.cuda.synchronize()

    def fwd():
        m.forward_raw(img.data_ptr(), _lib.MEM_DEVICE, batch, c.image_h, c.image_w, out.data_ptr(), _lib.MEM_DEVICE, s.cuda_stream)

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
    return dict(config=name, factory=f"{factory}(" + ", ".join(f"{k}={v}" for k, v in kw.items()) + ")", precision="bf16",
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
        raise SystemExit("tools/cct_bench.py measures on a CUDA device; none is visible")
    hw = card()
    lines = []
    for name in args.configs.split(","):
        line = dict(run(name, args.batch, args.steps, args.warmup), **hw)
        print(json.dumps(line), flush=True)
        lines.append(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "cct_bench.jsonl"), "a") as fh:
            for line in lines:
                fh.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()

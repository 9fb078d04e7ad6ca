"""Images per second of the MobileViT forward (bf16 engine) on three 256^2 ImageNet configurations.

    python tools/mobilevit_bench.py [--batch 256] [--steps 20] [--warmup 5] [--out DIR]

  mobilevit_xs   MobileViT(dims=(96, 120, 144), channels=(16, 32, 48, 48, 64, 64, 80, 80, 96, 96, 384))   the reference's usage block
  mobilevit_xxs  dims=(64, 80, 96), channels=(16, 16, 24, 24, 48, 48, 64, 64, 80, 80, 320), expansion=2     the paper's XXS widths
  mobilevit_s    dims=(144, 192, 240), channels=(16, 32, 64, 64, 96, 96, 128, 128, 160, 160, 640)          the paper's S widths

One JSON line per configuration: images/s and ms per forward over `steps` forwards on a CUDA stream (device-resident image and
logits, so the forward is captured into a CUDA graph and replayed), timed with CUDA events after `warmup` untimed forwards;
algorithmic GFLOP per image computed from the model's true shapes (not the zero-padded widths and heads the engine runs; not
measured); from a separate profiled eager forward (vb_profile_read, events around every launch): the MV2 depthwise kernel's time
and its bytes/s against the H100 SXM's 3.35 TB/s (in this model's bf16 forward the profile's "other" class holds that kernel
alone), the attention's share of the forward and the per-class split; and the card name and power limit read in the same run.
Nothing is written to the tree; --out writes the lines to DIR/mobilevit_bench.jsonl as well.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

from cct_bench import card  # noqa: E402
import mobilevit_oracle as mo  # noqa: E402

CONFIGS = mo.BENCH
HBM_TBPS = 3.35


def flops_per_image(cfg) -> dict:
    """2 * MACs of every convolution and matmul at the model's shapes (Conv2D as im2col GEMMs, depthwise 9 MACs per output, the
    attention's QK^T and PV per patch-position group, to_qkv / to_out / MLP, the head).  BatchNorm (folded), SiLU, softmax and the
    pooling are not counted."""
    ch, k = cfg["channels"], cfg["kernel_size"]
    h, w = (-(-s // 2) for s in cfg["image_size"])
    total = attn = dw = 0.0
    total += 2.0 * h * w * 27 * ch[0]
    blocks = mo.blocks(cfg)
    ph, pw = cfg["patch_size"]

    def mv2(h, w, b):
        nonlocal total, dw
        _, cin, hid, cout, stride, expand, _ = b
        if expand:
            total += 2.0 * h * w * cin * hid
        h, w = -(-h // stride), -(-w // stride)
        dw += 2.0 * h * w * 9 * hid
        total += 2.0 * h * w * hid * cout
        return h, w
    for b in blocks[:4]:
        h, w = mv2(h, w, b)
    for s in range(3):
        h, w = mv2(h, w, blocks[4 + s])
        d, c, cin, n = cfg["dims"][s], ch[5 + 2 * s], ch[4 + 2 * s], h * w
        mlp = int(d * (2, 4, 4)[s])
        total += 2.0 * n * (k * k * cin * c + c * d + d * c + k * k * (c + cin) * c)
        for _ in range(cfg["depths"][s]):
            total += 2.0 * n * (d * 96 + 32 * d + 2 * d * mlp)
            attn += 2.0 * 2 * n * (n // (ph * pw)) * 32
    total += 2.0 * h * w * ch[9] * ch[-1] + 2.0 * ch[-1] * cfg["num_classes"]
    total += attn + dw
    return dict(gflop_per_image=total / 1e9, attention_gflop_per_image=attn / 1e9, depthwise_gflop_per_image=dw / 1e9)


def run(name, batch, steps, warmup):
    import numpy as np
    import torch
    from vit_tensorflow_b200 import from_config, _lib
    cfg = mo.make_config(**CONFIGS[name])
    m = from_config(cfg, precision="bf16", seed=0)
    ih, iw = cfg["image_size"]
    img = torch.randn(batch, ih, iw, 3, device="cuda")
    out = torch.empty(batch, m.num_classes, device="cuda")
    s = torch.cuda.Stream()
    torch.cuda.synchronize()

    def fwd():
        m.forward_raw(img.data_ptr(), _lib.MEM_DEVICE, batch, ih, iw, out.data_ptr(), _lib.MEM_DEVICE, s.cuda_stream)

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
    f = flops_per_image(cfg)
    ips = batch / (ms / 1e3)
    prof_total = sum(v["ms"] for v in prof.values())
    dwp = prof["other"]
    return dict(config=name, model="MobileViT(" + ", ".join(f"{k}={v}" for k, v in CONFIGS[name].items()) + ")", precision="bf16",
                batch=batch, steps=steps, ms_per_forward=ms, images_per_s=ips, tflops_achieved=ips * f["gflop_per_image"] / 1e3, **f,
                graph_replays=graphs["replays"],
                depthwise_ms=dwp["ms"], depthwise_launches=dwp["launches"],
                depthwise_tb_per_s=dwp["bytes"] / (dwp["ms"] / 1e3) / 1e12 if dwp["ms"] else None,
                depthwise_share_of_hbm=dwp["bytes"] / (dwp["ms"] / 1e3) / 1e12 / HBM_TBPS if dwp["ms"] else None,
                attention_share_of_profiled_forward=prof["attention"]["ms"] / prof_total if prof_total else None,
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
        raise SystemExit("tools/mobilevit_bench.py measures on a CUDA device; none is visible")
    hw = card()
    lines = []
    for name in args.configs.split(","):
        line = dict(run(name, args.batch, args.steps, args.warmup), **hw)
        print(json.dumps(line), flush=True)
        lines.append(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "mobilevit_bench.jsonl"), "a") as fh:
            for line in lines:
                fh.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()

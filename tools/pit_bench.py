"""Images per second of the PiT forward (bf16 engine) at 224^2, on two models.

    python tools/pit_bench.py [--batch 256] [--steps 20] [--warmup 5] [--out DIR]

  pit_readme                PiT(image_size=224, patch_size=14, dim=256, num_classes=1000, depth=(3, 3, 3), heads=16, mlp_dim=2048)
                            the reference's usage block (dropout 0): 31 x 31 patches at stride 7, n = 962 tokens
  pit_readme_heads_4_8_16   the same with heads=(4, 8, 16): 4, 8 and 16 heads of 64 in the three stages

One JSON line per model: images/s and ms per forward over `steps` forwards on a CUDA stream (device-resident image and logits, so
the forward is captured into a CUDA graph and replayed), timed with CUDA events after `warmup` untimed forwards; algorithmic GFLOP
per image computed from the model's shapes (not measured), split into its parts; from a separate profiled eager forward
(vb_profile_read, events around every launch) the time per kernel class and its share of the profiled forward: attention, the GEMM
classes (plain: to_qkv; GELU epilogue: fc1; residual epilogue: patch embedding, to_out, fc2), im2col (the patch unfold) and
LayerNorm; and the card name and power limit read in the same run.  Nothing is written to the tree; --out writes the lines to
DIR/pit_bench.jsonl as well.
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
import pit_oracle as po  # noqa: E402

CONFIGS = po.BENCH


def flops_per_image(cfg) -> dict:
    """2 * MACs of every matmul at the model's shapes, by part: the patch embedding, to_qkv, attention (QK^T and PV), to_out, the
    MLPs and the head.  LayerNorm, GELU and softmax are not counted."""
    n_p = po.num_patches(cfg)
    n, d, dh, mlp = n_p + 1, cfg["dim"], cfg["dim_head"], cfg["mlp_dim"]
    parts = dict(patch=2.0 * n_p * cfg["patch_size"] ** 2 * 3 * d, qkv=0.0, attention=0.0, out=0.0, mlp=0.0,
                 head=2.0 * d * cfg["num_classes"])
    for _, _, heads, project_out in po.layer_plan(cfg):
        inner = heads * dh
        parts["qkv"] += 2.0 * n * d * 3 * inner
        parts["attention"] += 2.0 * 2 * heads * n * n * dh
        parts["out"] += 2.0 * n * inner * d if project_out else 0.0
        parts["mlp"] += 2.0 * 2 * n * d * mlp
    out = {f"{k}_gflop_per_image": v / 1e9 for k, v in parts.items()}
    out["gflop_per_image"] = sum(parts.values()) / 1e9
    return out


def run(name, batch, steps, warmup):
    import numpy as np
    import torch
    from vit_tensorflow_b200 import from_config, _lib
    cfg = po.make_config(**CONFIGS[name])
    m = from_config(cfg, precision="bf16", seed=0)
    side = cfg["image_size"]
    img = torch.randn(batch, side, side, 3, device="cuda")
    out = torch.empty(batch, m.num_classes, device="cuda")
    s = torch.cuda.Stream()
    torch.cuda.synchronize()

    def fwd():
        m.forward_raw(img.data_ptr(), _lib.MEM_DEVICE, batch, side, side, out.data_ptr(), _lib.MEM_DEVICE, s.cuda_stream)

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
    total = sum(v["ms"] for v in prof.values())
    return dict(config=name, model="PiT(" + ", ".join(f"{k}={v}" for k, v in CONFIGS[name].items()) + ")", precision="bf16",
                batch=batch, steps=steps, ms_per_forward=ms, images_per_s=ips, tflops_achieved=ips * f["gflop_per_image"] / 1e3, **f,
                graph_replays=graphs["replays"], profiled_forward_ms=total,
                profile_ms={k: round(v["ms"], 4) for k, v in prof.items() if v["launches"]},
                profile_share={k: round(v["ms"] / total, 4) for k, v in prof.items() if v["launches"]} if total else None,
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
        raise SystemExit("tools/pit_bench.py measures on a CUDA device; none is visible")
    hw = card()
    lines = []
    for name in args.configs.split(","):
        line = dict(run(name, args.batch, args.steps, args.warmup), **hw)
        print(json.dumps(line), flush=True)
        lines.append(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "pit_bench.jsonl"), "a") as fh:
            for line in lines:
                fh.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()

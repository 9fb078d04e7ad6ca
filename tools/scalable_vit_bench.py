"""Images per second of the ScalableViT forward (bf16 engine) at 256^2, on two models.

    python tools/scalable_vit_bench.py [--batch 256] [--steps 20] [--warmup 5] [--out DIR]

  scalable_vit_readme  ScalableViT(num_classes=1000, dim=64, heads=(2, 4, 8, 16), depth=(2, 2, 20, 2), ssa_dim_key=(40, 40, 40, 32),
                       reduction_factor=(8, 4, 2, 1), window_size=(64, 32, None, None))    the reference's usage block: stages 1-2
                       attend within one 4,096- / 1,024-token window
  scalable_vit_win8    the same with window_size=(8, 8, None, None)                         real 64-token windows at stages 1-2

224^2 is not benchmarked: there the README model's windows (64, 32) do not divide its maps (56, 28), and the reference fails.
One JSON line per model: images/s and ms per forward over `steps` forwards on a CUDA stream (device-resident image and logits, so
the forward is captured into a CUDA graph and replayed), timed with CUDA events after `warmup` untimed forwards; algorithmic GFLOP
per image computed from the model's true shapes (not the zero-padded widths and heads the engine runs; not measured), split into
its parts; from a separate profiled eager forward (vb_profile_read, events around every launch) the time per kernel class and its
share of the profiled forward: attention, the GEMM classes (plain, GELU epilogue, residual epilogue), im2col (the unfold
of every convolution: stem, SSA k|v, LIM, Downsample), LayerNorm / pooling and other (the PEG); and the card name and power limit
read in the same run.  Nothing is written to the tree; --out writes the lines to DIR/scalable_vit_bench.jsonl as well.
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
import scalable_vit_oracle as so  # noqa: E402

CONFIGS = so.BENCH


def flops_per_image(cfg) -> dict:
    """2 * MACs of every convolution and matmul at the model's shapes, by part: the SSA projections and attention, the IWSA
    projections and windowed attention, the LIM convolutions, the MLPs, and the stem, PEGs, Downsamples and head.  LayerNorm, GELU,
    softmax and the pooling are not counted."""
    h, w = (-(-s // 4) for s in cfg["image_size"])
    f = cfg["ff_expansion_factor"]
    parts = dict(ssa=0.0, iwsa_attention=0.0, iwsa_projections=0.0, lim=0.0, mlp=0.0, rest=2.0 * h * w * 49 * cfg["channels"] * cfg["dim"])
    sts = so.stages(cfg)
    for s, st in enumerate(sts):
        if s > 0:
            h, w = -(-h // 2), -(-w // 2)
        n, d, hd, r = h * w, st["dim"], st["heads"], st["reduction_factor"]
        nk = (h // r) * (w // r)
        sk, sv, ik, iv = (hd * st[k] for k in ("ssa_dim_key", "ssa_dim_value", "iwsa_dim_key", "iwsa_dim_value"))
        nw = st["window_size"] ** 2 if st["window_size"] else n
        for L in range(st["depth"]):
            parts["ssa"] += 2.0 * (n * d * sk + nk * r * r * d * (sk + sv) + n * nk * (sk + sv) + n * sv * d)
            parts["mlp"] += 2.0 * 2 * 2 * n * d * f * d
            parts["iwsa_projections"] += 2.0 * n * (d * (2 * ik + iv) + iv * d)
            parts["iwsa_attention"] += 2.0 * n * nw * (ik + iv)
            parts["lim"] += 2.0 * n * 9 * iv * iv
            if L == 0:
                parts["rest"] += 2.0 * n * 9 * d
        if s < len(sts) - 1:
            parts["rest"] += 2.0 * (-(-h // 2)) * (-(-w // 2)) * 9 * d * 2 * d
    parts["rest"] += 2.0 * sts[-1]["dim"] * cfg["num_classes"]
    out = {f"{k}_gflop_per_image": v / 1e9 for k, v in parts.items()}
    out["gflop_per_image"] = sum(parts.values()) / 1e9
    return out


def run(name, batch, steps, warmup):
    import numpy as np
    import torch
    from vit_tensorflow_b200 import from_config, _lib
    cfg = so.make_config(**CONFIGS[name])
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
    total = sum(v["ms"] for v in prof.values())
    return dict(config=name, model="ScalableViT(" + ", ".join(f"{k}={v}" for k, v in CONFIGS[name].items()) + ")", precision="bf16",
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
        raise SystemExit("tools/scalable_vit_bench.py measures on a CUDA device; none is visible")
    hw = card()
    lines = []
    for name in args.configs.split(","):
        line = dict(run(name, args.batch, args.steps, args.warmup), **hw)
        print(json.dumps(line), flush=True)
        lines.append(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "scalable_vit_bench.jsonl"), "a") as fh:
            for line in lines:
                fh.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()

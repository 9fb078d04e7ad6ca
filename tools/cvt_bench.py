"""Images per second of the CvT forward (bf16 engine) on two 224^2 ImageNet configurations.

    python tools/cvt_bench.py [--batch 256] [--steps 20] [--warmup 5] [--out DIR]

  cvt_readme  CvT(num_classes=1000, s3_heads=4)   the reference README's model
  cvt_13      CvT(num_classes=1000)               the constructor defaults: a CvT-13 shape (1 / 2 / 10 blocks of 64 / 192 / 384)

One JSON line per configuration: images/s over `steps` forwards on a CUDA stream (device-resident image and logits, so the
forward is captured into a CUDA graph and replayed, as a server calling forward_raw would run it), timed with CUDA events after
`warmup` untimed forwards; algorithmic GFLOP per image computed from the model's true shapes (not the zero-padded widths the
engine runs; not measured); the per-kernel-class time split of one profiled forward (vb_profile_read, events around every launch:
a separate eager run); the depthwise kernel's achieved bytes/s (the bytes its launches must move, from shapes, over the "other"
class time, which holds only those launches) against the H100 SXM's 3.35 TB/s; the attention share of stage 1 (one profiled forward
of the same model with s2_depth = s3_depth = 0, whose only attention is stage 1's); and the card name and power limit read in the
same run.  Nothing is written to the tree; --out writes the lines to DIR/cvt_bench.jsonl as well.
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
    "cvt_readme": dict(num_classes=1000, s3_heads=4),
    "cvt_13": dict(num_classes=1000),
}
IMAGE = 224
HBM_BYTES_PER_S = 3.35e12            # H100 SXM data sheet


def flops_per_image(m, image=IMAGE) -> dict:
    """2 * MACs at the model's shapes: the stem convolutions (as GEMMs of the im2col rows), per block the depthwise and pointwise
    q / k|v convolutions, QK^T, PV, to_out and the MLP, and the classifier.  LayerNorm, BatchNorm (folded), softmax and pooling are
    not counted."""
    h, w, cin, total, stem = image, image, 3, 0.0, 0.0
    for st in m.stages:
        h, w = -(-h // st["emb_stride"]), -(-w // st["emb_stride"])
        d, k, inner, s = st["emb_dim"], st["proj_kernel"], 64 * st["heads"], st["kv_proj_stride"]
        stem += 2.0 * h * w * st["emb_kernel"] ** 2 * cin * d
        n, nk = h * w, math.ceil(h / s) * math.ceil(w / s)
        total += st["depth"] * 2.0 * (k * k * d * (n + nk) + n * d * inner + nk * d * 2 * inner + 2 * n * nk * inner + n * inner * d
                                      + 2 * n * d * d * st["mlp_mult"])
        cin = d
    total += stem + 2.0 * cin * m.num_classes
    return dict(gflop_per_image=total / 1e9, stem_gflop_per_image=stem / 1e9)


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
    from vit_tensorflow_b200 import CvT
    kw = CONFIGS[name]
    m = CvT(**kw, precision="bf16", seed=0)
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
    dw = prof["other"]
    dw_bps = dw["bytes"] / (dw["ms"] / 1e3) if dw["ms"] > 0 else None
    s1 = CvT(**kw, s2_depth=0, s3_depth=0, precision="bf16", seed=0)   # stage 1's blocks only (the later stems stay)
    fwd1, _, _ = _forward_fn(s1, batch)
    fwd1()
    p1 = _profile(s1, fwd1)
    p1_total = sum(v["ms"] for v in p1.values())
    f = flops_per_image(m)
    ips = batch / (ms / 1e3)
    return dict(config=name, model="CvT(" + ", ".join(f"{k}={v}" for k, v in kw.items()) + ")", image=IMAGE, precision="bf16",
                batch=batch, steps=steps, ms_per_forward=ms, images_per_s=ips, tflops_achieved=ips * f["gflop_per_image"] / 1e3,
                **f, graph_replays=graphs["replays"],
                profile_ms={k: round(v["ms"], 4) for k, v in prof.items() if v["launches"]},
                profile_launches={k: v["launches"] for k, v in prof.items() if v["launches"]},
                dwconv_ms=dw["ms"], dwconv_bytes_per_s=dw_bps, dwconv_share_of_hbm_peak=(dw_bps / HBM_BYTES_PER_S) if dw_bps else None,
                stage1_attention_ms=p1["attention"]["ms"], stage1_profiled_ms=p1_total,
                stage1_attention_share=p1["attention"]["ms"] / p1_total if p1_total > 0 else None)


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
        raise SystemExit("tools/cvt_bench.py measures on a CUDA device; none is visible")
    hw = card()
    lines = []
    for name in args.configs.split(","):
        line = dict(run(name, args.batch, args.steps, args.warmup), **hw)
        print(json.dumps(line), flush=True)
        lines.append(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "cvt_bench.jsonl"), "a") as fh:
            for line in lines:
                fh.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()

"""Time the bf16 flash attention at the shapes of bench.py's two ViT workloads, on the fused q|k|v rows the to_qkv GEMM leaves,
through vb_op_attention_ex (the engine's own dispatch):

    vit_b16       ViT-B/16 224x224, batch 256: n = 197, 12 heads x 64, rows of pitch 2304   (resident-head kernel)
    vit_l16_384   ViT-L/16 384x384, batch 128: n = 577, 16 heads x 64, rows of pitch 3072   (streaming kernel)

    python tools/attention_shapes.py [--iters 100] [--json out.json]

For each shape: ms per call (CUDA events over --iters back-to-back calls after one warm-up call), the algorithmic bytes (q, k
and v read once, the output written once) over that time against the H100 SXM data-sheet HBM3 bandwidth (3.35 TB/s), and
TFLOP/s (4 B h n^2 dh).  The card's name, power limit and maximum SM clock are read in the same run and printed with them.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tools.gemm_shapes import card  # noqa: E402

DATASHEET_HBM_TBPS = 3.35          # H100 SXM HBM3, 700 W part
DH = 64

# name, B, n, heads
SHAPES = [("vit_b16", 256, 197, 12), ("vit_l16_384", 128, 577, 16)]


def time_shape(name, B, n, heads, iters, rng):
    from vit_tensorflow_b200 import _lib
    inner = heads * DH
    rows = rng.standard_normal((B, n, 3 * inner), dtype=np.float32)
    out = np.zeros((B, n, inner), np.float32)
    _lib.last_attention_path()
    _, ms = _lib.op_attention_ex(rows, heads, DH, out, k_off=inner, v_off=2 * inner, iters=iters)
    path = _lib.last_attention_path()
    gbytes = (3 + 1) * B * n * inner * 2 / 1e9
    tflop = 4.0 * B * heads * n * n * DH / 1e12
    return {"shape": name, "B": B, "n": n, "heads": heads, "ld": 3 * inner, "path": path, "ms": ms,
            "gb_per_s": gbytes / (ms * 1e-3), "frac_datasheet_hbm": gbytes / (ms * 1e-3) / (DATASHEET_HBM_TBPS * 1e3),
            "tflops": tflop / (ms * 1e-3)}


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--iters", type=int, default=100)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if args.iters < 50:
        ap.error("--iters must be at least 50")
    from vit_tensorflow_b200 import build
    build.build()
    c = card()
    rng = np.random.default_rng(0)
    rows = [time_shape(name, B, n, heads, args.iters, rng) for name, B, n, heads in SHAPES]
    print(f"{c['name']}, power limit {c['power_limit']}, max SM clock {c['max_sm_clock']}; {args.iters} calls per shape")
    print(f"{'shape':<12} {'B x n x heads':<16} {'path':<6} {'ms':>8} {'GB/s':>8} {'of 3.35 TB/s':>13} {'TFLOP/s':>8}")
    for r in rows:
        shp = f"{r['B']}x{r['n']}x{r['heads']}"
        print(f"{r['shape']:<12} {shp:<16} {r['path']:<6} {r['ms']:8.4f} {r['gb_per_s']:8.0f} {r['frac_datasheet_hbm']:13.3f} "
              f"{r['tflops']:8.1f}")
    if args.json:
        with open(args.json, "w") as fh:
            json.dump({"card": c, "iters": args.iters, "shapes": rows}, fh, indent=1)


if __name__ == "__main__":
    main()

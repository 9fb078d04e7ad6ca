"""Time the wgmma GEMM at the flagship's five shapes (ViT-B/16, 224x224, batch 256: M = 50 432 token rows) with the epilogues
the engine runs them with, through vb_op_gemm (the engine's own plan and dispatch).

    python tools/gemm_shapes.py [--iters 100] [--json out.json]

For each shape: ms per launch (CUDA events over --iters back-to-back launches after one warm-up launch), achieved TFLOP/s
(2 M N K over kernel time) and that rate as a fraction of the H100 SXM data-sheet dense BF16 rate (989 TFLOP/s, a figure for a
700 W card).  The card's name, power limit and maximum SM clock are read in the same run and printed with the numbers.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

DATASHEET_BF16_TFLOPS = 989.0     # H100 SXM, dense BF16, 700 W part
M = 256 * 197                     # batch 256 x (196 patches + class token)
D, MLP = 768, 3072

# name, N, K, epilogue
SHAPES = [
    ("patch_embed", D, 768, "bias + residual + row stats"),
    ("to_qkv", 3 * D, D, "folded LayerNorm"),
    ("to_out", D, D, "bias + in-place residual + row stats"),
    ("fc1", MLP, D, "folded LayerNorm + GELU"),
    ("fc2", D, MLP, "bias + LayerScale + in-place residual + row stats"),
]


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, check=True).stdout.splitlines()[0]
    name, power, clock = (x.strip() for x in q.split(","))
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def bf16(rng, shape, scale=1.0):
    """float32 values; vb_op_gemm rounds them to bf16 on upload"""
    return (scale * rng.standard_normal(shape)).astype(np.float32)


def time_shape(name, N, K, iters, rng):
    from vit_tensorflow_b200 import _lib
    a = bf16(rng, (M, K))
    wt = bf16(rng, (N, K), 1 / np.sqrt(K))
    bias = (0.1 * rng.standard_normal(N)).astype(np.float32)
    out = np.zeros((M, N), np.float32)
    kw = {}
    if name == "patch_embed":
        kw = dict(bias=bias, res=bf16(rng, (M, N)), want_stats=True)
    elif name in ("to_qkv", "fc1"):
        # (sum, sumsq) partials of the A rows per 64 columns, as the previous GEMM's stats_out leaves them
        c = a.astype(np.float64).reshape(M, K // 64, 64).transpose(1, 0, 2)
        stats = np.stack([c.sum(-1), (c ** 2).sum(-1)], -1).astype(np.float32)
        kw = dict(bias=bias, ln_stats=stats, ln_c1=wt.astype(np.float64).sum(1).astype(np.float32), gelu=name == "fc1")
    elif name == "to_out":
        out = bf16(rng, (M, N))
        kw = dict(bias=bias, res="out", want_stats=True)
    else:
        out = bf16(rng, (M, N))
        kw = dict(bias=bias, scale=rng.uniform(0.5, 1.5, N).astype(np.float32), res="out", want_stats=True)
    _, _, ms = _lib.op_gemm(a, wt, N, K, out, iters=iters, **kw)
    tflops = 2.0 * M * N * K / (ms * 1e-3) / 1e12
    return {"shape": name, "M": M, "N": N, "K": K, "ms": ms, "tflops": tflops, "frac_datasheet_peak": tflops / DATASHEET_BF16_TFLOPS}


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--iters", type=int, default=100)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if args.iters < 50:
        ap.error("--iters must be at least 50: one warm-up launch precedes the timed ones")
    from vit_tensorflow_b200 import build
    build.build()
    c = card()
    rng = np.random.default_rng(0)
    rows = []
    for name, N, K, epi in SHAPES:
        r = time_shape(name, N, K, args.iters, rng)
        r["epilogue"] = epi
        rows.append(r)
    print(f"{c['name']}, power limit {c['power_limit']}, max SM clock {c['max_sm_clock']}; {args.iters} launches per shape")
    print(f"{'shape':<12} {'M x N x K':<20} {'ms':>8} {'TFLOP/s':>8} {'of 989 (data sheet)':>20}  epilogue")
    for r in rows:
        mnk = f"{r['M']}x{r['N']}x{r['K']}"
        print(f"{r['shape']:<12} {mnk:<20} {r['ms']:8.3f} {r['tflops']:8.1f} {r['frac_datasheet_peak']:20.3f}  {r['epilogue']}")
    if args.json:
        with open(args.json, "w") as fh:
            json.dump({"card": c, "iters": args.iters, "shapes": rows}, fh, indent=1)


if __name__ == "__main__":
    main()

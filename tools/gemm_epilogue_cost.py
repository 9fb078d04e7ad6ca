"""What the GELU costs the fc1 GEMM of the flagship (ViT-B/16, 224x224, batch 256: M = 50 432 token rows, N = 3072, K = 768),
measured against the same launch without it and against to_qkv (N = 2304), which runs the same tile, ring and folded-LayerNorm
epilogue.  Everything goes through vb_op_gemm (the engine's own plan and dispatch).

    python tools/gemm_epilogue_cost.py [--iters 100] [--rounds 5] [--long-ms 600] [--json out.json]

short  fc1 with GELU, fc1 without it and to_qkv, alternated for --rounds rounds of --iters back-to-back launches each (CUDA
       events, one warm-up launch per call); the best and median ms per launch of each, and TFLOP/s (2 M N K over kernel time).
long   fc1 with GELU and fc1 without it, once each, over a window of about --long-ms of back-to-back launches, with nvidia-smi
       sampling the SM clock, power and throttle reasons (read-only) as bench.py's ClockSampler does.  A GELU that costs more
       here than in the short windows is paid in clock under the power limit rather than in instructions.

The card's name, power limit and maximum SM clock are read in the same run and printed with the numbers.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tools.gemm_shapes import M, D, MLP, card, bf16   # noqa: E402

K = D
SHAPES = {"fc1_gelu": (MLP, True), "fc1_plain": (MLP, False), "to_qkv": (3 * D, False)}


def operands(rng):
    """A [M, K] with its per-64-column (sum, sumsq) partials, and per N a weight, c2 bias and c1 = row sums of the weight"""
    a = bf16(rng, (M, K))
    c = a.astype(np.float64).reshape(M, K // 64, 64).transpose(1, 0, 2)
    stats = np.stack([c.sum(-1), (c ** 2).sum(-1)], -1).astype(np.float32)
    per_n = {}
    for n in sorted({n for n, _ in SHAPES.values()}):
        wt = bf16(rng, (n, K), 1 / np.sqrt(K))
        per_n[n] = dict(wt=wt, bias=(0.1 * rng.standard_normal(n)).astype(np.float32),
                        ln_c1=wt.astype(np.float64).sum(1).astype(np.float32))
    return a, stats, per_n


def run(name, a, stats, per_n, iters):
    from vit_tensorflow_b200 import _lib
    n, gelu = SHAPES[name]
    p = per_n[n]
    out = np.zeros((M, n), np.float32)
    _, _, ms = _lib.op_gemm(a, p["wt"], n, K, out, bias=p["bias"], ln_stats=stats, ln_c1=p["ln_c1"], gelu=gelu, iters=iters)
    return ms


def tflops(n, ms):
    return 2.0 * M * n * K / (ms * 1e-3) / 1e12


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--iters", type=int, default=100)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--long-ms", type=float, default=600.0, help="length of each long window (at least 500)")
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if args.iters < 50 or args.rounds < 1 or args.long_ms < 500:
        ap.error("--iters >= 50, --rounds >= 1 and --long-ms >= 500")
    from bench import ClockSampler
    from vit_tensorflow_b200 import build
    build.build()
    c = card()
    a, stats, per_n = operands(np.random.default_rng(0))

    for name in SHAPES:                                   # warm-up: module load, first-use attributes
        run(name, a, stats, per_n, 50)
    short = {name: [] for name in SHAPES}
    for _ in range(args.rounds):
        for name in SHAPES:
            short[name].append(run(name, a, stats, per_n, args.iters))

    long = {}
    for name in ("fc1_gelu", "fc1_plain"):
        iters = max(50, int(args.long_ms / min(short[name])))
        sampler = ClockSampler(0)                         # the device the library runs on, as in bench.py with one GPU
        sampler.wait_ready()
        ms = run(name, a, stats, per_n, iters)
        long[name] = dict(iters=iters, window_ms=ms * iters, ms=ms, tflops=tflops(SHAPES[name][0], ms), clocks=sampler.stop())

    rows = {name: dict(N=SHAPES[name][0], gelu=SHAPES[name][1], ms_all=v, ms_best=min(v), ms_median=statistics.median(v),
                       tflops_best=tflops(SHAPES[name][0], min(v)), tflops_median=tflops(SHAPES[name][0], statistics.median(v)))
            for name, v in short.items()}
    print(f"{c['name']}, power limit {c['power_limit']}, max SM clock {c['max_sm_clock']}; M = {M}, K = {K}")
    print(f"short windows: {args.rounds} alternating rounds of {args.iters} launches")
    print(f"{'launch':<10} {'N':>5} {'best ms':>8} {'median ms':>10} {'TFLOP/s best':>13} {'median':>8}")
    for name, r in rows.items():
        print(f"{name:<10} {r['N']:>5} {r['ms_best']:8.4f} {r['ms_median']:10.4f} {r['tflops_best']:13.1f} {r['tflops_median']:8.1f}")
    g, p, q = rows["fc1_gelu"], rows["fc1_plain"], rows["to_qkv"]
    print(f"fc1 GELU / fc1 plain time (median): {g['ms_median'] / p['ms_median']:.4f};  "
          f"fc1 GELU per-FLOP rate / to_qkv's: {g['tflops_median'] / q['tflops_median']:.4f};  "
          f"fc1 plain / to_qkv: {p['tflops_median'] / q['tflops_median']:.4f}")
    print("long windows:")
    for name, r in long.items():
        ck = r["clocks"]
        print(f"{name:<10} {r['iters']:>5} launches, {r['window_ms']:7.1f} ms: {r['ms']:.4f} ms/launch, {r['tflops']:.1f} TFLOP/s; "
              f"SM clock median {ck.get('sm_mhz')} MHz (max {ck.get('sm_max_mhz')}), power max {ck.get('power_w_max')} W "
              f"of {ck.get('power_limit_w')} W, reasons {ck.get('reasons')}")
    print(f"fc1 GELU / fc1 plain time (long): {long['fc1_gelu']['ms'] / long['fc1_plain']['ms']:.4f}")
    if args.json:
        with open(args.json, "w") as fh:
            json.dump({"card": c, "iters": args.iters, "rounds": args.rounds, "short": rows, "long": long}, fh, indent=1)


if __name__ == "__main__":
    main()

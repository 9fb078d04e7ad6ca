"""Images per second of the training-mode dropout forward (bf16 engine, vb_forward_train) against the inference forward.

    python tools/dropout_bench.py [--batch 256] [--steps 30] [--warmup 5] [--rounds 3] [--out DIR]

  vit_b16    ViT-B/16 at 224^2 (dim 768, depth 12, 12 heads of 64, mlp 3072, 1000 classes), dropout 0.1, emb_dropout 0.1
  crossvit   the reference README's CrossViT (image 256, sm_dim 192, lg_dim 384, depth 4, ...) at its default rates 0.1 / 0.1

Per configuration the two forwards run on one CUDA stream from device buffers (so both are captured into CUDA graphs and
replayed), timed with CUDA events after `warmup` calls and alternated over `rounds` rounds; then a profiled eager call of each
(vb_profile_read) gives the per-class GEMM times, where dropout adds its epilogue work.  Each JSON line carries the card name
and power limit read in the same run.  Nothing is written to the tree; --out writes the lines to DIR/dropout_bench.jsonl.
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

VIT_B16 = dict(image_size=224, patch_size=16, num_classes=1000, dim=768, depth=12, heads=12, mlp_dim=3072, dropout=0.1,
               emb_dropout=0.1)
CROSSVIT = dict(image_size=256, num_classes=1000, depth=4, sm_dim=192, sm_patch_size=16, sm_enc_depth=2, sm_enc_heads=8,
                sm_enc_mlp_dim=2048, lg_dim=384, lg_patch_size=64, lg_enc_depth=3, lg_enc_heads=8, lg_enc_mlp_dim=2048,
                cross_attn_depth=2, cross_attn_heads=8)                 # README; dropout / emb_dropout: the defaults, 0.1


def _timed(fn, stream, steps, warmup):
    import torch
    for _ in range(warmup):
        fn()
    stream.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(stream)
    for _ in range(steps):
        fn()
    b.record(stream)
    b.synchronize()
    return a.elapsed_time(b) / steps


def run(name, model, size, batch, steps, warmup, rounds):
    import torch
    from vit_tensorflow_b200 import _lib
    model.set_dropout_seed(0)
    img = torch.randn(batch, size, size, 3, device="cuda")
    out = torch.empty(batch, model.num_classes, device="cuda")
    s = torch.cuda.Stream()
    torch.cuda.synchronize()

    def fwd(training):
        return lambda: model.forward_raw(img.data_ptr(), _lib.MEM_DEVICE, batch, size, size, out.data_ptr(), _lib.MEM_DEVICE,
                                         s.cuda_stream, training=training)
    ms = {"inference": [], "training": []}
    for _ in range(rounds):
        for k, training in (("inference", False), ("training", True)):
            ms[k].append(_timed(fwd(training), s, steps, warmup))
    gemm = {}
    for k, training in (("inference", False), ("training", True)):
        model.profile(True)
        model.profile_read(reset=True)
        fwd(training)()                                    # profiling runs eagerly, with per-class events
        torch.cuda.synchronize()
        prof = model.profile_read(reset=True)
        model.profile(False)
        gemm[k] = {c: round(v["ms"], 4) for c, v in prof.items() if c.startswith("gemm") or c == "other"}
    best = {k: min(v) for k, v in ms.items()}
    return dict(config=name, batch=batch, **card(),
                images_per_s={k: round(batch / (v / 1e3), 1) for k, v in best.items()},
                ms_per_call={k: [round(x, 4) for x in v] for k, v in ms.items()},
                training_over_inference=round(best["training"] / best["inference"], 4),
                profile_ms=gemm)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    from vit_tensorflow_b200 import CrossViT, ViT
    lines = [run("vit_b16", ViT(**VIT_B16, precision="bf16", seed=0), 224, a.batch, a.steps, a.warmup, a.rounds),
             run("crossvit_readme", CrossViT(**CROSSVIT, precision="bf16", seed=0), 256, a.batch, a.steps, a.warmup, a.rounds)]
    for ln in lines:
        print(json.dumps(ln))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "dropout_bench.jsonl"), "w") as fh:
            fh.writelines(json.dumps(ln) + "\n" for ln in lines)


if __name__ == "__main__":
    main()

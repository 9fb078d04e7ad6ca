"""Images per second of the DistillWrapper call (bf16 engine) in a DeiT-B-like setup, against its parts timed alone.

    python tools/distill_bench.py [--batch 256] [--steps 20] [--warmup 5] [--out DIR]

  student   DistillableViT ViT-B/16 at 224^2 (dim 768, depth 12, 12 heads of 64, mlp 3072, 1000 classes)
  teacher   CaiT-S36 at 224^2 (patch 16, dim 384, 36 layers and 2 class-attention layers, 8 heads of 48, mlp 1536, 1000 classes),
            an engine model, so the wrapper runs it through its handle

Lines (JSON, one per measurement, each with the card name and power limit read in the same run):
  wrapper        images/s of wrapper.forward_raw (device image, labels and loss; a CUDA stream, so the wrapper's section and the
                 teacher's forward are captured into CUDA graphs and replayed), timed with CUDA events after `warmup` calls
  parts          images/s of the teacher's plain forward plus the student's distillation forward (vb_forward_distill), the two
                 timed alone on the same stream, and their sum
  profile        a separate torch.profiler run of one wrapper call: the device time of the loss kernels and of the three heads
                 (the teacher's, the student's and distill_mlp, each a row LayerNorm and a GEMM), and their shares of the call
Nothing is written to the tree; --out writes the lines to DIR/distill_bench.jsonl (and the profiler table beside them).
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from cct_bench import card  # noqa: E402

STUDENT = dict(image_size=224, patch_size=16, num_classes=1000, dim=768, depth=12, heads=12, mlp_dim=3072)
TEACHER = dict(image_size=224, patch_size=16, num_classes=1000, dim=384, depth=36, cls_depth=2, heads=8, dim_head=48, mlp_dim=1536)
LOSS_KERNELS = ("distill_rows_kernel", "mim_loss_final_kernel", "distill_out_kernel")


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


def run(batch, steps, warmup, out_dir):
    import numpy as np
    import torch
    from vit_tensorflow_b200 import CaiT, DistillableViT, DistillWrapper, _lib
    student = DistillableViT(**STUDENT, precision="bf16", seed=0)
    teacher = CaiT(**TEACHER, precision="bf16", seed=1)
    wrapper = DistillWrapper(teacher, student, temperature=3.0, alpha=0.5, seed=2)
    assert wrapper._engine_teacher()
    K, size = STUDENT["num_classes"], STUDENT["image_size"]
    img = torch.randn(batch, size, size, 3, device="cuda")
    labels = torch.nn.functional.one_hot(torch.randint(0, K, (batch,), device="cuda"), K).float()
    loss = torch.empty(batch, device="cuda")
    t_logits, s_logits, tokens = (torch.empty(batch, n, device="cuda") for n in (K, K, STUDENT["dim"]))
    token = np.ascontiguousarray(wrapper.distillation_token.reshape(-1))
    s = torch.cuda.Stream()
    torch.cuda.synchronize()

    def call():
        wrapper.forward_raw(img.data_ptr(), _lib.MEM_DEVICE, batch, size, size, labels.data_ptr(), _lib.MEM_DEVICE, 3.0, 0.5,
                            loss.data_ptr(), _lib.MEM_DEVICE, s.cuda_stream, teacher=teacher)

    def teacher_forward():
        teacher.forward_raw(img.data_ptr(), _lib.MEM_DEVICE, batch, size, size, t_logits.data_ptr(), _lib.MEM_DEVICE, s.cuda_stream)

    student._finalize()

    def student_forward():                                   # vb_forward_distill: eager, the token uploaded from the host
        _lib.check(student._lib.vb_forward_distill(student._h, C.c_void_p(img.data_ptr()), _lib.MEM_DEVICE, batch, size, size,
                                                   token.ctypes.data_as(C.c_void_p), C.c_void_p(s_logits.data_ptr()),
                                                   C.c_void_p(tokens.data_ptr()), _lib.MEM_DEVICE, C.c_void_p(s.cuda_stream)), student._h)

    hw = card()
    lines = []
    ms = _timed(call, s, steps, warmup)
    assert np.isfinite(loss.cpu().numpy()).all()
    lines.append(dict(line="wrapper", batch=batch, ms_per_call=ms, images_per_s=batch / (ms / 1e3),
                      graph_replays=wrapper.graph_stats()["replays"], teacher_graph_replays=teacher.graph_stats()["replays"], **hw))
    mt = _timed(teacher_forward, s, steps, warmup)
    ms_ = _timed(student_forward, s, steps, warmup)
    lines.append(dict(line="parts", batch=batch, teacher_ms=mt, student_distill_ms=ms_, sum_ms=mt + ms_,
                      images_per_s=batch / ((mt + ms_) / 1e3), **hw))

    from torch.profiler import ProfilerActivity, profile
    call()
    s.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        call()
        s.synchronize()
    kernels = {}
    for e in prof.key_averages():
        if e.device_type is not None and "CUDA" in str(e.device_type) and e.device_time_total > 0:
            kernels[e.key] = kernels.get(e.key, 0.0) + e.device_time_total / 1e3        # ms
    total = sum(kernels.values())
    loss_ms = sum(v for k, v in kernels.items() if any(n in k for n in LOSS_KERNELS))
    # distill_mlp runs as one pool_layernorm and one gemm_simt launch, as do the student's and the teacher's own heads: the time
    # of those two kernels over the call bounds distill_mlp's from above
    head_ms = sum(v for k, v in kernels.items() if "pool_layernorm" in k or "gemm_simt" in k)
    lines.append(dict(line="profile", batch=batch, call_device_ms=total, loss_kernels_ms=loss_ms, loss_share=loss_ms / total,
                      three_heads_ms=head_ms, three_heads_share=head_ms / total, **hw))
    if out_dir:
        os.makedirs(out_dir, exist_ok=True)
        with open(os.path.join(out_dir, "distill_bench_profile.txt"), "w") as fh:
            fh.write(prof.key_averages().table(sort_by="device_time_total", row_limit=40))
    return lines


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("tools/distill_bench.py measures on a CUDA device; none is visible")
    lines = run(args.batch, args.steps, args.warmup, args.out)
    for line in lines:
        print(json.dumps(line), flush=True)
    if args.out:
        with open(os.path.join(args.out, "distill_bench.jsonl"), "a") as fh:
            for line in lines:
                fh.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()

"""Images per second of the CrossFormer forward (bf16 engine) on two 224^2 ImageNet configurations.

    python tools/crossformer_bench.py [--batch 256] [--steps 20] [--warmup 5] [--out DIR]

  crossformer_readme  CrossFormer(num_classes=1000)                       the reference README's model (the constructor defaults)
  crossformer_96      CrossFormer(dim=(96, 192, 384, 768), depth=(2, 2, 6, 2), num_classes=1000)

One JSON line per configuration: images/s over `steps` forwards on a CUDA stream (device-resident image and logits, so the
forward is captured into a CUDA graph and replayed, as a server calling forward_raw would run it), timed with CUDA events after
`warmup` untimed forwards; GFLOP per image computed from shapes (not measured), both as the engine executes it (the cross-scale
embedding as one convolution of the largest kernel with the others nested in it, the v projection alone for one-token windows)
and as the reference defines it (one convolution per kernel size, the whole q|k|v); the per-kernel-class time split of one
profiled eager forward (vb_profile_read, events around every launch: a separate run); the windowed attention's device time,
summed over the windowed-bias flash kernel's launches in one torch.profiler trace of an eager forward (another separate run); and
the card name and power limit read in the same run.  Nothing is written to the tree; --out writes the lines to
DIR/crossformer_bench.jsonl as well.
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

CONFIGS = {
    "crossformer_readme": dict(num_classes=1000),
    "crossformer_96": dict(dim=(96, 192, 384, 768), depth=(2, 2, 6, 2), num_classes=1000),
}
IMAGE = 224
DIM_HEAD, MLP_MULT = 32, 4
ATTN_KERNEL = "attn_flash_kernel<32, true, true>"


def _dim_scales(dim, n):                                  # crossformer.py:38-39
    s = [int(dim / (2 ** i)) for i in range(1, n)]
    return s + [dim - sum(s)]


def flops_per_image(m, image=IMAGE) -> dict:
    """2 * MACs at the model's shapes: the cross-scale embeddings, per layer q|k|v, QK^T and PV inside the windows, to_out and both
    MLPs, and the classifier.  LayerNorm, softmax, the position-bias MLP (evaluated once per weight set) and pooling are not
    counted.  `executed` counts what the engine runs, `reference` what crossformer.py defines."""
    h, w, cin = image, image, 3
    ex = ref = stage1_ex = stage1_ref = 0.0
    for i, st in enumerate(m.stages):
        s, d, ks = st["stride"], st["dim"], st["kernels"]
        h, w = -(-h // s), -(-w // s)
        n, inner = h * w, DIM_HEAD * (d // DIM_HEAD)
        emb_ex = 2.0 * n * max(ks) ** 2 * cin * d
        emb_ref = sum(2.0 * n * k * k * cin * ds for k, ds in zip(ks, _dim_scales(d, len(ks))))
        lay_ex = lay_ref = 0.0
        for wsz in (st["local_wsz"], st["global_wsz"]):
            attn = 4.0 * n * wsz * wsz * inner + 2.0 * n * inner * d
            lay_ref += 2.0 * n * d * 3 * inner + attn
            lay_ex += 2.0 * n * d * inner if wsz == 1 else 2.0 * n * d * 3 * inner + attn
        mlp = 2 * 4.0 * n * d * MLP_MULT * d
        ex += emb_ex + st["depth"] * (lay_ex + mlp)
        ref += emb_ref + st["depth"] * (lay_ref + mlp)
        if i == 0:
            stage1_ex, stage1_ref = ex, ref
        cin = d
    head = 2.0 * cin * m.num_classes
    return dict(gflop_per_image_executed=(ex + head) / 1e9, gflop_per_image_reference=(ref + head) / 1e9,
                stage1_gflop_per_image_executed=stage1_ex / 1e9, stage1_gflop_per_image_reference=stage1_ref / 1e9)


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


def _attention_ms(fwd, s):
    """Device time of the windowed-bias flash kernel in one eager forward (profiling mode is eager: no graph replay)."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as p:
        fwd()
        s.synchronize()
    evs = [e for e in p.events() if ATTN_KERNEL in e.name]
    return sum(e.device_time_total for e in evs) / 1e3, len(evs)


def run(name, batch, steps, warmup):
    import numpy as np
    import torch
    from vit_tensorflow_b200 import CrossFormer
    kw = CONFIGS[name]
    m = CrossFormer(**kw, precision="bf16", seed=0)
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
    m.profile(True)                                  # eager, without events: the trace sees every kernel launch on its own
    attn_ms, attn_launches = _attention_ms(fwd, s)
    m.profile(False)
    f = flops_per_image(m)
    ips = batch / (ms / 1e3)
    return dict(config=name, model="CrossFormer(" + ", ".join(f"{k}={v}" for k, v in kw.items()) + ")", image=IMAGE, precision="bf16",
                batch=batch, steps=steps, ms_per_forward=ms, images_per_s=ips, tflops_achieved_executed=ips * f["gflop_per_image_executed"] / 1e3,
                **f, graph_replays=graphs["replays"],
                profile_ms={k: round(v["ms"], 4) for k, v in prof.items() if v["launches"]},
                profile_launches={k: v["launches"] for k, v in prof.items() if v["launches"]},
                attention_ms=attn_ms, attention_launches=attn_launches)


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
        raise SystemExit("tools/crossformer_bench.py measures on a CUDA device; none is visible")
    hw = card()
    lines = []
    for name in args.configs.split(","):
        line = dict(run(name, args.batch, args.steps, args.warmup), **hw)
        print(json.dumps(line), flush=True)
        lines.append(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "crossformer_bench.jsonl"), "a") as fh:
            for line in lines:
                fh.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()

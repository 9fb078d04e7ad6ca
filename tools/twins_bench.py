"""Images per second of the Twins-SVT forward (bf16 engine) on two 224^2 ImageNet configurations.

    python tools/twins_bench.py [--batch 256] [--steps 20] [--warmup 5] [--out DIR]

  twins_readme    TwinsSVT(num_classes=1000)                          the reference README's model (the constructor defaults)
  twins_2_2_10_4  TwinsSVT(num_classes=1000, s3_depth=9, s4_depth=3)  2 / 2 / 10 / 4 blocks per stage

One JSON line per configuration: images/s over `steps` forwards on a CUDA stream (device-resident image and logits, so the
forward is captured into a CUDA graph and replayed, as a server calling forward_raw would run it), timed with CUDA events after
`warmup` untimed forwards; algorithmic GFLOP per image computed from the model's true shapes (not the zero-padded widths the
engine runs; not measured); the per-kernel-class time split of one profiled eager forward (vb_profile_read, events around every
launch: a separate run); the local attention's device time, summed over the windowed flash kernel's launches in one
torch.profiler trace of an eager forward (another separate run); and the card name and power limit read in the same run.
Nothing is written to the tree; --out writes the lines to DIR/twins_bench.jsonl as well.
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
    "twins_readme": dict(num_classes=1000),
    "twins_2_2_10_4": dict(num_classes=1000, s3_depth=9, s4_depth=3),
}
IMAGE = 224
INNER, MLP_MULT = 512, 4             # 8 heads of 64 and an MLP multiplier of 4 in every stage
LOCAL_KERNEL = "attn_flash_kernel<false, true>"


def flops_per_image(m, image=IMAGE) -> dict:
    """2 * MACs at the model's shapes: the patch embeddings, per layer the local q|k|v, QK^T and PV inside the windows, to_out, the
    global to_q, the k x k stride-k to_kv, QK^T and PV against its keys, to_out and both MLPs, the PEGs and the classifier.
    LayerNorm, softmax and pooling are not counted.  Returns the total and stage 1's share."""
    h, w, cin, per_stage = image, image, 3, []
    for i, st in enumerate(m.stages):
        ps, d, k = st["patch_size"], st["emb_dim"], st["global_k"]
        h, w = h // ps, w // ps
        n, nk = h * w, (h // k) * (w // k)
        f = 2.0 * n * cin * ps * ps * d + 2.0 * n * m.peg_kernel_size ** 2 * d
        glob = 2.0 * n * d * INNER + 2.0 * nk * k * k * d * 2 * INNER + 4.0 * n * nk * INNER + 2.0 * n * INNER * d
        mlp = 4.0 * n * d * MLP_MULT * d
        local = 0.0
        if i < 3:
            p2 = st["local_patch_size"] ** 2
            local = 2.0 * n * d * 3 * INNER + 4.0 * n * p2 * INNER + 2.0 * n * INNER * d + mlp
        f += (1 + st["depth"]) * (local + glob + mlp)
        per_stage.append(f)
        cin = d
    total = sum(per_stage) + 2.0 * cin * m.num_classes
    return dict(gflop_per_image=total / 1e9, stage1_gflop_per_image=per_stage[0] / 1e9)


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


def _local_attention_ms(fwd, s):
    """Device time of the windowed flash kernel in one eager forward (profiling mode is eager: no graph replay)."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as p:
        fwd()
        s.synchronize()
    evs = [e for e in p.events() if LOCAL_KERNEL in e.name]
    return sum(e.device_time_total for e in evs) / 1e3, len(evs)


def run(name, batch, steps, warmup):
    import numpy as np
    import torch
    from vit_tensorflow_b200 import TwinsSVT
    kw = CONFIGS[name]
    m = TwinsSVT(**kw, precision="bf16", seed=0)
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
    local_ms, local_launches = _local_attention_ms(fwd, s)
    m.profile(False)
    f = flops_per_image(m)
    ips = batch / (ms / 1e3)
    return dict(config=name, model="TwinsSVT(" + ", ".join(f"{k}={v}" for k, v in kw.items()) + ")", image=IMAGE, precision="bf16",
                batch=batch, steps=steps, ms_per_forward=ms, images_per_s=ips, tflops_achieved=ips * f["gflop_per_image"] / 1e3,
                **f, graph_replays=graphs["replays"],
                profile_ms={k: round(v["ms"], 4) for k, v in prof.items() if v["launches"]},
                profile_launches={k: v["launches"] for k, v in prof.items() if v["launches"]},
                local_attention_ms=local_ms, local_attention_launches=local_launches)


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
        raise SystemExit("tools/twins_bench.py measures on a CUDA device; none is visible")
    hw = card()
    lines = []
    for name in args.configs.split(","):
        line = dict(run(name, args.batch, args.steps, args.warmup), **hw)
        print(json.dumps(line), flush=True)
        lines.append(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "twins_bench.jsonl"), "a") as fh:
            for line in lines:
                fh.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()

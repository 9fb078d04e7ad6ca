"""Golden fixtures of CrossFormer (reference crossformer.py) produced by the REFERENCE'S OWN CODE running over the numpy stand-in for
TensorFlow (oracle/tf_shim.py plus the layers of tests/cct_oracle.py, tests/levit_oracle.py and tests/cvt_oracle.py, which tests/crossformer_oracle.py reuses), the sibling of make_twins_golden.py.

    python tests/golden/make_crossformer_golden.py [--force] [--reference /root/reference]

For every case of crossformer_oracle.SMALL and crossformer_oracle.BENCH (batch 2) this builds `crossformer.CrossFormer(**kwargs)`, calls it once so that
Keras builds its variables, loads the seeded weights by attribute path, calls `model(img)` (training=True: no BatchNorm, dropout 0) and stores
logits_ref_f32 (and logits_ref_f64 for the small cases) in
tests/golden/<name>__<weights>__refshim.npz.  The reference checkout is absent where the GPU tests run, hence the fixtures.
"""
import json
import os
import sys
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))
import crossformer_oracle as lo  # noqa: E402


def main():
    ref_root = sys.argv[sys.argv.index("--reference") + 1] if "--reference" in sys.argv else "/root/reference"
    ref_dir = os.path.join(ref_root, "vit_tensorflow")
    if not os.path.isdir(ref_dir):
        raise SystemExit(f"{ref_dir} not found: these fixtures can only be generated where the reference checkout exists")
    for dtype, tag in ((np.float32, "f32"), (np.float64, "f64")):
        with lo.reference_module(ref_dir, dtype) as mod:
            for group, cases in (("small", lo.SMALL), ("bench", lo.BENCH)):
                if group == "bench" and tag == "f64":
                    continue
                for name, kw in cases.items():
                    cfg = lo.make_config(**kw)
                    img = lo.make_image(cfg, lo.BATCH, lo.IMAGE_SEED)
                    for wname in ("init_weights", "stress_weights"):
                        path = os.path.join(HERE, f"{name}__{wname}__refshim.npz")
                        if os.path.exists(path) and "--force" not in sys.argv and tag == "f32":   # never rewritten silently
                            continue
                        if tag == "f64" and not os.path.exists(path):
                            continue
                        t0 = time.time()
                        w = getattr(lo, wname)(cfg, lo.WEIGHT_SEED)
                        got = lo.reference_logits(mod, cfg, w, img, dtype)
                        out = dict(np.load(path)) if tag == "f64" else {}
                        logits = got
                        out[f"logits_ref_{tag}"] = logits.astype(dtype)
                        meta = dict(config=kw, weights=wname, weight_seed=lo.WEIGHT_SEED, image_seed=lo.IMAGE_SEED, batch=lo.BATCH,
                                    generator="tests/golden/make_crossformer_golden.py",
                                    reference="vit_tensorflow/crossformer.py (unmodified) over the numpy shim", numpy=np.__version__)
                        out["meta"] = json.dumps(meta)
                        np.savez(path, **out)
                        print(f"{name} {wname} {tag}: |logits| mean {np.abs(logits).mean():.3f} ({time.time() - t0:.1f} s)")


if __name__ == "__main__":
    main()

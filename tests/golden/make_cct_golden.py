"""Golden fixtures of the CCT (reference cct.py) produced by the REFERENCE'S OWN CODE running over the numpy stand-in for
TensorFlow (oracle/tf_shim.py plus the Conv2D / MaxPool2D / ReLU of tests/cct_oracle.py), the sibling of make_ref_golden.py.

    python tests/golden/make_cct_golden.py [--force] [--reference /root/reference]

For every case of cct_oracle.SMALL and cct_oracle.BENCH (batch 2) this builds `cct.CCT(**kwargs)`, loads the seeded weights by
attribute path, calls `model(img, training=False)` and stores logits_ref_f32 (and logits_ref_f64 for the small cases) in
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
import cct_oracle as co  # noqa: E402


def main():
    ref_root = sys.argv[sys.argv.index("--reference") + 1] if "--reference" in sys.argv else "/root/reference"
    ref_dir = os.path.join(ref_root, "vit_tensorflow")
    if not os.path.isdir(ref_dir):
        raise SystemExit(f"{ref_dir} not found: these fixtures can only be generated where the reference checkout exists")
    for group, cases in (("small", co.SMALL), ("bench", co.BENCH)):
        for name, kw in cases.items():
            cfg = co.make_config(**kw)
            img = co.make_image(cfg, co.BATCH, co.IMAGE_SEED)
            for wname in ("init_weights", "stress_weights"):
                path = os.path.join(HERE, f"{name}__{wname}__refshim.npz")
                if os.path.exists(path) and "--force" not in sys.argv:      # committed fixtures are never rewritten silently
                    continue
                t0 = time.time()
                w = getattr(co, wname)(cfg, co.WEIGHT_SEED)
                out = dict(logits_ref_f32=co.reference_logits(cfg, w, img, np.float32, ref_dir).astype(np.float32))
                if group == "small":
                    out["logits_ref_f64"] = co.reference_logits(cfg, w, img, np.float64, ref_dir)
                meta = dict(config=kw, weights=wname, weight_seed=co.WEIGHT_SEED, image_seed=co.IMAGE_SEED, batch=co.BATCH,
                            generator="tests/golden/make_cct_golden.py", reference="vit_tensorflow/cct.py (unmodified) over the numpy shim",
                            numpy=np.__version__)
                np.savez(path, meta=json.dumps(meta), **out)
                print(f"{name} {wname}: {out['logits_ref_f32'].shape}, |logits| mean {np.abs(out['logits_ref_f32']).mean():.3f} "
                      f"({time.time() - t0:.1f} s)")


if __name__ == "__main__":
    main()

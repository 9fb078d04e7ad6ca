"""Golden fixtures of DistillableT2TViT (reference distill.py:61-72) produced by the REFERENCE'S OWN CODE running over the numpy
stand-in for TensorFlow (oracle/tf_shim.py).

    python tests/golden/make_distill_golden.py [--force] [--reference /root/reference]

For every case of distill_oracle.CASES (batch 2) and both weight sets (Keras' initial values, and 'stress' with every bias, beta and
gamma nonzero) this builds `distill.DistillableT2TViT(**kwargs)`, calls it once so that Keras builds its variables, loads the seeded
weights by attribute path, calls `model(img, distill_token=token, training=False)` in float32 and in float64 and stores
logits_ref_f32 / distill_ref_f32 / logits_ref_f64 / distill_ref_f64 in tests/golden/<name>__<weights>__refshim.npz.  Weights,
image and token are regenerated from the seeds in `meta`.  The reference checkout is absent where the GPU tests run, hence the
fixtures.
"""
import json
import os
import sys
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))
import distill_oracle as do  # noqa: E402


def main():
    ref_root = sys.argv[sys.argv.index("--reference") + 1] if "--reference" in sys.argv else "/root/reference"
    ref_dir = os.path.join(ref_root, "vit_tensorflow")
    if not os.path.isdir(ref_dir):
        raise SystemExit(f"{ref_dir} not found: these fixtures can only be generated where the reference checkout exists")
    for name in do.CASES:
        for gen in do.WEIGHTS:
            path = os.path.join(HERE, do.fixture_name(name, gen))
            if os.path.exists(path) and "--force" not in sys.argv:          # committed fixtures are never rewritten silently
                continue
            t0 = time.time()
            _, w, img, tok = do.inputs(name, gen)
            out = {}
            for dtype, tag in ((np.float32, "f32"), (np.float64, "f64")):
                logits, dist, _ = do.reference_distill(ref_dir, name, w, img, tok, dtype)
                out[f"logits_ref_{tag}"], out[f"distill_ref_{tag}"] = logits.astype(dtype), dist.astype(dtype)
            meta = dict(config={k: [list(p) for p in v] if k == "t2t_layers" else v for k, v in do.CASES[name].items()}, weights=gen,
                        weight_seed=do.WEIGHT_SEED, image_seed=do.IMAGE_SEED, token_seed=do.TOKEN_SEED, batch=do.BATCH,
                        generator="tests/golden/make_distill_golden.py",
                        reference="vit_tensorflow/distill.py DistillableT2TViT (unmodified) over oracle/tf_shim.py", numpy=np.__version__)
            np.savez(path, meta=json.dumps(meta), **out)
            print(f"{name} {gen}: |logits| max {np.abs(out['logits_ref_f64']).max():.3f}, "
                  f"|distill| max {np.abs(out['distill_ref_f64']).max():.3f} ({time.time() - t0:.1f} s)")


if __name__ == "__main__":
    main()

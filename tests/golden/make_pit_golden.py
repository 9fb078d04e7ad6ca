"""Golden fixtures of PiT (reference pit.py) produced by the REFERENCE'S OWN CODE running over the numpy stand-in for TensorFlow
(oracle/tf_shim.py, whose extract_patches has the VALID padding PiT's Unfold uses).

    python tests/golden/make_pit_golden.py [--force] [--reference /root/reference]

For every case of pit_oracle.SMALL (batch 2) and both weight sets (Keras' initial values, and 'stress' with every bias, beta and
gamma nonzero) this builds `pit.PiT(**kwargs)`, calls it once so that Keras builds its variables, loads the seeded weights by
attribute path, calls `model(img, training=False)` in float32 and in float64 and stores logits_ref_f32 / logits_ref_f64 in
tests/golden/<name>__<weights>__refshim.npz.  The reference checkout is absent where the GPU tests run, hence the fixtures.
"""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))
import pit_oracle as po  # noqa: E402


def main():
    ref_root = sys.argv[sys.argv.index("--reference") + 1] if "--reference" in sys.argv else "/root/reference"
    ref_dir = os.path.join(ref_root, "vit_tensorflow")
    if not os.path.isdir(ref_dir):
        raise SystemExit(f"{ref_dir} not found: these fixtures can only be generated where the reference checkout exists")
    todo = [(n, g) for n in po.SMALL for g in po.WEIGHTS
            if "--force" in sys.argv or not os.path.exists(os.path.join(HERE, po.fixture_name(n, g)))]   # never rewritten silently
    runs = {}
    for dtype, tag in ((np.float32, "f32"), (np.float64, "f64")):
        with po.reference_module(ref_dir, dtype) as mod:
            for name, gen in todo:
                cfg = po.make_config(**po.SMALL[name])
                img = po.make_image(cfg, po.BATCH, po.IMAGE_SEED)
                runs[name, gen, tag] = po.reference_logits(mod, cfg, getattr(po, gen)(cfg, po.WEIGHT_SEED), img, dtype)
    for name, gen in todo:
        meta = dict(config={k: list(v) if isinstance(v, tuple) else v for k, v in po.SMALL[name].items()}, weights=gen,
                    weight_seed=po.WEIGHT_SEED, image_seed=po.IMAGE_SEED, batch=po.BATCH, generator="tests/golden/make_pit_golden.py",
                    reference="vit_tensorflow/pit.py (unmodified) over the numpy shim", numpy=np.__version__)
        np.savez(os.path.join(HERE, po.fixture_name(name, gen)), logits_ref_f32=runs[name, gen, "f32"].astype(np.float32),
                 logits_ref_f64=runs[name, gen, "f64"].astype(np.float64), meta=json.dumps(meta))
        print(f"{name} {gen}: |logits| max {np.abs(runs[name, gen, 'f64']).max():.3f}")


if __name__ == "__main__":
    main()

"""Golden fixtures of the small-dataset ViT (reference vit_for_small_dataset.py) produced by the REFERENCE'S OWN CODE running over
the numpy stand-in for TensorFlow (oracle/tf_shim.py plus the gaps tests/small_vit_oracle.installed fills).

    python tests/golden/make_small_vit_golden.py [--force] [--reference /root/reference]

For every case of small_vit_oracle.SMALL and both weight sets (WEIGHTS: Keras' initial values, and 'stress' with every bias,
beta and gamma nonzero) this builds `vit_for_small_dataset.ViT`, calls it once so that Keras builds its variables, loads the
weights by attribute path and calls it with training=False.  Stored in tests/golden/small_vit_<name>__<weights>__refshim.npz:
logits_ref_f32 / logits_ref_f64.  The reference checkout is absent where the GPU tests run, hence the fixtures.
"""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))
import small_vit_oracle as o  # noqa: E402


def path(name, kind):
    return os.path.join(HERE, f"small_vit_{name}__{kind}__refshim.npz")


def main():
    ref_root = sys.argv[sys.argv.index("--reference") + 1] if "--reference" in sys.argv else "/root/reference"
    ref_dir = os.path.join(ref_root, "vit_tensorflow")
    if not os.path.isdir(ref_dir):
        raise SystemExit(f"{ref_dir} not found: these fixtures can only be generated where the reference checkout exists")
    todo = {n: c for n, c in o.SMALL.items() if "--force" in sys.argv or not all(os.path.exists(path(n, k)) for k in o.WEIGHTS)}
    if not todo:
        return
    runs = {tag: o.reference_run(ref_dir, todo, dt) for dt, tag in ((np.float32, "f32"), (np.float64, "f64"))}
    for name, cfg in todo.items():
        for kind in o.WEIGHTS:
            meta = dict(config=cfg, weights=kind, batch=o.BATCH, generator="tests/golden/make_small_vit_golden.py",
                        reference="vit_tensorflow/vit_for_small_dataset.py (unmodified) over the numpy shim", numpy=np.__version__)
            np.savez(path(name, kind), logits_ref_f32=runs["f32"][name, kind].astype(np.float32),
                     logits_ref_f64=runs["f64"][name, kind].astype(np.float64), meta=json.dumps(meta))
            print(f"{name} {kind}: |logits| max {np.abs(runs['f64'][name, kind]).max():.3f}")


if __name__ == "__main__":
    main()

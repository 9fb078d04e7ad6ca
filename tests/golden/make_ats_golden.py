"""Golden fixtures of ATS-ViT (reference ats_vit.py) produced by the REFERENCE'S OWN CODE running over the numpy stand-in for
TensorFlow (oracle/tf_shim.py plus the gaps tests/ats_oracle.installed fills), with tf.random.uniform returning the engine's
Philox noise (seed ats_oracle.SEED, the draw counter counting the calls).

    python tests/golden/make_ats_golden.py [--force] [--reference /root/reference]

For every case of ats_oracle.SMALL this builds `ats_vit.ViT`, calls it once so that Keras builds its variables, loads the
seeded weights by attribute path, resets the draw counter and calls `model(img, True)`.  Stored in
tests/golden/ats_<name>__refshim.npz: logits_ref_f32 / logits_ref_f64 and token_ids_f32 / token_ids_f64 (the returned ids),
noise_shapes (the [b, K, n - 1] of each sampling layer's noise), and margin: the smallest top-2 gap of any Gumbel-max draw,
computed by the float64 restatement (ats_oracle.forward), which the tests check against these logits and ids.  The reference
checkout is absent where the GPU tests run, hence the fixtures.
"""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))
import ats_oracle as o  # noqa: E402


def main():
    ref_root = sys.argv[sys.argv.index("--reference") + 1] if "--reference" in sys.argv else "/root/reference"
    ref_dir = os.path.join(ref_root, "vit_tensorflow")
    if not os.path.isdir(ref_dir):
        raise SystemExit(f"{ref_dir} not found: these fixtures can only be generated where the reference checkout exists")
    todo = {n: c for n, c in o.SMALL.items() if "--force" in sys.argv or not os.path.exists(os.path.join(HERE, f"ats_{n}__refshim.npz"))}
    if not todo:
        return
    runs = {tag: o.reference_run(ref_dir, todo, dt) for dt, tag in ((np.float32, "f32"), (np.float64, "f64"))}
    for name, cfg in todo.items():
        spec = o.forward(o.weights(cfg), o.images(cfg, o.BATCH), cfg, seed=o.SEED)
        out = {f"logits_ref_{t}": runs[t][name]["logits"].astype(np.float32 if t == "f32" else np.float64) for t in runs}
        out.update({f"token_ids_{t}": runs[t][name]["token_ids"].astype(np.int32) for t in runs})
        out["noise_shapes"] = runs["f64"][name]["noise_shapes"]
        out["margin"] = np.float64(spec["margin"])
        meta = dict(config={k: list(v) if isinstance(v, tuple) else v for k, v in cfg.items()}, batch=o.BATCH, noise_seed=o.SEED,
                    generator="tests/golden/make_ats_golden.py", reference="vit_tensorflow/ats_vit.py (unmodified) over the numpy shim",
                    numpy=np.__version__)
        out["meta"] = json.dumps(meta)
        np.savez(os.path.join(HERE, f"ats_{name}__refshim.npz"), **out)
        print(f"{name}: sampled noise {out['noise_shapes'].tolist()}, margin {spec['margin']:.4f}")


if __name__ == "__main__":
    main()

"""Golden fixtures of MAE and SimMIM (reference mae.py, simmim.py) produced by the REFERENCE'S OWN CODE running over the numpy
stand-in for TensorFlow (oracle/tf_shim.py), with tf.random.uniform returning the engine's Philox noise (tests/mim_oracle.installed).

    python tests/golden/make_mim_golden.py [--force] [--reference /root/reference]

For every case of mim_oracle.ALL_CASES and both weight variants (init, stress) this builds the reference's encoder ViT and MAE /
SimMIM, calls the wrapper once so that Keras builds its variables, binds every weight by attribute path, resets the draw counter and
calls it again, in float64 and float32.  Stored in tests/golden/<case>__<variant>__refshim.npz: loss_ref_f64 / loss_ref_f32 (the
returned loss), indices (the float64 run's argsort [b, n] for MAE, top_k ids [b, num_masked] for SimMIM; the float32 run's are
checked equal), and the first `rows` masked rows of every image of pred_ref (the float64 run's to_pixels output, stored as float32)
and masked_patches (the patches at the masked ids): all of them, or 4 for the README configurations, which keeps the files small.
noise_seed is the Philox key of the case.  The reference checkout is absent where the GPU tests run, hence the fixtures.
"""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))
import mim_oracle as o  # noqa: E402

VARIANTS = ("init", "stress")


def path(name, variant):
    return os.path.join(HERE, f"{name}__{variant}__refshim.npz")


def main():
    ref_root = sys.argv[sys.argv.index("--reference") + 1] if "--reference" in sys.argv else "/root/reference"
    ref_dir = os.path.join(ref_root, "vit_tensorflow")
    if not os.path.isdir(ref_dir):
        raise SystemExit(f"{ref_dir} not found: these fixtures can only be generated where the reference checkout exists")
    for name, (kind, cfg) in o.ALL_CASES.items():
        for variant in VARIANTS:
            if os.path.exists(path(name, variant)) and "--force" not in sys.argv:
                continue
            r64 = o.reference_run(ref_dir, name, variant, np.float64)
            r32 = o.reference_run(ref_dir, name, variant, np.float32)
            assert np.array_equal(r64["indices"], r32["indices"]), name
            rows = 4 if name.endswith("_readme") else r64["pred"].shape[1]
            out = dict(loss_ref_f64=np.float64(r64["loss"]), loss_ref_f32=np.float64(r32["loss"]), indices=r64["indices"],
                       pred_ref=r64["pred"][:, :rows].astype(np.float32), masked_patches=r64["masked_patches"][:, :rows].astype(np.float32),
                       rows=np.int64(rows), noise_seed=np.int64(o.case_seed(name)))
            meta = dict(kind=kind, config={k: list(v) if isinstance(v, tuple) else v for k, v in cfg.items()}, variant=variant,
                        batch=o.BATCH, generator="tests/golden/make_mim_golden.py",
                        reference=f"vit_tensorflow/{kind}.py (unmodified) over the numpy shim", numpy=np.__version__)
            out["meta"] = json.dumps(meta)
            np.savez_compressed(path(name, variant), **out)
            print(f"{name} {variant}: loss {r64['loss']:.6f}, num_masked {r64['pred'].shape[1]}, seed {o.case_seed(name)}")


if __name__ == "__main__":
    main()

"""Golden fixtures of training-mode dropout (include/vitb200.h, vb_set_dropout), written from the reference's own classes run
unmodified over the numpy stand-in for TensorFlow, with its Dropout drawing from the engine's Philox stream
(tests/dropout_oracle.py, philox_dropout).

    python tests/golden/make_dropout_golden.py [--force]

For every case of dropout_oracle.CASES and both weight variants (init, stress): tests/golden/dropout_<case>__<variant>__refshim.npz
with logits_d0_f64, logits_d1_f64 (float64) and logits_d0_f32, logits_d1_f32 (the reference computing in float32): the call at
draw 0 and at draw 1 of the stream keyed by `seed`.  The weights and images are regenerated from their seeds by dropout_oracle.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))
import dropout_oracle as o  # noqa: E402

REF_DIR = os.environ.get("VB_REFERENCE_DIR", "/root/reference/vit_tensorflow")


def main():
    for name in o.CASES:
        for gen in o.WEIGHTS:
            path = os.path.join(HERE, o.fixture_name(name, gen))
            if os.path.exists(path) and "--force" not in sys.argv:
                continue
            out = {}
            for d in (0, 1):
                out[f"logits_d{d}_f64"] = o.reference(REF_DIR, name, gen, d, np.float64)[0].astype(np.float64)
                out[f"logits_d{d}_f32"] = o.reference(REF_DIR, name, gen, d, np.float32)[0].astype(np.float32)
            np.savez_compressed(path, seed=np.uint64(o.SEED), meta=o.meta(name, gen), **out)
            print(f"{name} {gen}: |logits| mean {np.abs(out['logits_d0_f64']).mean():.3f}")


if __name__ == "__main__":
    main()

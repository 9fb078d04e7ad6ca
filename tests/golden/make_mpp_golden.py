"""Golden fixtures of MPP (reference mpp.py) as the engine defines it: the float64 restatement of tests/mpp_oracle.py, which the CPU
tests check against the reference's own MPP run over the numpy stand-in for TensorFlow (mask ids, coins and random ids exactly;
logits and loss with the corruption off, which is what the reference computes under TF 2).

    python tests/golden/make_mpp_golden.py [--force]

For every case of mpp_oracle.ALL_CASES and both weight variants (init, stress): tests/golden/<case>__<variant>__refshim.npz with
loss_f64 (the restatement's loss), logits (float32 [b, k, K], masked rows ascending), mask_ids [b, k], source [b, n] and noise_seed
(the Philox key of the case).  The weights and images are regenerated from their seeds by mpp_oracle.
"""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))
import mpp_oracle as o  # noqa: E402

VARIANTS = ("init", "stress")


def path(name, variant):
    return os.path.join(HERE, f"{name}__{variant}__refshim.npz")


def main():
    for name, cfg in o.ALL_CASES.items():
        for variant in VARIANTS:
            if os.path.exists(path(name, variant)) and "--force" not in sys.argv:
                continue
            s = o.spec(name, variant)
            meta = dict(config={k: list(v) if isinstance(v, tuple) else v for k, v in cfg.items()}, variant=variant,
                        generator="tests/golden/make_mpp_golden.py", numpy=np.__version__)
            np.savez_compressed(path(name, variant), loss_f64=np.float64(s["loss"]), logits=s["logits"].astype(np.float32),
                                mask_ids=s["mask_ids"], source=s["source"], noise_seed=np.int64(o.case_seed(name)), meta=json.dumps(meta))
            print(f"{name} {variant}: loss {s['loss']:.6f}, k {s['mask_ids'].shape[1]}, seed {o.case_seed(name)}")


if __name__ == "__main__":
    main()

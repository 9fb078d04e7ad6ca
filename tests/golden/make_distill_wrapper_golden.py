"""Golden fixtures of DistillWrapper (reference distill.py:87-134), written from the reference's own class run unmodified over the
numpy stand-in for TensorFlow, in float64 and in float32 (tests/distill_wrapper_oracle.py sets its token and distill_mlp).

    python tests/golden/make_distill_wrapper_golden.py [--force]

For every case of distill_wrapper_oracle.CASES and both weight variants (init, stress):
tests/golden/distill_wrapper_<case>__<variant>__refshim.npz with loss_ref_f64 and loss_ref_f32 (the returned vector [b]) and
student_logits, distill_logits, teacher_logits (float64 [b, num_classes]).  The weights, images and labels are regenerated from
their seeds by distill_wrapper_oracle.
"""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))
import distill_wrapper_oracle as o  # noqa: E402

REF_DIR = os.environ.get("VB_REFERENCE_DIR", "/root/reference/vit_tensorflow")


def main():
    for name, case in o.CASES.items():
        for gen in o.WEIGHTS:
            path = os.path.join(HERE, o.fixture_name(name, gen))
            if os.path.exists(path) and "--force" not in sys.argv:
                continue
            r64 = o.reference_wrapper(REF_DIR, name, gen, np.float64)
            r32 = o.reference_wrapper(REF_DIR, name, gen, np.float32)
            meta = dict(case=json.loads(json.dumps(case)), variant=gen, generator="tests/golden/make_distill_wrapper_golden.py",
                        numpy=np.__version__)
            np.savez_compressed(path, loss_ref_f64=r64["loss"].astype(np.float64), loss_ref_f32=r32["loss"].astype(np.float32),
                                student_logits=r64["student_logits"], distill_logits=r64["distill_logits"],
                                teacher_logits=r64["teacher_logits"], meta=json.dumps(meta))
            print(f"{name} {gen}: loss {r64['loss']}")


if __name__ == "__main__":
    main()

"""GPU parity at the BASELINE.json configurations' OWN width / depth / heads (batch 2), bf16 engine vs the oracle.

The small / mid cases of test_gpu_models.py stop at dim 256 and depth 2-4; bf16 error growth over 12-38 layers at
dim 768-1024, n = 197-577 is what this file measures and bounds.  Every case prints max|err|, the error quantiles and
|ref| statistics and asserts the per-config tolerance below.

Reference lines: vit.py:71-85,159-177 (C2, C5), deepvit.py:73-91 (C3), cait.py:107-131,180-194 (C4).
"""
import json
import os

import numpy as np
import pytest

import oracle
from oracle import ref_torch
from cases import FULL, README  # BASELINE.json configs[1..4] and the README's CrossViT / T2TViT examples, at batch 2

pytestmark = pytest.mark.gpu

# |err| <= ATOL + RTOL * |ref| on logits of standard deviation ~1 (|ref| max 2.4 - 4.3): bf16 operands and activations over
# 12-38 layers.  Rule: each bound is about 1.5-3x the largest error measured, so reordered fp32 sums pass and a wrong kernel
# does not.  Max |err| (stress / init weights) measured on an H100 80GB HBM3 (400 W limit) is in the comment of each line
# whose path is the one shipped; the DeepViT / CaiT lines run the materialised-scores head-mix path (test_gpu_models.py and
# test_gpu_ops.py bound it at smaller sizes).
CROSSVIT_README_TOL = (7.0e-2, 1.5e-2)      # 0.023 / 0.034
T2T_README_TOL = (4.5e-2, 1.0e-2)           # 0.016 / 0.017
TOL = {   # (atol, rtol)
    "c2_vit_b16_224": (4.0e-2, 1.0e-2),        # 0.027 / 0.029
    "c3_deepvit_1024x24": (6.0e-2, 2.0e-2),
    "c4_cait_s36_dh48": (7.0e-2, 2.0e-2),
    "c4_cait_s36_dh64": (9.0e-2, 2.0e-2),
    "c5_vit_l16_384": (6.0e-2, 1.5e-2),        # 0.037 / 0.033
    "crossvit_readme": CROSSVIT_README_TOL,
    "t2t_readme": T2T_README_TOL,
}


def _record(name, gen, rec):
    out = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "gpurun_out")
    if not os.path.isdir(out):
        return
    path = os.path.join(out, "config_size_parity.json")
    try:
        d = json.load(open(path))
    except (OSError, ValueError):
        d = {}
    d[f"{name}/{gen}"] = rec
    with open(path, "w") as fh:
        json.dump(d, fh, indent=1, sort_keys=True)


@pytest.mark.parametrize("gen", ["stress_weights", "init_weights"])
@pytest.mark.parametrize("name", sorted(FULL) + sorted(README))
def test_bf16_vs_oracle_at_config_size(lib, name, gen):
    from vit_tensorflow_b200 import from_config
    c = dict({**FULL, **README}[name])
    cfg = oracle.make_config(c.pop("kind"), **c)
    w = getattr(oracle, gen)(cfg, 11)
    img = oracle.make_image(cfg, 2, 12)
    m = from_config(cfg, precision="bf16")
    m.set_weights_dict(w)
    got = m(img, training=False)
    ref = ref_torch.forward(img, w, cfg).astype(np.float64)       # torch-CPU fp32 restatement (== float64 spec to 3e-6)
    assert got.shape == ref.shape == (2, 1000) and np.isfinite(got).all()
    err = np.abs(got - ref)
    atol, rtol = TOL[name]
    rec = dict(max_err=float(err.max()), p99_err=float(np.quantile(err, 0.99)), mean_err=float(err.mean()),
               ref_abs_mean=float(np.abs(ref).mean()), ref_abs_max=float(np.abs(ref).max()), ref_std=float(ref.std()),
               worst_ratio=float((err / (atol + rtol * np.abs(ref))).max()), launches=int(m.last_launch_count),
               argmax_agree=float((got.argmax(-1) == ref.argmax(-1)).mean()))
    print(f"\n[config-size parity] {name} {gen}: " + ", ".join(f"{k}={v:.4g}" for k, v in rec.items()))
    _record(name, gen, rec)
    assert (err <= atol + rtol * np.abs(ref)).all(), f"max err {err.max():.4f}, worst ratio {rec['worst_ratio']:.2f}"
    # the same bound against what the REFERENCE'S OWN CODE computed for this configuration (unmodified vit_tensorflow classes
    # over the numpy TensorFlow stand-in, float32; tests/golden/make_ref_golden.py) -- the oracle above agrees with it to 6e-6
    zr = np.load(os.path.join(os.path.dirname(__file__), "golden", f"{name}__{gen}__refshim.npz"))["logits_ref_f32"].astype(np.float64)
    assert np.abs(zr - ref).max() < 5e-5
    assert (np.abs(got - zr) <= atol + rtol * np.abs(zr)).all(), f"vs reference-code logits: max err {np.abs(got - zr).max():.4f}"

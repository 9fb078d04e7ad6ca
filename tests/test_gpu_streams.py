"""GPU: the multi-stream branches of the engine (forked / joined inside the forward, and inside its captured graph) give the
SAME bits as the single-stream forward.

  * T2T soft-split attention: images on 2 - 4 streams (engine.cu layer_t2t, VB_T2T_STREAMS)
  * CrossViT: the two towers of a multi-scale block on two streams (VB_CROSSVIT_STREAMS)
  * ViT: the batch as two half-batches on two streams (VB_FWD_STREAMS=2; off by default, kept as a measured experiment)

The switches are read once per process, so every setting runs in its own subprocess; each prints the sha256 of the logits of
three consecutive calls (eager, graph capture, graph replay) on seeded weights and images."""
import hashlib
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

CHILD = r"""
import sys, hashlib
sys.path.insert(0, %(root)r); sys.path.insert(0, %(tests)r)
import numpy as np
import oracle
from cases import cfg_of
from vit_tensorflow_b200 import from_config
cfg = cfg_of(%(case)r) if %(case)r != "vit_b128" else oracle.make_config("vit", image_size=64, patch_size=8, num_classes=50, dim=128, depth=2, heads=2, mlp_dim=256)
w = oracle.stress_weights(cfg, 3)
img = oracle.make_image(cfg, %(batch)d, 4)
m = from_config(cfg, precision="bf16")
m.set_weights_dict(w)
h = hashlib.sha256()
for _ in range(3):
    out = m(img, training=False)
    assert np.isfinite(out).all()
    h.update(out.tobytes())
print("DIGEST", h.hexdigest())
"""


def _digest(case, batch, env):
    e = dict(os.environ, **env)
    r = subprocess.run([sys.executable, "-c", CHILD % dict(root=ROOT, tests=os.path.join(ROOT, "tests"), case=case, batch=batch)],
                       env=e, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    lines = [l for l in r.stdout.splitlines() if l.startswith("DIGEST ")]
    assert lines, r.stdout[-500:]
    return lines[-1].split()[1]


@pytest.mark.parametrize("case,batch,var,values", [
    ("t2t_mid", 6, "VB_T2T_STREAMS", ("1", "2", "4")),              # n = 3136 and n = 784 soft-split layers on the tensor-core path
    ("crossvit_small", 5, "VB_CROSSVIT_STREAMS", ("1", "2")),
    ("vit_b128", 130, "VB_FWD_STREAMS", ("1", "2")),                 # 2 x 65 images: above the half-batch threshold of the split
    ("cait_small", 130, "VB_FWD_STREAMS", ("1", "2")),               # head-mixing attention: one scratch per stream
    ("deepvit_small", 130, "VB_FWD_STREAMS", ("1", "2")),
])
def test_stream_count_does_not_change_the_bits(lib, case, batch, var, values):
    digests = {v: _digest(case, batch, {var: v}) for v in values}
    assert len(set(digests.values())) == 1, digests

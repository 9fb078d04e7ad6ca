"""GPU: the multi-stream branches of the engine (forked / joined inside the forward, and inside its captured graph) give the
SAME bits as the single-stream forward.

  * T2T soft-split attention: images on 2 - 4 streams (engine.cu layer_t2t, VB_T2T_STREAMS)
  * CrossViT: the two towers of a multi-scale block on two streams (VB_CROSSVIT_STREAMS)
  * ViT: the batch as two half-batches on two streams (VB_FWD_STREAMS=2; off by default, kept as a measured experiment)

The switches are read once per process, so every setting runs in its own subprocess.  Each runs the forward of seeded weights
and images three times on a torch side stream with device buffers -- eager, graph capture, graph replay, which the child checks
through graph_stats() -- and three times eagerly on the NULL stream, and prints the sha256 of each triple of logits."""
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

CHILD = r"""
import sys, hashlib
sys.path.insert(0, %(root)r); sys.path.insert(0, %(tests)r)
import numpy as np, torch
import oracle
from cases import cfg_of
from vit_tensorflow_b200 import from_config, _lib
cfg = cfg_of(%(case)r) if %(case)r != "vit_b128" else oracle.make_config("vit", image_size=64, patch_size=8, num_classes=50, dim=128, depth=2, heads=2, mlp_dim=256)
w = oracle.stress_weights(cfg, 3)
img = oracle.make_image(cfg, %(batch)d, 4)
m = from_config(cfg, precision="bf16")
m.set_weights_dict(w)
eager = hashlib.sha256()
for _ in range(3):
    out = m(img, training=False)
    assert np.isfinite(out).all()
    eager.update(out.tobytes())
s = torch.cuda.Stream()
x = torch.from_numpy(img).cuda()
logits = torch.empty((%(batch)d, cfg["num_classes"]), device="cuda")
torch.cuda.synchronize()
st0 = m.graph_stats()
graph = hashlib.sha256()
for _ in range(3):
    m.forward_raw(x.data_ptr(), _lib.MEM_DEVICE, %(batch)d, cfg["image_h"], cfg["image_w"], logits.data_ptr(), _lib.MEM_DEVICE,
                  s.cuda_stream)
    s.synchronize()
    graph.update(logits.cpu().numpy().tobytes())
st = m.graph_stats()
delta = (st["captures"] - st0["captures"], st["replays"] - st0["replays"], st["failures"] - st0["failures"])
assert delta == (1, 1, 0), (delta, st["last_failure"])
print("DIGEST", eager.hexdigest(), graph.hexdigest())
"""


def _digests(case, batch, env):
    e = dict(os.environ, **env)
    r = subprocess.run([sys.executable, "-c", CHILD % dict(root=ROOT, tests=os.path.join(ROOT, "tests"), case=case, batch=batch)],
                       env=e, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    lines = [l for l in r.stdout.splitlines() if l.startswith("DIGEST ")]
    assert lines, r.stdout[-500:]
    return tuple(lines[-1].split()[1:])


@pytest.mark.parametrize("case,batch,var,values", [
    ("t2t_mid", 6, "VB_T2T_STREAMS", ("1", "2", "4")),              # n = 3136 and n = 784 soft-split layers on the tensor-core path
    ("crossvit_small", 5, "VB_CROSSVIT_STREAMS", ("1", "2")),
    ("vit_b128", 130, "VB_FWD_STREAMS", ("1", "2")),                 # 2 x 65 images: above the half-batch threshold of the split
    ("cait_small", 130, "VB_FWD_STREAMS", ("1", "2")),               # head-mixing attention: one scratch per stream
    ("deepvit_small", 130, "VB_FWD_STREAMS", ("1", "2")),
])
def test_stream_count_does_not_change_the_bits(lib, case, batch, var, values):
    digests = {v: _digests(case, batch, {var: v}) for v in values}
    eager, graph = {d[0] for d in digests.values()}, {d[1] for d in digests.values()}
    assert len(eager) == 1 and eager == graph, digests

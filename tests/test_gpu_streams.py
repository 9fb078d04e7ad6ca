"""GPU: the multi-stream branches of the engine (forked / joined inside the forward, and inside its captured graph) give the
SAME bits as the single-stream forward.

  * T2T soft-split attention: images on 2 - 4 streams (engine.cu layer_t2t)
  * CrossViT: the two towers of a multi-scale block on two streams

Profiling is the single-stream reference: while it is on, layer_t2t keeps one stream and CrossViT runs both towers on the
forward's own.  Each case runs the forward of seeded weights and images three times eagerly on the NULL stream, three times on
a torch side stream with device buffers -- eager, graph capture, graph replay, checked through graph_stats() -- and once under
profiling, and every one of those logits must be bit-identical."""
import numpy as np
import pytest
import torch

import oracle
from cases import cfg_of
from vit_tensorflow_b200 import _lib, from_config

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("case,batch", [
    ("t2t_mid", 6),          # n = 3136 soft-split layer on 2 streams, n = 784 on 4, both on the tensor-core path
    ("crossvit_small", 5),
])
def test_stream_count_does_not_change_the_bits(lib, case, batch):
    cfg = cfg_of(case)
    m = from_config(cfg, precision="bf16")
    m.set_weights_dict(oracle.stress_weights(cfg, 3))
    img = oracle.make_image(cfg, batch, 4)
    runs = {f"eager {i}": np.asarray(m(img, training=False)) for i in range(3)}
    assert np.isfinite(runs["eager 0"]).all()

    s = torch.cuda.Stream()
    x = torch.from_numpy(img).cuda()
    logits = torch.empty((batch, cfg["num_classes"]), device="cuda")
    torch.cuda.synchronize()
    st0 = m.graph_stats()
    for call in ("first call", "capture", "replay"):
        m.forward_raw(x.data_ptr(), _lib.MEM_DEVICE, batch, cfg["image_h"], cfg["image_w"], logits.data_ptr(), _lib.MEM_DEVICE,
                      s.cuda_stream)
        s.synchronize()
        runs[f"side stream {call}"] = logits.cpu().numpy()
    st = m.graph_stats()
    delta = (st["captures"] - st0["captures"], st["replays"] - st0["replays"], st["failures"] - st0["failures"])
    assert delta == (1, 1, 0), (delta, st["last_failure"])

    m.profile(True)
    try:
        runs["profiled"] = np.asarray(m(img, training=False))
    finally:
        m.profile(False)
    assert sum(v["launches"] for v in m.profile_read().values()) > 0

    ref = runs["eager 0"].tobytes()
    differ = [k for k, v in runs.items() if v.tobytes() != ref]
    assert not differ, f"{differ} differ from the first eager forward"

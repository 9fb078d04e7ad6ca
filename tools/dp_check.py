"""Multi-GPU check of the C-ABI data-parallel path (SURVEY.md 8e), run under torchrun on 2 / 8 GPUs:

    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29511 tools/dp_check.py

Every rank runs its shard through (a) `NativeDataParallel` (vb_dp_init + vb_forward_allgather: forward + in-place ncclAllGather
inside the library; three calls on a side stream, so that the second captures the forward into a CUDA graph and the third replays
it) and (b) `DataParallel` (torch.distributed all_gather_into_tensor); rank 0 additionally runs the WHOLE batch on its own GPU.  All three gathered logit matrices must be bit-identical on every rank (images are independent and the kernels
deterministic, tests/test_gpu_models.py::test_batch_independence_and_determinism)."""
import json
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import oracle  # noqa: E402
from vit_tensorflow_b200 import from_config  # noqa: E402
from vit_tensorflow_b200.runtime import DataParallel, NativeDataParallel, bind_to_gpu_numa, init_distributed  # noqa: E402


def main():
    node = bind_to_gpu_numa(int(os.environ.get("LOCAL_RANK", "0")))
    rank, world, local = init_distributed("nccl")
    torch.cuda.set_device(local)
    out = {}
    for name, kw, B in (("vit_mid", dict(kind="vit", image_size=224, patch_size=16, num_classes=1000, dim=256, depth=2, heads=4, mlp_dim=512), 8),
                        ("cait_small", dict(kind="cait", image_size=64, patch_size=16, num_classes=10, dim=64, depth=2, cls_depth=2, heads=4, mlp_dim=128, dim_head=16), 6)):
        kw = dict(kw)
        cfg = oracle.make_config(kw.pop("kind"), **kw)
        m = from_config(cfg, precision="bf16", device=local, seed=3)
        full = oracle.make_image(cfg, world * B, 5)
        shard = torch.from_numpy(full[rank * B:(rank + 1) * B]).cuda(local)
        h, w = cfg["image_h"], cfg["image_w"]
        a = DataParallel(m, B, (h, w), rank, world).forward_device(shard).clone()
        ndp = NativeDataParallel(m, B, (h, w), rank, world)
        # on a side stream (the default stream is never captured): eager, graph capture, then the captured CUDA graph replays in
        # front of the collective
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        st0 = m.graph_stats()
        with torch.cuda.stream(side):
            b = ndp.forward_device(shard).clone()
            b2 = ndp.forward_device(shard).clone()
            b3 = ndp.forward_device(shard).clone()
        torch.cuda.synchronize()
        st = m.graph_stats()
        graphs = dict(captures=st["captures"] - st0["captures"], replays=st["replays"] - st0["replays"],
                      failures=st["failures"] - st0["failures"])
        same = bool(torch.equal(a, b) and torch.equal(b, b2) and torch.equal(b, b3)) and graphs == dict(captures=1, replays=1, failures=0)
        if rank == 0:
            whole = m(full, training=False)
            same = same and bool(np.array_equal(whole, b.cpu().numpy()))
        flag = torch.tensor([1 if same else 0], device=f"cuda:{local}")
        dist.all_reduce(flag, op=dist.ReduceOp.MIN)
        out[name] = dict(bit_identical=bool(flag.item()), gathered_shape=list(b.shape), checksum=float(b.double().sum().item()),
                         graphs_rank0=graphs)
    if rank == 0:
        print(json.dumps(dict(world=world, numa_node_rank0=node, results=out)), flush=True)
        assert all(v["bit_identical"] for v in out.values()), out
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()

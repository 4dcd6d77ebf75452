"""Exchange-step microbenchmark: glic_p2p_allreduce_mean vs NCCL all_reduce on the cfg2 gradient payload.
Launch: python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 scripts/p2p_bench.py"""
import json
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from gaussian_lic_b200 import dist as gdist  # noqa: E402

P, M, ITERS = 500000, 15, 30
rank, world, local = (int(os.environ[k]) for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK"))
dev = torch.device("cuda", local)
torch.cuda.set_device(dev)
dist.init_process_group("nccl", device_id=dev)


def timed(fn):
    for _ in range(5):
        fn()
    torch.cuda.synchronize()
    dist.barrier()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(ITERS):
        fn()
    e1.record()
    torch.cuda.synchronize()
    t = torch.tensor([e0.elapsed_time(e1) / ITERS], device=dev)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t.item())


radii = torch.ones(P, dtype=torch.int32, device=dev)
ex = gdist.P2PGradAllReduce(P, M, dev)
ex.packed.flat.normal_()
ms_p2p = timed(lambda: ex(radii))
nc = gdist.GradAllReduce(P, M, dev)
nc.packed.flat.normal_()
ms_nccl = timed(lambda: nc(radii))
payload = ex.packed.payload_bytes()
if rank == 0:
    print(json.dumps({"world": world, "payload_bytes": payload, "p2p_ms": round(ms_p2p, 4), "nccl_ms": round(ms_nccl, 4),
                      "p2p_busbw_GBs": round(2 * (world - 1) / world * payload / ms_p2p / 1e6, 1),
                      "nccl_busbw_GBs": round(2 * (world - 1) / world * payload / ms_nccl / 1e6, 1)}))
ex.close()
dist.destroy_process_group()

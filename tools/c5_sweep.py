"""Round-2 sweep of BASELINE configs[4] (one N = 2^30 transform over all ranks, peer-memory exchange): pipelined
row-block chunks, natural and transposed output, and the N1 x N2 split.  torchrun, one rank per GPU:
    PYTHONPATH=. python -m torch.distributed.run --nproc-per-node 8 --master-addr 127.0.0.1 tools/c5_sweep.py [log2 N]
Prints one JSON line "C5SWEEP {...}" (ms per transform, max over ranks, CUDA events)."""
import json
import os
import sys

import torch
import torch.distributed as dist

import fourier_b200 as fb
from fourier_b200.distributed import CudaBackend, DistributedFft

k = int(sys.argv[1]) if len(sys.argv) > 1 else 30
rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
torch.cuda.set_device(local)
fb.set_device(local)
dist.init_process_group("nccl", device_id=torch.device("cuda", local))
be = CudaBackend("f32")


def allmax(v):
    t = torch.tensor([float(v)], device="cuda", dtype=torch.float64)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return t.item()


def timed(fn, steps=8, warmup=3):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    dist.barrier()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return allmax(e0.elapsed_time(e1) / steps)


res = {"log2n": k, "gpus": world, "ms": {}}
for k1 in (k // 2, k // 2 - 1):
    n1, n2 = 1 << k1, 1 << (k - k1)
    n = n1 * n2
    blk = n // world
    plan = DistributedFft(n1, n2, rank, world, be, exchange="peer")
    a, b = plan.buffers()
    fb.fill_input(a.view(1, blk), first_transform=rank)
    state = [a, b]

    def step(natural=True):
        out = plan.transform(state[0], state[1], natural_order=natural)
        state[0], state[1] = out, (state[0] if out is state[1] else state[1])

    for chunks in (1, 4):
        plan.chunks = chunks
        res["ms"][f"{n1}x{n2} chunks={chunks} natural"] = timed(step)
        res["ms"][f"{n1}x{n2} chunks={chunks} transposed"] = timed(lambda: step(False))
    plan.chunks = 1
    r1 = n1 // world
    res["ms"][f"{n1}x{n2} exchange only"] = timed(lambda: plan._fft_then_exchange(a, b, r1, n2, 0, True, None))
    res["ms"][f"{n1}x{n2} row FFTs of length {n1}"] = timed(lambda: be.fft_rows(a, n1, True))
    res["ms"][f"{n1}x{n2} row FFTs of length {n2}"] = timed(lambda: be.fft_rows(a, n2, True))
    plan.close()
    del a, b, state
if rank == 0:
    best = min(res["ms"].items(), key=lambda kv: kv[1] if "natural" in kv[0] else 1e9)
    res["best_natural"] = best
    print("C5SWEEP " + json.dumps(res), flush=True)
dist.destroy_process_group()

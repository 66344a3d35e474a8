"""Worker of tests/test_gpu_multirank.py: one process per GPU (launched by torch.distributed.run).

Checks, with REAL peer memory (CUDA IPC over NVLink) and real NCCL collectives between the ranks:
  * DistributedFft(exchange="peer") and ("nccl"): natural-order and transposed output against the single-GPU plan
    and against the oracle (N = 2^20);
  * the forward + inverse round trip;
  * peer mode re-entrancy (ADVICE r1): the result of call 1 is consumed while a deliberately delayed rank is still
    busy and the other ranks have already entered call 2 -- the entry barrier of transform() must keep the fast
    ranks from overwriting the slow rank's result buffer.
  * DistributedFft(exchange="fused") (row FFTs whose last stage stores into the peers) at N = 2^23;
Prints "MULTIRANK OK" on rank 0 when everything passed on every rank.
"""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import fourier_b200 as fb  # noqa: E402
from fourier_b200.distributed import CudaBackend, DistributedFft  # noqa: E402
from oracle import oracle as O  # noqa: E402

rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
torch.cuda.set_device(local)
fb.set_device(local)
dist.init_process_group("nccl", device_id=torch.device("cuda", local))

K1, K2 = 10, 10
n1, n2 = 1 << K1, 1 << K2
n = n1 * n2
blk = n // world
failures = []


def check(name, cond, detail=""):
    if not cond:
        failures.append(f"rank {rank}: {name} {detail}")


def gather(t):
    parts = [torch.empty_like(t) for _ in range(world)]
    dist.all_gather([torch.view_as_real(p) for p in parts], torch.view_as_real(t).contiguous())
    return torch.cat(parts)


# single-GPU references (every rank computes them: cheap at 2^20)
full = torch.empty(n, dtype=torch.complex64, device="cuda")
fb.fill_input(full.view(1, n))
ref = torch.empty_like(full)
fb.create_fft_f32(n).transform(full.view(1, n), ref.view(1, n), fb.Transform.Fft)
want = torch.from_numpy(O.transform(O.fill_input(1, n, np.complex64)[0], O.FFT)).cuda()
scale = float(ref.abs().max())
check("single-GPU plan vs oracle", float((ref - want).abs().max()) / scale < 1e-5)
ref_t = ref.view(n2, n1).t().contiguous().view(-1)       # Y[k1][k2] = X[k1 + n1*k2]

for mode in ("peer", "nccl"):
    plan = DistributedFft(n1, n2, rank, world, CudaBackend("f32"), exchange=mode)
    x, scratch = plan.buffers()
    mine = full[rank * blk:(rank + 1) * blk]
    for natural in (True, False):
        x.copy_(mine)
        out = plan.transform(x, scratch, natural_order=natural)
        got = gather(out)
        target = ref if natural else ref_t
        err = float((got - target).abs().max()) / scale
        check(f"{mode} natural={natural} vs single-GPU plan", err < 1e-5, f"rel err {err:.3e}")
        err_o = float((got - (want if natural else want.view(n2, n1).t().contiguous().view(-1))).abs().max()) / scale
        check(f"{mode} natural={natural} vs oracle", err_o < 1e-5, f"rel err {err_o:.3e}")
    # forward + inverse round trip
    x.copy_(mine)
    out = plan.transform(x, scratch)
    back = plan.transform(out, x if out is scratch else scratch, forward=False) / n
    rt = float((back - mine).abs().max())
    check(f"{mode} round trip", rt < 1e-4, f"abs err {rt:.3e}")
    if mode == "peer":
        # re-entrancy: rank 0 is slow to consume its result; the others rush into the next call
        x.copy_(mine)
        out1 = plan.transform(x, scratch)
        if rank == 0:
            torch.cuda._sleep(int(2e8))                      # ~0.1 s of GPU time on rank 0's stream
        kept = out1.clone()                                  # the consumer of call 1 (stream-ordered)
        other = x if out1 is scratch else scratch
        other.copy_(mine)                                    # next input (same signal), then call 2 right away
        out2 = plan.transform(other, out1)
        torch.cuda.synchronize()
        got1 = gather(kept)
        err = float((got1 - ref).abs().max()) / scale
        check("peer re-entrancy: result of call 1 intact on a delayed rank", err < 1e-5, f"rel err {err:.3e}")
        err2 = float((gather(out2) - ref).abs().max()) / scale
        check("peer re-entrancy: call 2", err2 < 1e-5, f"rel err {err2:.3e}")
    plan.close()

# the exchange of each row block overlapping the FFTs of the next, with real peers
plan = DistributedFft(n1, n2, rank, world, CudaBackend("f32"), exchange="peer", chunks=4)
x, scratch = plan.buffers()
x.copy_(full[rank * blk:(rank + 1) * blk])
err = float((gather(plan.transform(x, scratch)) - ref).abs().max()) / scale
check("peer, 4 pipelined chunks", err < 1e-5, f"rel err {err:.3e}")
plan.close()

# exchange="fused": the exchanges after the row FFTs are folded into the FFTs' last stage (csrc/dist_kernels.cuh);
# needs two-pass row lengths, so N = 2^11 x 2^12 here; natural and transposed output, round trip, against the
# single-GPU plan of 2^23 points and the stand-alone exchange kernel
f1, f2 = 1 << 11, 1 << 12
fn = f1 * f2
fblk = fn // world
ffull = torch.empty(fn, dtype=torch.complex64, device="cuda")
fb.fill_input(ffull.view(1, fn))
fref = torch.empty_like(ffull)
fb.create_fft_f32(fn).transform(ffull.view(1, fn), fref.view(1, fn), fb.Transform.Fft)
fscale = float(fref.abs().max())
fref_t = fref.view(f2, f1).t().contiguous().view(-1)
results = {}
for mode in ("fused", "peer"):
    be = CudaBackend("f32")
    plan = DistributedFft(f1, f2, rank, world, be, exchange=mode)
    x, scratch = plan.buffers()
    if mode == "fused":
        check("fused mode is taken", plan.fused and be.can_fuse(x, f1, f2 // world) and be.can_fuse(x, f2, f1 // world))
    mine = ffull[rank * fblk:(rank + 1) * fblk]
    for natural in (True, False):
        x.copy_(mine)
        got = gather(plan.transform(x, scratch, natural_order=natural))
        err = float((got - (fref if natural else fref_t)).abs().max()) / fscale
        check(f"{mode} 2^23 natural={natural} vs single-GPU plan", err < 1e-5, f"rel err {err:.3e}")
        results[(mode, natural)] = got
    x.copy_(mine)
    out = plan.transform(x, scratch)
    back = plan.transform(out, x if out is scratch else scratch, forward=False) / fn
    rt = float((back - mine).abs().max())
    check(f"{mode} 2^23 round trip", rt < 1e-4, f"abs err {rt:.3e}")
    plan.close()
for natural in (True, False):
    d = float((results[("fused", natural)] - results[("peer", natural)]).abs().max()) / fscale
    check(f"fused vs peer natural={natural}", d < 2e-6, f"rel diff {d:.3e}")

bad = torch.tensor([len(failures)], device="cuda")
dist.all_reduce(bad)
for f in failures:
    print("FAILED:", f, flush=True)
if rank == 0:
    print("MULTIRANK OK" if int(bad.item()) == 0 else f"MULTIRANK FAILED ({int(bad.item())} checks)", flush=True)
dist.destroy_process_group()
sys.exit(0 if not failures else 1)

"""Runs one batched transform with FOURIER_B200_TRACE set (phase timestamps of CTA 0 of the fused kernel) and prints
where the tile period goes: median and 90th percentile of each phase, in cycles and as a share of the median tile period.
usage: PYTHONPATH=. FOURIER_B200_TRACE=out.txt [FOURIER_B200_TRACE_FROM=k] python tools/trace_run.py [f32|f64] [log2 N] [batch]
       python tools/trace_run.py --read out.txt          (summarise an existing trace file)
The kernel records 64 tiles per warp, from tile FOURIER_B200_TRACE_FROM (default 0: the start of the queue, where the
ring and lag dependencies act differently); set it to about half the tiles per group for a steady-state window.

Trace file: one line per (warp row w, tile k): `w k t0 .. t7` (csrc/twopass.cu).  Consumer warps: t0 loop start,
t1 `full` landed, t2 samples in registers and staging released, t3 stage A done (the group's first warp: and the
exchange lock taken), t4 scattered, t5 gathered (and the lock released), t6 stage B and stores issued; t7 of a group's
first warp = the tile's pass.  Producer lanes (rows after the consumer warps, one per group): t0 iteration start,
t1 dependencies met, t2 the group's `empty` landed, t3 tile issued; a phase lasts from the previous timestamp in
time order to its own, so the table holds whichever order the producer loop takes them in."""
import os
import sys

import numpy as np

SKIP = 4   # first tiles of each warp: start-up, not steady state


def load(path):
    rows = np.loadtxt(path, dtype=np.int64, ndmin=2)
    nw, nk = int(rows[:, 0].max()) + 1, int(rows[:, 1].max()) + 1
    t = np.zeros((nw, nk, 8), dtype=np.int64)
    t[rows[:, 0], rows[:, 1]] = rows[:, 2:]
    return t


def stats(x, period):
    x = np.asarray(x, dtype=np.float64)
    if x.size == 0:
        return "      --"
    med, p90 = np.median(x), np.percentile(x, 90)
    return f"{med:8.0f} {p90:8.0f}   {100 * med / period:5.1f} %"


def summarise(t):
    used = (t[:, :, :7] != 0).any(axis=(1, 2))
    consumer = [w for w in range(t.shape[0]) if used[w] and (t[w, :, 6] != 0).any()]
    producer = [w for w in range(t.shape[0]) if used[w] and w not in consumer]
    leaders = [w for w in consumer if (t[w, :, 7] != 0).any()]
    group_of = {w: max(i for i, l in enumerate(leaders) if l <= w) for w in consumer}
    print(f"{len(leaders)} consumer groups, {len(consumer)} consumer warps, {len(producer)} producer lanes (CTA 0)")

    def valid(w, k, phases):
        return all(t[w, k, p] != 0 for p in phases)

    periods = [t[l, k + 1, 0] - t[l, k, 0] for l in leaders for k in range(SKIP, t.shape[1] - 1)
               if valid(l, k, (0,)) and valid(l, k + 1, (0,))]
    period = float(np.median(periods))
    print(f"tile period of a group: median {period:.0f} cycles, p90 {np.percentile(periods, 90):.0f}\n")
    print(f"{'phase':34s} {'median':>8s} {'p90':>8s}   of period")

    ph = {name: [] for name in ("wait on full", "load + release", "stage A", "lock wait", "exchange", "stage B + store")}
    for w in consumer:
        for k in range(SKIP, t.shape[1]):
            if not valid(w, k, range(7)):
                continue
            r = t[w, k]
            ph["wait on full"].append(r[1] - r[0])
            ph["load + release"].append(r[2] - r[1])
            ph["exchange"].append(r[5] - r[3])
            ph["stage B + store"].append(r[6] - r[5])
            if w in leaders:
                # the first warp takes the lock between stage A and t3: its excess over the group's other warps
                others = [t[o, k, 3] - t[o, k, 2] for o in consumer
                          if o != w and group_of[o] == group_of[w] and valid(o, k, (2, 3))]
                sa = float(np.median(others)) if others else 0.0
                ph["lock wait"].append(max(0.0, (r[3] - r[2]) - sa))
            else:
                ph["stage A"].append(r[3] - r[2])
    print("consumer warps")
    for name, x in ph.items():
        print(f"  {name:32s} {stats(x, period)}")

    names = {1: "claim + dependency wait", 2: "empty wait", 3: "issue"}
    pp = {i: [] for i in names}
    for w in producer:
        for k in range(SKIP, t.shape[1]):
            if not valid(w, k, range(4)):
                continue
            order = sorted(range(4), key=lambda i: t[w, k, i])
            for j in range(1, 4):
                pp[order[j]].append(t[w, k, order[j]] - t[w, k, order[j - 1]])
    print("producer lanes")
    for i, name in names.items():
        print(f"  {name:32s} {stats(pp[i], period)}")


if __name__ == "__main__":
    if len(sys.argv) > 2 and sys.argv[1] == "--read":
        summarise(load(sys.argv[2]))
        sys.exit(0)
    import torch
    import fourier_b200 as fb

    real = sys.argv[1] if len(sys.argv) > 1 else "f32"
    k = int(sys.argv[2]) if len(sys.argv) > 2 else (20 if real == "f32" else 16)
    batch = int(sys.argv[3]) if len(sys.argv) > 3 else (256 if real == "f32" else 4096)
    p = fb.create_fft_f32(1 << k) if real == "f32" else fb.create_fft_f64(1 << k)
    dt = torch.complex64 if real == "f32" else torch.complex128
    x = torch.empty((batch, 1 << k), dtype=dt, device="cuda")
    fb.fill_input(x)
    y = torch.empty_like(x)
    for _ in range(2):   # the second call's trace is kept: warm caches and module load
        p.transform(x, y, fb.Transform.Fft)
    torch.cuda.synchronize()
    print(p.info())
    print({k: v for k, v in os.environ.items() if k.startswith("FOURIER_B200")})
    n1, n2 = p.info()["n1"], p.info()["n2"]
    per_cta = batch * (n1 + n2) / 8 / torch.cuda.get_device_properties(0).multi_processor_count
    start = int(os.environ.get("FOURIER_B200_TRACE_FROM", "0"))
    print(f"window: tiles {start + SKIP} .. {start + 63} of each warp of CTA 0; the CTA's groups share about "
          f"{per_cta:.0f} tiles")
    summarise(load(os.environ["FOURIER_B200_TRACE"]))

"""How fast HBM serves the access pattern of the persistent two-pass kernel at f32 2^20, without the FFT: compiles
tools/hbm_pattern.cu (nvcc, sm_90a, into a temporary directory), runs its tile copies of a batch of 1024 x 1024
complex-f32 transforms and a contiguous device copy of the same bytes, alternated over rounds, and prints the card, a
table of GB/s (bytes read + bytes written over time) with the spread over the rounds, and one JSON line.

    python tools/hbm_pattern_bench.py [--batch 4096] [--rounds 5]

Variants (see hbm_pattern.cu): group8 = one 8-column tile per group, 64-byte pieces (the kernel today); pair16 = two
adjacent tiles per CTA, loaded as 16-column boxes (128-byte lines) and stored by both groups at once; pair8 = the same
pairs loaded as 8-column boxes; contiguous = cudaMemcpy device to device, the ceiling.
"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def card():
    out = {"name": "unknown", "power_limit": "unknown", "sm_clock_max": "unknown"}
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        if r.returncode == 0 and r.stdout.strip():
            out["name"], out["power_limit"], out["sm_clock_max"] = [v.strip() for v in r.stdout.strip().split(",")[:3]]
    except (OSError, subprocess.SubprocessError):
        pass
    return out


def build(tmp):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    exe = os.path.join(tmp, "hbm_pattern")
    csrc = os.path.join(ROOT, "fourier_b200", "csrc")
    subprocess.run([nvcc, "-std=c++17", "-O3", "--expt-relaxed-constexpr", "-gencode", "arch=compute_90a,code=sm_90a",
                    "-I", csrc, os.path.join(ROOT, "tools", "hbm_pattern.cu"), "-o", exe], check=True)
    return exe


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=4096)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    with tempfile.TemporaryDirectory() as tmp:
        exe = build(tmp)
        info = card()
        print(f"card: {info['name']}, power limit {info['power_limit']}, max SM clock {info['sm_clock_max']}", flush=True)
        r = subprocess.run([exe, str(args.batch), str(args.rounds)], capture_output=True, text=True)
    sys.stdout.write(r.stdout)
    if r.returncode != 0:
        sys.stderr.write(r.stderr)
        raise SystemExit(f"hbm_pattern failed with exit code {r.returncode}")
    times = {}
    for line in r.stdout.splitlines():
        f = line.split()
        if f and f[0] == "time":
            times.setdefault(f[1], []).append(float(f[3]))
    moved = 2 * args.batch * (1 << 20) * 8   # every byte read once and written once
    rows = {}
    print(f"\n{'variant':12s} {'ms median':>10s} {'GB/s median':>12s} {'GB/s range':>16s}")
    for name, ms in times.items():
        gbs = sorted(moved / (t * 1e-3) / 1e9 for t in ms)
        med = sorted(ms)[len(ms) // 2]
        rows[name] = {"ms": ms, "ms_median": med, "gb_per_s_median": round(moved / (med * 1e-3) / 1e9, 1),
                      "gb_per_s_min": round(gbs[0], 1), "gb_per_s_max": round(gbs[-1], 1)}
        print(f"{name:12s} {med:10.3f} {rows[name]['gb_per_s_median']:12.1f} {gbs[0]:7.1f} - {gbs[-1]:7.1f}")
    print(json.dumps({"card": info, "batch": args.batch, "rounds": args.rounds, "bytes_moved": moved, "variants": rows}))


if __name__ == "__main__":
    main()

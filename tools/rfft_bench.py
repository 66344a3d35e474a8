"""Times device-resident real-input transforms (RealFft) next to the complex plan of the same length N at the same
batch, with CUDA events: warm-up, then rounds of back-to-back calls, median round.  Prints the card, its power limit
and SM clock (before and after the timed runs), a table, and one JSON line.

    python tools/rfft_bench.py [--calls 10] [--rounds 5]

Algorithmic bytes per row: forward f32 reads 4N and writes 8(N/2+1) (f64 twice that), the inverse the other way
round; the complex plan reads and writes N complex values.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

# (precision, N, batch): the complex plan of each case holds 2 GB of input
CASES = [("f32", 2048, 1 << 17), ("f32", 1 << 21, 128), ("f64", 512, 1 << 18), ("f64", 1 << 17, 1024)]


def card():
    import torch
    out = {"name": torch.cuda.get_device_name(0), "power_limit": "unknown", "sm_clock": "unknown"}
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        if r.returncode == 0 and r.stdout.strip():
            out["power_limit"], out["sm_clock"] = [v.strip() for v in r.stdout.strip().split(",")[:2]]
    except (OSError, subprocess.SubprocessError):
        pass
    return out


def time_calls(fn, calls, rounds):
    import torch
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(rounds):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(calls):
            fn()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b) / calls)
    return sorted(times)[len(times) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    import torch
    import fourier_b200 as fb
    if not torch.cuda.is_available():
        raise SystemExit("rfft_bench.py needs a CUDA device")
    info = card()
    print(f"card: {info['name']}, power limit {info['power_limit']}, SM clock {info['sm_clock']}")
    results = []
    for prec, n, batch in CASES:
        rdt, cdt = (torch.float32, torch.complex64) if prec == "f32" else (torch.float64, torch.complex128)
        rb = 4 if prec == "f32" else 8
        bins = n // 2 + 1
        real = fb.create_rfft_f32(n) if prec == "f32" else fb.create_rfft_f64(n)
        cplx = fb.create_fft_f32(n) if prec == "f32" else fb.create_fft_f64(n)
        x = torch.randn((batch, n), dtype=rdt, device="cuda")
        X = torch.empty((batch, bins), dtype=cdt, device="cuda")
        y = torch.empty_like(x)
        row = {"precision": prec, "n": n, "batch": batch, "real_path": real.info()["path_name"],
               "inner_path": real.info()["inner_path_name"], "complex_path": cplx.info()["path_name"]}
        ms_f = time_calls(lambda: real.rfft(x, X), args.calls, args.rounds)
        ms_i = time_calls(lambda: real.irfft(X, y), args.calls, args.rounds)
        launches = real.info()["last_launches"]
        del y
        z = torch.empty((batch, n), dtype=cdt, device="cuda")
        z.real.copy_(x)
        zo = torch.empty_like(z)
        del x, X
        ms_c = time_calls(lambda: cplx.transform(z, zo, fb.Transform.Fft), args.calls, args.rounds)
        del z, zo
        spec_bytes = bins * 2 * rb
        real_bytes = batch * (n * rb + spec_bytes)
        cplx_bytes = batch * 2 * n * 2 * rb
        for name, ms, nbytes in (("rfft", ms_f, real_bytes), ("irfft", ms_i, real_bytes), ("complex_fft", ms_c, cplx_bytes)):
            row[name] = {"ms_per_call": round(ms, 4), "samples_per_s": float(f"{batch * n / (ms * 1e-3):.4g}"),
                         "gb_per_s": round(nbytes / (ms * 1e-3) / 1e9, 1)}
        row["real_launches"] = launches
        row["rfft_speedup_vs_complex"] = round(ms_c / ms_f, 3)
        results.append(row)
        print(f"{prec} N={n} batch={batch} [{row['real_path']}/{row['inner_path']} vs {row['complex_path']}]: "
              f"rfft {ms_f:.3f} ms ({row['rfft']['gb_per_s']} GB/s), irfft {ms_i:.3f} ms ({row['irfft']['gb_per_s']} GB/s), "
              f"complex {ms_c:.3f} ms ({row['complex_fft']['gb_per_s']} GB/s)", flush=True)
        real.close()
        cplx.close()
        torch.cuda.empty_cache()
    info["sm_clock_after"] = card()["sm_clock"]
    print(f"SM clock after the timed runs: {info['sm_clock_after']}")
    print(json.dumps({"card": info, "calls_per_round": args.calls, "rounds": args.rounds, "results": results}))


if __name__ == "__main__":
    main()

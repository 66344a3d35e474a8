"""Times the analytic signal and envelope of real rows on device buffers: RealFft.hilbert and RealFft.envelope next to
the compositions a PyTorch caller would otherwise write, and next to the plan's rfft alone:
  * "composition": the same plan's convolve(x, G) for y, then torch.complex(x, y) (torch.hypot(x, y) for the envelope);
  * "torch": scipy's method on torch.fft: fft, times h (1 at bins 0 and N/2, 2 between, 0 above), ifft (then .abs());
  * "rfft": the plan's rfft alone: the same N reals in, N/2+1 complex values out.
CUDA events: warm-up, then rounds of back-to-back calls; the median round is reported with the fastest and slowest.
Prints the card, its power limit and SM clock (before and after the timed runs), one line per case, and one JSON line.

    python tools/hilbert_bench.py [--calls 5] [--rounds 5]

Algorithmic bytes per row: N reals in and N complex values out (analytic), or N reals in and N reals out (envelope).
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from mel_bench import time_rounds  # noqa: E402
from rfft_bench import card  # noqa: E402

# (precision, N, rows): the fused path at f32 N = 1024, 2048 and f64 N = 512, real_half at f32 N = 4096; 256 MB of input
# per call
CASES = [("f32", 1024, 1 << 16), ("f32", 2048, 1 << 15), ("f32", 4096, 1 << 14), ("f64", 512, 1 << 16)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    import torch
    import fourier_b200 as fb
    if not torch.cuda.is_available():
        raise SystemExit("hilbert_bench.py needs a CUDA device")
    info = card()
    print(f"card: {info['name']}, power limit {info['power_limit']}, SM clock {info['sm_clock']}")
    results = []
    for prec, n, rows in CASES:
        rdt = torch.float32 if prec == "f32" else torch.float64
        cdt = torch.complex64 if prec == "f32" else torch.complex128
        rb = 4 if prec == "f32" else 8
        plan = fb.create_rfft_f32(n) if prec == "f32" else fb.create_rfft_f64(n)
        g = torch.Generator(device="cuda").manual_seed(n)
        x = torch.randn((rows, n), dtype=rdt, device="cuda", generator=g)
        z = torch.empty((rows, n), dtype=cdt, device="cuda")
        e = torch.empty_like(x)
        y = torch.empty_like(x)
        V = torch.empty((rows, n // 2 + 1), dtype=cdt, device="cuda")
        G = torch.full((n // 2 + 1,), -1j, dtype=cdt, device="cuda")
        G[0] = 0
        G[n // 2] = 0
        h = torch.zeros(n, dtype=rdt, device="cuda")
        h[0] = h[n // 2] = 1
        h[1:n // 2] = 2
        row = {"precision": prec, "n": n, "rows": rows, "path": plan.info()["path_name"]}

        def comp_z():
            plan.convolve(x, G, y)
            return torch.complex(x, y)

        def comp_e():
            plan.convolve(x, G, y)
            return torch.hypot(x, y)

        def torch_z():
            return torch.fft.ifft(torch.fft.fft(x) * h)

        t = {"hilbert": time_rounds(lambda: plan.hilbert(x, z), args.calls, args.rounds)}
        row["launches_hilbert"] = plan.info()["last_launches"]
        t["envelope"] = time_rounds(lambda: plan.envelope(x, e), args.calls, args.rounds)
        row["launches_envelope"] = plan.info()["last_launches"]
        t["composition_hilbert"] = time_rounds(comp_z, args.calls, args.rounds)
        t["composition_envelope"] = time_rounds(comp_e, args.calls, args.rounds)
        t["torch_hilbert"] = time_rounds(torch_z, args.calls, args.rounds)
        t["torch_envelope"] = time_rounds(lambda: torch_z().abs(), args.calls, args.rounds)
        t["rfft"] = time_rounds(lambda: plan.rfft(x, V), args.calls, args.rounds)
        plan.hilbert(x, z)
        plan.envelope(x, e)
        ref_z, ref_e = comp_z(), comp_e()
        torch.cuda.synchronize()
        row["max_rel_diff_hilbert_vs_composition"] = float(
            f"{float(((z - ref_z).abs().amax(-1) / ref_z.abs().amax(-1)).max()):.3e}")
        row["max_rel_diff_envelope_vs_composition"] = float(
            f"{float(((e - ref_e).abs().amax(-1) / ref_e.abs().amax(-1)).max()):.3e}")
        del ref_z, ref_e
        nbytes = {"hilbert": 3 * rows * n * rb, "envelope": 2 * rows * n * rb, "rfft": rows * (n + 2 * (n // 2 + 1)) * rb}
        for name, ts in t.items():
            ms = ts[len(ts) // 2]
            b = nbytes["rfft" if name == "rfft" else "envelope" if name.endswith("envelope") else "hilbert"]
            row[name] = {"ms_per_call": round(ms, 4), "ms_min": round(ts[0], 4), "ms_max": round(ts[-1], 4),
                         "gb_per_s": round(b / (ms * 1e-3) / 1e9, 1)}
        for op in ("hilbert", "envelope"):
            d = row[op]["ms_per_call"]
            row[f"speedup_{op}_vs_composition"] = round(row[f"composition_{op}"]["ms_per_call"] / d, 3)
            row[f"speedup_{op}_vs_torch"] = round(row[f"torch_{op}"]["ms_per_call"] / d, 3)
            row[f"{op}_over_rfft"] = round(d / row["rfft"]["ms_per_call"], 3)
        results.append(row)
        line = f"{prec} N={n} rows={rows} [{row['path']}]:"
        for op in ("hilbert", "envelope"):
            a, c, tt = t[op], t[f"composition_{op}"], t[f"torch_{op}"]
            line += (f" {op} {a[len(a) // 2]:.3f} ms [{a[0]:.3f}, {a[-1]:.3f}] ({row[op]['gb_per_s']} GB/s), "
                     f"composition {c[len(c) // 2]:.3f} [{c[0]:.3f}, {c[-1]:.3f}], torch {tt[len(tt) // 2]:.3f} "
                     f"[{tt[0]:.3f}, {tt[-1]:.3f}];")
        r = t["rfft"]
        line += f" rfft alone {r[len(r) // 2]:.3f} ms [{r[0]:.3f}, {r[-1]:.3f}]"
        print(line, flush=True)
        del x, z, e, y, V
        plan.close()
        torch.cuda.empty_cache()
    info["sm_clock_after"] = card()["sm_clock"]
    print(f"SM clock after the timed runs: {info['sm_clock_after']}")
    print(json.dumps({"card": info, "calls_per_round": args.calls, "rounds": args.rounds, "results": results}))


if __name__ == "__main__":
    main()

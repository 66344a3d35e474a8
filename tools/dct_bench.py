"""Times the discrete cosine transforms of real rows on device buffers: RealFft.dct (types 2 and 3, norm backward) next
to the compositions a PyTorch caller would otherwise write, and next to the plan's rfft alone.  Compositions (Makhoul's
algorithm, as in the header's definition):
  * "composition": torch reorder (or twiddle), the same plan's rfft (type 2) or irfft (type 3), then the twiddle and the
    assembly (or the reorder back) in torch;
  * "torch": the same composition on torch.fft.rfft / irfft;
  * "rfft": the plan's rfft alone: the same N reals in, N/2+1 complex values out.
CUDA events: warm-up, then rounds of back-to-back calls; the median round is reported with the fastest and slowest.
Prints the card, its power limit and SM clock (before and after the timed runs), one line per case, and one JSON line.

    python tools/dct_bench.py [--calls 5] [--rounds 5]

Algorithmic bytes of a dct: N reals in and N reals out per row.
"""
import argparse
import json
import math
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from mel_bench import time_rounds  # noqa: E402
from rfft_bench import card  # noqa: E402

# (precision, N, rows): the fused path at three sizes and real_half at two, each moving at least 256 MB per call
CASES = [("f32", 512, 1 << 16), ("f32", 2048, 1 << 14), ("f64", 512, 1 << 15), ("f32", 400, 84000),
         ("f32", 4096, 1 << 13)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    import torch
    import fourier_b200 as fb
    if not torch.cuda.is_available():
        raise SystemExit("dct_bench.py needs a CUDA device")
    info = card()
    print(f"card: {info['name']}, power limit {info['power_limit']}, SM clock {info['sm_clock']}")
    results = []
    for prec, n, rows in CASES:
        rdt = torch.float32 if prec == "f32" else torch.float64
        cdt = torch.complex64 if prec == "f32" else torch.complex128
        rb = 4 if prec == "f32" else 8
        half = n // 2
        plan = fb.create_rfft_f32(n) if prec == "f32" else fb.create_rfft_f64(n)
        g = torch.Generator(device="cuda").manual_seed(n)
        x = torch.randn((rows, n), dtype=rdt, device="cuda", generator=g)
        y = torch.empty_like(x)
        V = torch.empty((rows, half + 1), dtype=cdt, device="cuda")
        u = torch.empty_like(x)
        k = torch.arange(half + 1, device="cuda", dtype=torch.float64)
        W = torch.polar(torch.ones_like(k), -math.pi * k / (2 * n)).to(cdt)
        row = {"precision": prec, "n": n, "rows": rows, "path": plan.info()["path_name"]}

        def reorder(x):
            return torch.cat((x[..., ::2], x[..., 1::2].flip(-1)), -1)

        def assemble(X):
            Y = X * W
            return torch.cat((2 * Y.real, (-2 * Y.imag[..., 1:half]).flip(-1)), -1)

        def pre3(x):
            xr = torch.cat((torch.zeros_like(x[..., :1]), x[..., half:].flip(-1)), -1)
            return W.conj() * torch.complex(x[..., :half + 1], -xr)

        def back3(v):
            return torch.stack((v[..., :half], v[..., half:].flip(-1)), -1).reshape(v.shape)

        def comp2():
            plan.rfft(reorder(x), V)
            return assemble(V)

        def comp3():
            plan.irfft(pre3(x), u, fb.Transform.UnscaledIfft)
            return back3(u)

        def torch2():
            return assemble(torch.fft.rfft(reorder(x)))

        def torch3():
            return back3(torch.fft.irfft(pre3(x), n=n) * n)

        t = {}
        diffs = {}
        for typ, comp, tc in ((2, comp2, torch2), (3, comp3, torch3)):
            t[f"dct{typ}"] = time_rounds(lambda: plan.dct(x, y, type=typ), args.calls, args.rounds)
            launches = plan.info()["last_launches"]
            t[f"composition{typ}"] = time_rounds(comp, args.calls, args.rounds)
            t[f"torch{typ}"] = time_rounds(tc, args.calls, args.rounds)
            plan.dct(x, y, type=typ)
            ref = comp()
            torch.cuda.synchronize()
            diffs[typ] = float(((y - ref).abs().amax(-1) / ref.abs().amax(-1)).max())
            row[f"launches_dct{typ}"] = launches
            del ref
        t["rfft"] = time_rounds(lambda: plan.rfft(x, V), args.calls, args.rounds)
        nbytes = 2 * rows * n * rb
        for name, ts in t.items():
            ms = ts[len(ts) // 2]
            row[name] = {"ms_per_call": round(ms, 4), "ms_min": round(ts[0], 4), "ms_max": round(ts[-1], 4),
                         "gb_per_s": round((nbytes if name != "rfft" else rows * (n + 2 * (half + 1)) * rb)
                                           / (ms * 1e-3) / 1e9, 1)}
        row["algorithmic_bytes"] = nbytes
        for typ in (2, 3):
            d = row[f"dct{typ}"]["ms_per_call"]
            row[f"speedup{typ}_vs_composition"] = round(row[f"composition{typ}"]["ms_per_call"] / d, 3)
            row[f"speedup{typ}_vs_torch"] = round(row[f"torch{typ}"]["ms_per_call"] / d, 3)
            row[f"dct{typ}_over_rfft"] = round(d / row["rfft"]["ms_per_call"], 3)
            row[f"max_rel_diff{typ}_vs_composition"] = float(f"{diffs[typ]:.3e}")
        results.append(row)
        line = f"{prec} N={n} rows={rows} [{row['path']}]:"
        for typ in (2, 3):
            a, c, tt = t[f"dct{typ}"], t[f"composition{typ}"], t[f"torch{typ}"]
            line += (f" dct{typ} {a[len(a) // 2]:.3f} ms [{a[0]:.3f}, {a[-1]:.3f}] ({row[f'dct{typ}']['gb_per_s']} GB/s), "
                     f"composition {c[len(c) // 2]:.3f} [{c[0]:.3f}, {c[-1]:.3f}], torch {tt[len(tt) // 2]:.3f} "
                     f"[{tt[0]:.3f}, {tt[-1]:.3f}], diff {diffs[typ]:.1e};")
        r = t["rfft"]
        line += f" rfft alone {r[len(r) // 2]:.3f} ms [{r[0]:.3f}, {r[-1]:.3f}]"
        print(line, flush=True)
        del x, y, V, u
        plan.close()
        torch.cuda.empty_cache()
    info["sm_clock_after"] = card()["sm_clock"]
    print(f"SM clock after the timed runs: {info['sm_clock_after']}")
    print(json.dumps({"card": info, "calls_per_round": args.calls, "rounds": args.rounds, "results": results}))


if __name__ == "__main__":
    main()

"""Times the linear convolution of long real rows by overlap-save on device buffers: RealFft.convolve_linear next to the
caller-side composition on the same plan (F.pad + unfold into a contiguous (batch * G, N) tensor of segments,
RealFft.convolve in place, drop the first K-1 samples of each segment, crop and copy into y) and, as an informative
column only, torch.fft.irfft(rfft(x, n) * rfft(h, n)) at a power of two n >= L + K - 1.  CUDA events: warm-up, then
rounds of back-to-back calls, median round.  Prints the card, its power limit and SM clock (before and after the timed
runs), one line per case, and one JSON line.

    python tools/lconv_bench.py [--calls 5] [--rounds 5]

Algorithmic bytes: in_len + out_len reals per row plus the F spectra once, for every column (what the job needs).
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from rfft_bench import card, time_calls  # noqa: E402

# (precision, N, K, rows, L, F), mode full: long rows filtered with one filter, or one filter per row
CASES = [("f32", 2048, 129, 64, 1 << 22, 1), ("f32", 2048, 129, 64, 1 << 22, 64), ("f32", 2048, 1025, 64, 1 << 22, 1),
         ("f64", 512, 65, 64, 1 << 21, 1), ("f64", 512, 65, 64, 1 << 21, 64)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    import torch
    import torch.nn.functional as F_
    import fourier_b200 as fb
    if not torch.cuda.is_available():
        raise SystemExit("lconv_bench.py needs a CUDA device")
    info = card()
    print(f"card: {info['name']}, power limit {info['power_limit']}, SM clock {info['sm_clock']}")
    results = []
    for prec, n, k, rows, length, F in CASES:
        rdt = torch.float32 if prec == "f32" else torch.float64
        rb = 4 if prec == "f32" else 8
        bins = n // 2 + 1
        s = n - k + 1
        out_len = length + k - 1
        G = -(-out_len // s)
        plan = fb.create_rfft_f32(n) if prec == "f32" else fb.create_rfft_f64(n)
        g = torch.Generator(device="cuda").manual_seed(n + k + F)
        x = torch.randn((rows, length), dtype=rdt, device="cuda", generator=g)
        h = torch.randn((F, k), dtype=rdt, device="cuda", generator=g)
        H = torch.fft.rfft(h, n=n)          # (F, bins), in the plan's layout
        Hs = H[0].contiguous() if F == 1 else H.contiguous()
        y = torch.empty((rows, out_len), dtype=rdt, device="cuda")
        row = {"precision": prec, "n": n, "taps": k, "rows": rows, "in_len": length, "filters": F, "mode": "full",
               "segments_per_row": G, "path": plan.info()["path_name"]}
        ms_fused = time_calls(lambda: plan.convolve_linear(x, Hs, k, y, "full"), args.calls, args.rounds)
        launches = plan.info()["last_launches"]

        # the composition: segments materialised, circular convolution in place, valid parts cropped into y2
        Hc = Hs if F == 1 else Hs[:, None, :].expand(rows, G, bins).contiguous()   # per-segment spectra, built once
        y2 = torch.empty_like(y)
        padded = (G - 1) * s + n

        def composition():
            xp = F_.pad(x, (k - 1, padded - (k - 1) - length))
            seg = xp.unfold(-1, n, s).contiguous()            # (rows, G, N)
            plan.convolve(seg, Hc, seg)
            y2.copy_(seg[..., k - 1:].reshape(rows, G * s)[:, :out_len])

        ms_comp = time_calls(composition, args.calls, args.rounds)
        launches_comp = plan.info()["last_launches"] + 3   # + pad, segment copy, crop copy
        torch.cuda.synchronize()
        diff = float(((y - y2).abs().amax(-1) / y2.abs().amax(-1)).max())
        del Hc, y2
        torch.cuda.empty_cache()
        nt = 1 << (out_len - 1).bit_length()
        hf = torch.fft.rfft(h, n=nt)
        ms_torch = time_calls(lambda: torch.fft.irfft(torch.fft.rfft(x, n=nt) * (hf[0] if F == 1 else hf), n=nt),
                              args.calls, 3)
        del hf
        nbytes = rows * (length + out_len) * rb + F * bins * 2 * rb
        for name, ms in (("convolve_linear", ms_fused), ("composition", ms_comp), ("torch_fft", ms_torch)):
            row[name] = {"ms_per_call": round(ms, 4), "gb_per_s": round(nbytes / (ms * 1e-3) / 1e9, 1)}
        row["algorithmic_bytes"] = nbytes
        row["launches"] = launches
        row["launches_composition"] = launches_comp
        row["speedup_vs_composition"] = round(ms_comp / ms_fused, 3)
        row["max_rel_diff_vs_composition"] = float(f"{diff:.3e}")
        results.append(row)
        print(f"{prec} N={n} K={k} rows={rows} L={length} F={F} [{row['path']}]: convolve_linear {ms_fused:.3f} ms "
              f"({row['convolve_linear']['gb_per_s']} GB/s, {launches} launches), composition {ms_comp:.3f} ms "
              f"({row['composition']['gb_per_s']} GB/s), torch.fft {ms_torch:.3f} ms, max rel diff {diff:.2e}",
              flush=True)
        del x, y, h, H, Hs
        plan.close()
        torch.cuda.empty_cache()
    info["sm_clock_after"] = card()["sm_clock"]
    print(f"SM clock after the timed runs: {info['sm_clock_after']}")
    print(json.dumps({"card": info, "calls_per_round": args.calls, "rounds": args.rounds, "results": results}))


if __name__ == "__main__":
    main()

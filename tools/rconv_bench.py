"""Times the convolution of real rows, y = irfft(rfft(x) * H), on device buffers: RealFft.convolve next to the
three-call composition through the same plan (rfft -> torch multiply -> irfft) and, as an informative column only, the
same composition through torch.fft.  CUDA events: warm-up, then rounds of back-to-back calls, median round.  Prints
the card, its power limit and SM clock (before and after the timed runs), one line per case, and one JSON line.

    python tools/rconv_bench.py [--calls 10] [--rounds 5]

Algorithmic bytes: convolve reads x and writes y once (2 N reals per row) and reads the F spectra once.  The
composition also writes and reads the spectrum twice per row (rfft store, multiply load and store, irfft load):
2 N reals + 4 (N/2+1) complex values per row, plus the F spectra.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from rfft_bench import card, time_calls  # noqa: E402

# (precision, N, batch, F): the fused path at the two largest on-chip classes (one filter, and one per channel of 64),
# the half path on the persistent two-pass inner plans, the odd path
CASES = [("f32", 2048, 1 << 17, 1), ("f32", 2048, 1 << 17, 64), ("f64", 512, 1 << 18, 1), ("f32", 1 << 21, 128, 1),
         ("f64", 1 << 17, 1024, 1), ("f32", 1009, 1 << 17, 1)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    import torch
    import fourier_b200 as fb
    if not torch.cuda.is_available():
        raise SystemExit("rconv_bench.py needs a CUDA device")
    info = card()
    print(f"card: {info['name']}, power limit {info['power_limit']}, SM clock {info['sm_clock']}")
    results = []
    for prec, n, batch, F in CASES:
        rdt = torch.float32 if prec == "f32" else torch.float64
        cdt = torch.complex64 if prec == "f32" else torch.complex128
        rb = 4 if prec == "f32" else 8
        bins = n // 2 + 1
        plan = fb.create_rfft_f32(n) if prec == "f32" else fb.create_rfft_f64(n)
        g = torch.Generator(device="cuda").manual_seed(n + F)
        x = torch.randn((batch // F, F, n), dtype=rdt, device="cuda", generator=g)
        H = torch.empty((F, bins), dtype=cdt, device="cuda")
        plan.rfft(torch.randn((F, n), dtype=rdt, device="cuda", generator=g), H)
        Hs = H[0] if F == 1 else H
        y = torch.empty_like(x)
        row = {"precision": prec, "n": n, "batch": batch, "filters": F, "path": plan.info()["path_name"],
               "inner_path": plan.info()["inner_path_name"]}
        ms_conv = time_calls(lambda: plan.convolve(x, Hs, y), args.calls, args.rounds)
        launches = plan.info()["last_launches"]
        X = torch.empty((batch // F, F, bins), dtype=cdt, device="cuda")
        P = torch.empty_like(X)
        y3 = torch.empty_like(x)

        def three_calls():
            plan.rfft(x, X)
            torch.mul(X, H, out=P)
            plan.irfft(P, y3)

        ms_three = time_calls(three_calls, args.calls, args.rounds)
        plan.rfft(x, X)
        launches_three = plan.info()["last_launches"] + 1
        plan.irfft(P, y3)
        launches_three += plan.info()["last_launches"]
        torch.cuda.synchronize()
        diff = float(((y - y3).abs().amax(-1) / y3.abs().amax(-1)).max())
        del X, P, y3
        torch.cuda.empty_cache()
        ms_torch = time_calls(lambda: torch.fft.irfft(torch.fft.rfft(x) * H, n=n), args.calls, args.rounds)
        spec = F * bins * 2 * rb
        conv_bytes = batch * 2 * n * rb + spec
        three_bytes = batch * (2 * n * rb + 4 * bins * 2 * rb) + spec
        for name, ms, nbytes in (("convolve", ms_conv, conv_bytes), ("three_calls", ms_three, three_bytes),
                                 ("torch_fft", ms_torch, three_bytes)):
            row[name] = {"ms_per_call": round(ms, 4), "algorithmic_bytes": nbytes,
                         "gb_per_s": round(nbytes / (ms * 1e-3) / 1e9, 1)}
        row["launches"] = launches
        row["launches_three_calls"] = launches_three
        row["speedup_vs_three_calls"] = round(ms_three / ms_conv, 3)
        row["max_rel_diff_vs_three_calls"] = float(f"{diff:.3e}")
        results.append(row)
        print(f"{prec} N={n} batch={batch} F={F} [{row['path']}/{row['inner_path']}]: convolve {ms_conv:.3f} ms "
              f"({row['convolve']['gb_per_s']} GB/s, {launches} launches), three calls {ms_three:.3f} ms "
              f"({row['three_calls']['gb_per_s']} GB/s, {launches_three} launches), torch.fft {ms_torch:.3f} ms, "
              f"max rel diff {diff:.2e}", flush=True)
        del x, y, H
        plan.close()
        torch.cuda.empty_cache()
    info["sm_clock_after"] = card()["sm_clock"]
    print(f"SM clock after the timed runs: {info['sm_clock_after']}")
    print(json.dumps({"card": info, "calls_per_round": args.calls, "rounds": args.rounds, "results": results}))


if __name__ == "__main__":
    main()

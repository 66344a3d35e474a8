"""Times the short-time Fourier transform of real rows on device buffers: RealFft.stft next to the caller-side
composition on the same plan (F.pad reflect + unfold + contiguous * window + RealFft.rfft), RealFft.istft next to
torch.istft, and, as an informative column only, torch.stft.  CUDA events: warm-up, then rounds of back-to-back calls,
median round.  Prints the card, its power limit and SM clock (before and after the timed runs), one line per case, and
one JSON line.

    python tools/stft_bench.py [--calls 5] [--rounds 5]

Algorithmic bytes: L reals in plus F * (N/2+1) complex values out per row for the stft, the reverse for the istft.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from rfft_bench import card, time_calls  # noqa: E402

# (precision, N, hop, rows, L)
CASES = [("f32", 512, 128, 64, 1 << 20), ("f32", 2048, 512, 64, 1 << 20), ("f32", 400, 160, 256, 480000),
         ("f64", 512, 128, 64, 1 << 20)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    import torch
    import torch.nn.functional as F_
    import fourier_b200 as fb
    if not torch.cuda.is_available():
        raise SystemExit("stft_bench.py needs a CUDA device")
    info = card()
    print(f"card: {info['name']}, power limit {info['power_limit']}, SM clock {info['sm_clock']}")
    results = []
    for prec, n, hop, rows, length in CASES:
        rdt = torch.float32 if prec == "f32" else torch.float64
        cdt = torch.complex64 if prec == "f32" else torch.complex128
        rb = 4 if prec == "f32" else 8
        bins = n // 2 + 1
        plan = fb.create_rfft_f32(n) if prec == "f32" else fb.create_rfft_f64(n)
        frames = plan.stft_frames(length, hop)
        g = torch.Generator(device="cuda").manual_seed(n + hop)
        x = torch.randn((rows, length), dtype=rdt, device="cuda", generator=g)
        w = torch.hann_window(n, dtype=rdt, device="cuda")
        S = torch.empty((rows, frames, bins), dtype=cdt, device="cuda")
        row = {"precision": prec, "n": n, "hop": hop, "rows": rows, "in_len": length, "frames": frames,
               "path": plan.info()["path_name"]}
        ms_stft = time_calls(lambda: plan.stft(x, w, hop, S), args.calls, args.rounds)
        launches = plan.info()["last_launches"]

        S2 = torch.empty_like(S)

        def composition():
            u = F_.pad(x[:, None], (n // 2, n // 2), mode="reflect")[:, 0].unfold(-1, n, hop).contiguous() * w
            plan.rfft(u, S2)

        ms_comp = time_calls(composition, args.calls, args.rounds)
        launches_comp = plan.info()["last_launches"] + 3   # + pad, unfold copy, window multiply
        torch.cuda.synchronize()
        diff = float(((S - S2).abs().amax((-1, -2)) / S2.abs().amax((-1, -2))).max())
        del S2
        torch.cuda.empty_cache()
        ms_tstft = time_calls(lambda: torch.stft(x, n, hop, window=w, return_complex=True), args.calls, 3)

        y = torch.empty((rows, length), dtype=rdt, device="cuda")
        ms_istft = time_calls(lambda: plan.istft(S, w, hop, y), args.calls, args.rounds)
        launches_inv = plan.info()["last_launches"]
        St = S.transpose(-1, -2)
        ms_tistft = time_calls(lambda: torch.istft(St, n, hop, window=w, length=length), args.calls, args.rounds)
        yt = torch.istft(St, n, hop, window=w, length=length)
        torch.cuda.synchronize()
        diff_inv = float(((y - yt).abs().amax(-1) / yt.abs().amax(-1)).max())
        del yt, St
        nbytes = rows * (length * rb + frames * bins * 2 * rb)
        for name, ms in (("stft", ms_stft), ("composition", ms_comp), ("torch_stft", ms_tstft), ("istft", ms_istft),
                         ("torch_istft", ms_tistft)):
            row[name] = {"ms_per_call": round(ms, 4), "gb_per_s": round(nbytes / (ms * 1e-3) / 1e9, 1)}
        row["algorithmic_bytes"] = nbytes
        row["launches_stft"] = launches
        row["launches_composition"] = launches_comp
        row["launches_istft"] = launches_inv
        row["speedup_vs_composition"] = round(ms_comp / ms_stft, 3)
        row["speedup_vs_torch_istft"] = round(ms_tistft / ms_istft, 3)
        row["max_rel_diff_vs_composition"] = float(f"{diff:.3e}")
        row["max_rel_diff_vs_torch_istft"] = float(f"{diff_inv:.3e}")
        results.append(row)
        print(f"{prec} N={n} H={hop} rows={rows} L={length} F={frames} [{row['path']}]: stft {ms_stft:.3f} ms "
              f"({row['stft']['gb_per_s']} GB/s, {launches} launches), composition {ms_comp:.3f} ms "
              f"({row['composition']['gb_per_s']} GB/s), torch.stft {ms_tstft:.3f} ms; istft {ms_istft:.3f} ms "
              f"({row['istft']['gb_per_s']} GB/s, {launches_inv} launches), torch.istft {ms_tistft:.3f} ms; "
              f"max rel diff {diff:.2e} / {diff_inv:.2e}", flush=True)
        del x, w, S, y
        plan.close()
        torch.cuda.empty_cache()
    info["sm_clock_after"] = card()["sm_clock"]
    print(f"SM clock after the timed runs: {info['sm_clock_after']}")
    print(json.dumps({"card": info, "calls_per_round": args.calls, "rounds": args.rounds, "results": results}))


if __name__ == "__main__":
    main()

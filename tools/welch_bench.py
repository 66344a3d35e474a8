"""Times Welch's power spectral density of real rows on device buffers: RealFft.welch next to two compositions a caller
would otherwise write, and next to the plan's stft alone.  Hann window, density scaling.  Compositions:
  * "composition": the same plan's stft(center=False), then |S|^2 summed over the two real components, the mean over
    the frames, the one-sided factor and the scale (detrend False; welch is timed with detrend False against it);
  * "torch": unfold, subtract each frame's mean, window, torch.fft.rfft, |.|^2, the mean over the frames, factor and
    scale (detrend "constant"; welch is timed with detrend "constant" against it);
  * "stft": the plan's stft(center=False) alone, which stores every frame's spectrum.
CUDA events: warm-up, then rounds of back-to-back calls; the median round is reported with the fastest and slowest.
Prints the card, its power limit and SM clock (before and after the timed runs), one line per case, and one JSON line.

    python tools/welch_bench.py [--calls 5] [--rounds 5]

Algorithmic bytes of welch: L reals in plus N/2+1 reals out per row (those of the stft: L reals in plus F * (N/2+1)
complex values out).
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

# (precision, N, hop, rows, L): the fused path at three sizes, Whisper's frames on real_half, and many short rows
CASES = [("f32", 1024, 512, 64, 1 << 20), ("f32", 2048, 1024, 64, 1 << 20), ("f64", 512, 256, 64, 1 << 20),
         ("f32", 400, 160, 256, 480000), ("f32", 1024, 512, 1 << 14, 4096)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    import torch
    import fourier_b200 as fb
    if not torch.cuda.is_available():
        raise SystemExit("welch_bench.py needs a CUDA device")
    info = card()
    print(f"card: {info['name']}, power limit {info['power_limit']}, SM clock {info['sm_clock']}")
    results = []
    for prec, n, hop, rows, length in CASES:
        rdt = torch.float32 if prec == "f32" else torch.float64
        cdt = torch.complex64 if prec == "f32" else torch.complex128
        rb = 4 if prec == "f32" else 8
        bins = n // 2 + 1
        plan = fb.create_rfft_f32(n) if prec == "f32" else fb.create_rfft_f64(n)
        frames = plan.stft_frames(length, hop, center=False)
        g = torch.Generator(device="cuda").manual_seed(n + hop)
        x = torch.randn((rows, length), dtype=rdt, device="cuda", generator=g)
        w = torch.hann_window(n, dtype=rdt, device="cuda")
        scale = 1.0 / float((w.double() ** 2).sum())
        P = torch.empty((rows, bins), dtype=rdt, device="cuda")
        row = {"precision": prec, "n": n, "hop": hop, "rows": rows, "in_len": length, "frames": frames,
               "path": plan.info()["path_name"]}
        t_welch_none = time_rounds(lambda: plan.welch(x, w, hop, P, detrend=False), args.calls, args.rounds)
        t_welch = time_rounds(lambda: plan.welch(x, w, hop, P), args.calls, args.rounds)
        launches = plan.info()["last_launches"]
        S = torch.empty((rows, frames, bins), dtype=cdt, device="cuda")

        def onesided(p):
            p[..., 1:(n + 1) // 2] *= 2
            return p

        def composition():
            plan.stft(x, w, hop, S, center=False)
            return onesided(torch.view_as_real(S).square().sum(-1).mean(-2) * scale)

        def torch_composition():
            f = x.unfold(-1, n, hop)
            return onesided((torch.fft.rfft((f - f.mean(-1, keepdim=True)) * w).abs() ** 2).mean(-2) * scale)

        t_comp = time_rounds(composition, args.calls, args.rounds)
        plan.welch(x, w, hop, P, detrend=False)
        ref = composition()
        torch.cuda.synchronize()
        diff_comp = float(((P - ref).abs().amax(-1) / ref.abs().amax(-1)).max())
        t_stft = time_rounds(lambda: plan.stft(x, w, hop, S, center=False), args.calls, args.rounds)
        del S, ref
        torch.cuda.empty_cache()
        t_torch = time_rounds(torch_composition, args.calls, args.rounds)
        plan.welch(x, w, hop, P)
        ref = torch_composition()
        torch.cuda.synchronize()
        diff_torch = float(((P - ref).abs().amax(-1) / ref.abs().amax(-1)).max())
        del ref
        torch.cuda.empty_cache()
        bytes_welch = rows * (length + bins) * rb
        bytes_stft = rows * (length + frames * bins * 2) * rb
        for name, t, nbytes in (("welch", t_welch, bytes_welch), ("welch_detrend_none", t_welch_none, bytes_welch),
                                ("composition", t_comp, bytes_welch), ("torch", t_torch, bytes_welch),
                                ("stft", t_stft, bytes_stft)):
            ms = t[len(t) // 2]
            row[name] = {"ms_per_call": round(ms, 4), "ms_min": round(t[0], 4), "ms_max": round(t[-1], 4),
                         "gb_per_s": round(nbytes / (ms * 1e-3) / 1e9, 1)}
        row["algorithmic_bytes_welch"] = bytes_welch
        row["algorithmic_bytes_stft"] = bytes_stft
        row["launches_welch"] = launches
        row["speedup_vs_composition"] = round(row["composition"]["ms_per_call"] / row["welch_detrend_none"]["ms_per_call"], 3)
        row["speedup_vs_torch"] = round(row["torch"]["ms_per_call"] / row["welch"]["ms_per_call"], 3)
        row["speedup_vs_stft"] = round(row["stft"]["ms_per_call"] / row["welch"]["ms_per_call"], 3)
        row["max_rel_diff_vs_composition"] = float(f"{diff_comp:.3e}")
        row["max_rel_diff_vs_torch"] = float(f"{diff_torch:.3e}")
        results.append(row)
        print(f"{prec} N={n} H={hop} rows={rows} L={length} F={frames} [{row['path']}]: welch "
              f"{row['welch']['ms_per_call']:.3f} ms [{t_welch[0]:.3f}, {t_welch[-1]:.3f}] ({row['welch']['gb_per_s']} "
              f"GB/s, {launches} launches), detrend none {row['welch_detrend_none']['ms_per_call']:.3f} ms; "
              f"composition {row['composition']['ms_per_call']:.3f} ms [{t_comp[0]:.3f}, {t_comp[-1]:.3f}], torch "
              f"{row['torch']['ms_per_call']:.3f} ms [{t_torch[0]:.3f}, {t_torch[-1]:.3f}], stft alone "
              f"{row['stft']['ms_per_call']:.3f} ms [{t_stft[0]:.3f}, {t_stft[-1]:.3f}]; max rel diff "
              f"{diff_comp:.2e} / {diff_torch:.2e}", flush=True)
        del x, w, P
        plan.close()
        torch.cuda.empty_cache()
    info["sm_clock_after"] = card()["sm_clock"]
    print(f"SM clock after the timed runs: {info['sm_clock_after']}")
    print(json.dumps({"card": info, "calls_per_round": args.calls, "rounds": args.rounds, "results": results}))


if __name__ == "__main__":
    main()

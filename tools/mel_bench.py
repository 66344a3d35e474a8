"""Times the mel spectrogram of real rows on device buffers: RealFft.mel_spectrogram next to the caller-side composition
on the same plan (RealFft.stft + view_as_real(S).square().sum(-1) + @ filters.T), next to RealFft.stft alone, and, as
an informative column only, torchaudio's MelSpectrogram on the GPU.  Hann window, center with reflect padding, power 2,
torchaudio's HTK bank.  CUDA events: warm-up, then rounds of back-to-back calls; the median round is reported with the
fastest and slowest.  Prints the card, its power limit and SM clock (before and after the timed runs), one line per
case, and one JSON line.

    python tools/mel_bench.py [--calls 5] [--rounds 5]

Algorithmic bytes of the mel spectrogram: L reals in plus F * n_mels reals out per row (those of the stft: L reals in
plus F * (N/2+1) complex values out).
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from rfft_bench import card  # noqa: E402

# (precision, N, hop, n_mels, rows, L)
CASES = [("f32", 512, 128, 80, 64, 1 << 20), ("f32", 2048, 512, 128, 64, 1 << 20), ("f64", 512, 128, 80, 64, 1 << 20),
         ("f32", 400, 160, 80, 256, 480000)]


def time_rounds(fn, calls, rounds):
    """ms per call of each round, sorted"""
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
    return sorted(times)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    import torch
    import torchaudio
    import fourier_b200 as fb
    if not torch.cuda.is_available():
        raise SystemExit("mel_bench.py needs a CUDA device")
    info = card()
    print(f"card: {info['name']}, power limit {info['power_limit']}, SM clock {info['sm_clock']}")
    results = []
    for prec, n, hop, n_mels, rows, length in CASES:
        rdt = torch.float32 if prec == "f32" else torch.float64
        cdt = torch.complex64 if prec == "f32" else torch.complex128
        rb = 4 if prec == "f32" else 8
        bins = n // 2 + 1
        plan = fb.create_rfft_f32(n) if prec == "f32" else fb.create_rfft_f64(n)
        frames = plan.stft_frames(length, hop)
        g = torch.Generator(device="cuda").manual_seed(n + hop)
        x = torch.randn((rows, length), dtype=rdt, device="cuda", generator=g)
        w = torch.hann_window(n, dtype=rdt, device="cuda")
        fbank = torchaudio.functional.melscale_fbanks(bins, 0.0, 8000.0, n_mels, 16000).to("cuda", rdt)
        filters = fbank.T.contiguous()
        M = torch.empty((rows, frames, n_mels), dtype=rdt, device="cuda")
        row = {"precision": prec, "n": n, "hop": hop, "n_mels": n_mels, "rows": rows, "in_len": length,
               "frames": frames, "path": plan.info()["path_name"]}
        t_mel = time_rounds(lambda: plan.mel_spectrogram(x, w, hop, filters, M), args.calls, args.rounds)
        launches = plan.info()["last_launches"]

        S = torch.empty((rows, frames, bins), dtype=cdt, device="cuda")

        def composition():
            plan.stft(x, w, hop, S)
            return torch.view_as_real(S).square().sum(-1) @ filters.T

        t_comp = time_rounds(composition, args.calls, args.rounds)
        M2 = composition()
        torch.cuda.synchronize()
        diff = float(((M - M2).abs().amax((-1, -2)) / M2.abs().amax((-1, -2))).max())
        del M2
        torch.cuda.empty_cache()
        t_stft = time_rounds(lambda: plan.stft(x, w, hop, S), args.calls, args.rounds)
        del S
        torch.cuda.empty_cache()
        ta = torchaudio.transforms.MelSpectrogram(sample_rate=16000, n_fft=n, hop_length=hop, n_mels=n_mels).to("cuda",
                                                                                                              rdt)
        t_ta = time_rounds(lambda: ta(x), args.calls, 3)
        del ta
        torch.cuda.empty_cache()
        bytes_mel = rows * (length + frames * n_mels) * rb
        bytes_stft = rows * (length + frames * bins * 2) * rb
        for name, t, nbytes in (("mel", t_mel, bytes_mel), ("composition", t_comp, bytes_mel), ("stft", t_stft, bytes_stft),
                                ("torchaudio", t_ta, bytes_mel)):
            ms = t[len(t) // 2]
            row[name] = {"ms_per_call": round(ms, 4), "ms_min": round(t[0], 4), "ms_max": round(t[-1], 4),
                         "gb_per_s": round(nbytes / (ms * 1e-3) / 1e9, 1)}
        row["algorithmic_bytes_mel"] = bytes_mel
        row["algorithmic_bytes_stft"] = bytes_stft
        row["launches_mel"] = launches
        row["speedup_vs_composition"] = round(row["composition"]["ms_per_call"] / row["mel"]["ms_per_call"], 3)
        row["speedup_vs_stft"] = round(row["stft"]["ms_per_call"] / row["mel"]["ms_per_call"], 3)
        row["max_rel_diff_vs_composition"] = float(f"{diff:.3e}")
        results.append(row)
        print(f"{prec} N={n} H={hop} mels={n_mels} rows={rows} L={length} F={frames} [{row['path']}]: mel "
              f"{row['mel']['ms_per_call']:.3f} ms [{t_mel[0]:.3f}, {t_mel[-1]:.3f}] ({row['mel']['gb_per_s']} GB/s, "
              f"{launches} launches), composition {row['composition']['ms_per_call']:.3f} ms [{t_comp[0]:.3f}, "
              f"{t_comp[-1]:.3f}], stft alone {row['stft']['ms_per_call']:.3f} ms [{t_stft[0]:.3f}, {t_stft[-1]:.3f}], "
              f"torchaudio {row['torchaudio']['ms_per_call']:.3f} ms; max rel diff {diff:.2e}", flush=True)
        del x, w, M, filters, fbank
        plan.close()
        torch.cuda.empty_cache()
    info["sm_clock_after"] = card()["sm_clock"]
    print(f"SM clock after the timed runs: {info['sm_clock_after']}")
    print(json.dumps({"card": info, "calls_per_round": args.calls, "rounds": args.rounds, "results": results}))


if __name__ == "__main__":
    main()

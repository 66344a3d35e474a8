"""Times the MFCC and log-mel spectrogram of real rows on device buffers: RealFft.mfcc next to the caller-side
composition on the same plan (RealFft.mel_spectrogram, then torch's clamp, log, amax, maximum and matmul), next to
RealFft.mel_spectrogram alone, and, as an informative column only, torchaudio's MFCC on the GPU (not for Whisper's
log-mel, which torchaudio has no module for).  Hann window, center with reflect padding, power 2, torchaudio's HTK bank,
librosa's orthonormal DCT-II matrix; the clamp groups are single rows.  CUDA events: warm-up, then rounds of back-to-back
calls; the median round is reported with the fastest and slowest.  Prints the card, its power limit and SM clock (before
and after the timed runs), one line per case, and one JSON line.

    python tools/mfcc_bench.py [--calls 5] [--rounds 5]

Algorithmic bytes of the MFCC: L reals in plus F * n_out reals out per row (of the mel spectrogram: F * n_mels out).
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

# (name, precision, N, hop, n_mels, n_out (None: the log-mel), top_db, rows, L)
CASES = [("mfcc", "f32", 512, 128, 80, 40, None, 64, 1 << 20), ("mfcc", "f32", 512, 128, 80, 40, 80.0, 64, 1 << 20),
         ("mfcc", "f32", 2048, 512, 128, 40, 80.0, 64, 1 << 20), ("mfcc", "f64", 512, 128, 80, 40, 80.0, 64, 1 << 20),
         ("whisper", "f32", 400, 160, 80, None, 2.0, 256, 480000)]


def dct_matrix(n_mels, n_out, dtype):
    import torch
    m = torch.arange(n_mels, dtype=torch.float64)[:, None]
    j = torch.arange(n_out, dtype=torch.float64)[None, :]
    d = torch.cos(math.pi / n_mels * (m + 0.5) * j) * math.sqrt(2.0 / n_mels)
    d[:, 0] /= math.sqrt(2.0)
    return d.to("cuda", dtype).contiguous()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    import torch
    import torchaudio
    import fourier_b200 as fb
    if not torch.cuda.is_available():
        raise SystemExit("mfcc_bench.py needs a CUDA device")
    info = card()
    print(f"card: {info['name']}, power limit {info['power_limit']}, SM clock {info['sm_clock']}")
    results = []
    for name, prec, n, hop, n_mels, n_out, top_db, rows, length in CASES:
        rdt = torch.float32 if prec == "f32" else torch.float64
        rb = 4 if prec == "f32" else 8
        bins = n // 2 + 1
        plan = fb.create_rfft_f32(n) if prec == "f32" else fb.create_rfft_f64(n)
        frames = plan.stft_frames(length, hop)
        g = torch.Generator(device="cuda").manual_seed(n + hop)
        x = torch.randn((rows, length), dtype=rdt, device="cuda", generator=g)
        w = torch.hann_window(n, dtype=rdt, device="cuda")
        mel_scale = "slaney" if name == "whisper" else "htk"
        fbank = torchaudio.functional.melscale_fbanks(bins, 0.0, 8000.0, n_mels, 16000, norm=mel_scale if name ==
                                                      "whisper" else None, mel_scale=mel_scale).to("cuda", rdt)
        filters = fbank.T.contiguous()
        if name == "whisper":
            dct, kw = None, dict(log_scale=1.0 / (4.0 * math.log(10.0)), top_db=top_db, bias=1.0)
            n_out = n_mels
        else:
            dct, kw = dct_matrix(n_mels, n_out, rdt), dict(top_db=top_db)
        out = torch.empty((rows, frames, n_out), dtype=rdt, device="cuda")
        row = {"case": name, "precision": prec, "n": n, "hop": hop, "n_mels": n_mels, "n_out": n_out, "top_db": top_db,
               "rows": rows, "in_len": length, "frames": frames, "path": plan.info()["path_name"]}
        t_mfcc = time_rounds(lambda: plan.mfcc(x, w, hop, filters, dct, out, **kw), args.calls, args.rounds)
        launches = plan.info()["last_launches"]
        M = torch.empty((rows, frames, n_mels), dtype=rdt, device="cuda")

        def composition():
            plan.mel_spectrogram(x, w, hop, filters, M)
            if name == "whisper":
                lm = M.clamp(min=1e-10).log10()
                lm = torch.maximum(lm, lm.amax((-1, -2), keepdim=True) - 8.0)
                return (lm + 4.0) / 4.0
            lm = 10.0 * M.clamp(min=1e-10).log10()
            if top_db is not None:
                lm = torch.maximum(lm, lm.amax((-1, -2), keepdim=True) - top_db)
            return lm @ dct

        t_comp = time_rounds(composition, args.calls, args.rounds)
        ref = composition()
        torch.cuda.synchronize()
        diff = float(((out - ref).abs().amax((-1, -2)) / ref.abs().amax((-1, -2))).max())
        del ref
        torch.cuda.empty_cache()
        t_mel = time_rounds(lambda: plan.mel_spectrogram(x, w, hop, filters, M), args.calls, args.rounds)
        del M
        torch.cuda.empty_cache()
        t_ta = None
        if name != "whisper":
            ta = torchaudio.transforms.MFCC(sample_rate=16000, n_mfcc=n_out, melkwargs={
                "n_fft": n, "hop_length": hop, "n_mels": n_mels}).to("cuda", rdt)
            if top_db is None:
                ta.top_db = None
                ta.amplitude_to_DB.top_db = None
            t_ta = time_rounds(lambda: ta(x), args.calls, 3)
            del ta
            torch.cuda.empty_cache()
        bytes_mfcc = rows * (length + frames * n_out) * rb
        bytes_mel = rows * (length + frames * n_mels) * rb
        for key, t, nbytes in (("mfcc", t_mfcc, bytes_mfcc), ("composition", t_comp, bytes_mfcc),
                               ("mel", t_mel, bytes_mel), ("torchaudio", t_ta, bytes_mfcc)):
            if t is None:
                continue
            ms = t[len(t) // 2]
            row[key] = {"ms_per_call": round(ms, 4), "ms_min": round(t[0], 4), "ms_max": round(t[-1], 4),
                        "gb_per_s": round(nbytes / (ms * 1e-3) / 1e9, 1)}
        row["algorithmic_bytes_mfcc"] = bytes_mfcc
        row["launches_mfcc"] = launches
        row["speedup_vs_composition"] = round(row["composition"]["ms_per_call"] / row["mfcc"]["ms_per_call"], 3)
        row["time_vs_mel"] = round(row["mfcc"]["ms_per_call"] / row["mel"]["ms_per_call"], 3)
        row["max_rel_diff_vs_composition"] = float(f"{diff:.3e}")
        results.append(row)
        ta_txt = f"{row['torchaudio']['ms_per_call']:.3f} ms" if t_ta else "n/a"
        print(f"{name} {prec} N={n} H={hop} mels={n_mels} out={n_out} top_db={top_db} rows={rows} L={length} F={frames} "
              f"[{row['path']}]: mfcc {row['mfcc']['ms_per_call']:.3f} ms [{t_mfcc[0]:.3f}, {t_mfcc[-1]:.3f}] "
              f"({launches} launches), composition {row['composition']['ms_per_call']:.3f} ms [{t_comp[0]:.3f}, "
              f"{t_comp[-1]:.3f}], mel alone {row['mel']['ms_per_call']:.3f} ms [{t_mel[0]:.3f}, {t_mel[-1]:.3f}], "
              f"torchaudio {ta_txt}; max rel diff {diff:.2e}", flush=True)
        del x, w, out, filters, fbank
        plan.close()
        torch.cuda.empty_cache()
    info["sm_clock_after"] = card()["sm_clock"]
    print(f"SM clock after the timed runs: {info['sm_clock_after']}")
    print(json.dumps({"card": info, "calls_per_round": args.calls, "rounds": args.rounds, "results": results}))


if __name__ == "__main__":
    main()

"""Times the cross-spectral density and coherence of real rows on device buffers: RealFft.csd and coherence next to the
compositions a caller would otherwise write.  Hann window, density scaling, one y row per x row.  Compositions:
  * "composition": two stft(center=False) calls of the same plan, conj(X) * Y, the mean over the frames, the one-sided
    factor and the scale (detrend False; csd is timed with detrend False against it);
  * "torch": unfold x and y, subtract each frame's mean, window, torch.fft.rfft, conj(X) * Y, the mean, factor and scale
    (detrend "constant"; csd is timed with detrend "constant" against it);
  * "welch": the plan's welch of x alone, which reads half the bytes;
  * "coherence composition": welch(x), welch(y) and csd(x, y) of the same plan, then |Pxy|^2 / (Pxx Pyy).
CUDA events: warm-up, then rounds of back-to-back calls; the median round is reported with the fastest and slowest.
Prints the card, its power limit and SM clock (before and after the timed runs), one line per case, and one JSON line.

    python tools/csd_bench.py [--calls 5] [--rounds 5]

Algorithmic bytes of csd: 2 L reals in plus N/2+1 complex values out per row; of the coherence: 2 L reals in plus N/2+1
reals out.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from welch_bench import card, time_rounds  # noqa: E402

# (precision, N, hop, rows, L): the fused path at three sizes, Whisper's frames on real_half, and many short rows
CASES = [("f32", 1024, 512, 64, 1 << 20), ("f32", 2048, 1024, 64, 1 << 20), ("f64", 512, 256, 64, 1 << 20),
         ("f32", 400, 160, 256, 480000), ("f32", 1024, 512, 1 << 14, 4096)]


def stat(t, nbytes):
    ms = t[len(t) // 2]
    return {"ms_per_call": round(ms, 4), "ms_min": round(t[0], 4), "ms_max": round(t[-1], 4),
            "gb_per_s": round(nbytes / (ms * 1e-3) / 1e9, 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    import torch
    import fourier_b200 as fb
    if not torch.cuda.is_available():
        raise SystemExit("csd_bench.py needs a CUDA device")
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
        y = torch.randn((rows, length), dtype=rdt, device="cuda", generator=g) + 0.5 * x
        w = torch.hann_window(n, dtype=rdt, device="cuda")
        scale = 1.0 / float((w.double() ** 2).sum())
        P = torch.empty((rows, bins), dtype=cdt, device="cuda")
        Cxy = torch.empty((rows, bins), dtype=rdt, device="cuda")
        Pxx = torch.empty((rows, bins), dtype=rdt, device="cuda")
        Pyy = torch.empty((rows, bins), dtype=rdt, device="cuda")
        row = {"precision": prec, "n": n, "hop": hop, "rows": rows, "in_len": length, "frames": frames,
               "path": plan.info()["path_name"]}
        t_csd_none = time_rounds(lambda: plan.csd(x, y, w, hop, P, detrend=False), args.calls, args.rounds)
        t_csd = time_rounds(lambda: plan.csd(x, y, w, hop, P), args.calls, args.rounds)
        launches_csd = plan.info()["last_launches"]
        t_coh = time_rounds(lambda: plan.coherence(x, y, w, hop, Cxy), args.calls, args.rounds)
        launches_coh = plan.info()["last_launches"]
        t_welch = time_rounds(lambda: plan.welch(x, w, hop, Pxx), args.calls, args.rounds)
        SX = torch.empty((rows, frames, bins), dtype=cdt, device="cuda")
        SY = torch.empty_like(SX)

        def onesided(p):
            p[..., 1:(n + 1) // 2] *= 2
            return p

        def composition():
            plan.stft(x, w, hop, SX, center=False)
            plan.stft(y, w, hop, SY, center=False)
            return onesided((SX.conj() * SY).mean(-2) * scale)

        def torch_composition():
            fx, fy = x.unfold(-1, n, hop), y.unfold(-1, n, hop)
            X = torch.fft.rfft((fx - fx.mean(-1, keepdim=True)) * w)
            Y = torch.fft.rfft((fy - fy.mean(-1, keepdim=True)) * w)
            return onesided((X.conj() * Y).mean(-2) * scale)

        def coherence_composition():
            plan.welch(x, w, hop, Pxx)
            plan.welch(y, w, hop, Pyy)
            plan.csd(x, y, w, hop, P)
            return P.abs() ** 2 / (Pxx * Pyy)

        t_comp = time_rounds(composition, args.calls, args.rounds)
        plan.csd(x, y, w, hop, P, detrend=False)
        ref = composition()
        torch.cuda.synchronize()
        diff_comp = float(((P - ref).abs().amax(-1) / ref.abs().amax(-1)).max())
        del SX, SY, ref
        torch.cuda.empty_cache()
        t_torch = time_rounds(torch_composition, args.calls, args.rounds)
        plan.csd(x, y, w, hop, P)
        ref = torch_composition()
        torch.cuda.synchronize()
        diff_torch = float(((P - ref).abs().amax(-1) / ref.abs().amax(-1)).max())
        del ref
        torch.cuda.empty_cache()
        t_coh_comp = time_rounds(coherence_composition, args.calls, args.rounds)
        plan.coherence(x, y, w, hop, Cxy)
        ref = coherence_composition()
        torch.cuda.synchronize()
        diff_coh = float((Cxy - ref).abs().max())
        del ref
        bytes_csd = rows * (2 * length + 2 * bins) * rb
        bytes_coh = rows * (2 * length + bins) * rb
        bytes_welch = rows * (length + bins) * rb
        for name, t, nbytes in (("csd", t_csd, bytes_csd), ("csd_detrend_none", t_csd_none, bytes_csd),
                                ("composition", t_comp, bytes_csd), ("torch", t_torch, bytes_csd),
                                ("welch_x", t_welch, bytes_welch), ("coherence", t_coh, bytes_coh),
                                ("coherence_composition", t_coh_comp, bytes_coh)):
            row[name] = stat(t, nbytes)
        row["launches_csd"] = launches_csd
        row["launches_coherence"] = launches_coh
        row["speedup_vs_composition"] = round(row["composition"]["ms_per_call"] / row["csd_detrend_none"]["ms_per_call"], 3)
        row["speedup_vs_torch"] = round(row["torch"]["ms_per_call"] / row["csd"]["ms_per_call"], 3)
        row["csd_over_welch_x"] = round(row["csd"]["ms_per_call"] / row["welch_x"]["ms_per_call"], 3)
        row["coherence_speedup_vs_composition"] = round(
            row["coherence_composition"]["ms_per_call"] / row["coherence"]["ms_per_call"], 3)
        row["max_rel_diff_vs_composition"] = float(f"{diff_comp:.3e}")
        row["max_rel_diff_vs_torch"] = float(f"{diff_torch:.3e}")
        row["max_abs_diff_coherence"] = float(f"{diff_coh:.3e}")
        results.append(row)
        med = {k: row[k]["ms_per_call"] for k in ("csd", "csd_detrend_none", "composition", "torch", "welch_x",
                                                  "coherence", "coherence_composition")}
        print(f"{prec} N={n} H={hop} rows={rows} L={length} F={frames} [{row['path']}]: csd {med['csd']:.3f} ms "
              f"[{t_csd[0]:.3f}, {t_csd[-1]:.3f}] ({row['csd']['gb_per_s']} GB/s, {launches_csd} launches), detrend none "
              f"{med['csd_detrend_none']:.3f} ms; composition {med['composition']:.3f} ms [{t_comp[0]:.3f}, "
              f"{t_comp[-1]:.3f}], torch {med['torch']:.3f} ms [{t_torch[0]:.3f}, {t_torch[-1]:.3f}], welch(x) "
              f"{med['welch_x']:.3f} ms [{t_welch[0]:.3f}, {t_welch[-1]:.3f}]; coherence {med['coherence']:.3f} ms "
              f"[{t_coh[0]:.3f}, {t_coh[-1]:.3f}] ({launches_coh} launches), welch+welch+csd "
              f"{med['coherence_composition']:.3f} ms [{t_coh_comp[0]:.3f}, {t_coh_comp[-1]:.3f}]; max diff "
              f"{diff_comp:.2e} / {diff_torch:.2e} / {diff_coh:.2e}", flush=True)
        del x, y, w, P, Cxy, Pxx, Pyy
        plan.close()
        torch.cuda.empty_cache()
    info["sm_clock_after"] = card()["sm_clock"]
    print(f"SM clock after the timed runs: {info['sm_clock_after']}")
    print(json.dumps({"card": info, "calls_per_round": args.calls, "rounds": args.rounds, "results": results}))


if __name__ == "__main__":
    main()

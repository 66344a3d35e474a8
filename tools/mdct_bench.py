"""Times the MDCT and IMDCT of real rows on device buffers (RealFft.mdct / imdct, center, norm backward, a sine window)
next to the compositions a PyTorch caller would otherwise write, and next to the plan's rfft over the same samples:
  * "composition": torch pads, frames (unfold), windows and folds the rows, then the same plan's dct4; for the imdct, the
    plan's dct4 of the coefficients, then torch unfolds, windows and overlap-adds them (torch.nn.functional.fold);
  * "torch": a pure-torch MDCT: frames, window and fold, the pre-twiddle, torch.fft.fft of length N/2 and the
    post-twiddle;
  * "rfft": the plan's rfft of the same samples as rows of N reals: the same bytes in, about the same out.
CUDA events: warm-up, then rounds of back-to-back calls; the median round is reported with the fastest and slowest.
Prints the card, its power limit and SM clock (before and after the timed runs), one line per case, and one JSON line.

    python tools/mdct_bench.py [--calls 5] [--rounds 5]

Algorithmic bytes of an mdct (and of its imdct): L reals in and F N reals out per row (the reverse for the imdct).
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

# (precision, N, rows): rows of 64 N samples (65 frames with center); the fused path at three sizes and real_half at
# Opus's 960, each call moving at least 256 MB
CASES = [("f32", 256, 2048), ("f32", 1024, 512), ("f64", 512, 512), ("f32", 960, 560)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    import torch
    import torch.nn.functional as tf
    import fourier_b200 as fb
    if not torch.cuda.is_available():
        raise SystemExit("mdct_bench.py needs a CUDA device")
    info = card()
    print(f"card: {info['name']}, power limit {info['power_limit']}, SM clock {info['sm_clock']}")
    results = []
    for prec, n, rows in CASES:
        rdt = torch.float32 if prec == "f32" else torch.float64
        cdt = torch.complex64 if prec == "f32" else torch.complex128
        rb = 4 if prec == "f32" else 8
        length = 64 * n
        plan = fb.create_rfft_f32(n) if prec == "f32" else fb.create_rfft_f64(n)
        F = plan.mdct_frames(length)
        g = torch.Generator(device="cuda").manual_seed(n)
        x = torch.randn((rows, length), dtype=rdt, device="cuda", generator=g)
        w = torch.sin(math.pi * (torch.arange(2 * n, device="cuda", dtype=torch.float64) + 0.5) / (2 * n)).to(rdt)
        X = torch.empty((rows, F, n), dtype=rdt, device="cuda")
        y = torch.empty_like(x)
        u = torch.empty_like(X)
        V = torch.empty((rows * length // n, n // 2 + 1), dtype=cdt, device="cuda")
        j = torch.arange(n // 2, device="cuda", dtype=torch.float64)
        pre = torch.polar(torch.ones_like(j), -math.pi * (4 * j + 1) / (4 * n)).to(cdt)   # W^{2j} exp(-i pi / (4N))
        post = torch.polar(torch.ones_like(j), -math.pi * j / n).to(cdt) * 2                # 2 W^{2k}
        row = {"precision": prec, "n": n, "rows": rows, "in_len": length, "frames": F, "path": plan.info()["path_name"]}

        def folded():
            xp = tf.pad(x, (n, (F + 1) * n - length - n))
            fr = xp.unfold(-1, 2 * n, n) * w
            a, b, c, d = fr.split(n // 2, -1)
            return torch.cat((-c.flip(-1) - d, a - b.flip(-1)), -1)

        def comp_mdct():
            plan.dct4(folded().contiguous(), u)
            return u

        def torch_mdct():
            v = folded()
            z = torch.complex(v[..., ::2], v.flip(-1)[..., ::2]) * pre
            P = torch.fft.fft(z) * post
            return _post_layout(P, n)

        def comp_imdct():
            plan.dct4(X, u, norm="forward")
            h = n // 2
            fr = torch.cat((u[..., h:], -u.flip(-1), -u[..., :h]), -1) * w   # (rows, F, 2N)
            out = tf.fold(fr.transpose(1, 2), output_size=(1, (F + 1) * n), kernel_size=(1, 2 * n), stride=(1, n))
            return out.view(rows, (F + 1) * n)[:, n:n + length]

        t = {}
        t["mdct"] = time_rounds(lambda: plan.mdct(x, w, X), args.calls, args.rounds)
        row["launches_mdct"] = plan.info()["last_launches"]
        t["composition_mdct"] = time_rounds(comp_mdct, args.calls, args.rounds)
        t["torch_mdct"] = time_rounds(torch_mdct, args.calls, args.rounds)
        t["imdct"] = time_rounds(lambda: plan.imdct(X, w, y), args.calls, args.rounds)
        row["launches_imdct"] = plan.info()["last_launches"]
        t["composition_imdct"] = time_rounds(comp_imdct, args.calls, args.rounds)
        t["rfft"] = time_rounds(lambda: plan.rfft(x.view(-1, n), V), args.calls, args.rounds)
        plan.mdct(x, w, X)
        ref = comp_mdct().clone()
        tor = torch_mdct()
        torch.cuda.synchronize()
        scale = X.abs().amax(-1).clamp_min(1e-30)
        row["max_rel_diff_mdct_vs_composition"] = float(f"{float(((X - ref).abs().amax(-1) / scale).max()):.3e}")
        row["max_rel_diff_mdct_vs_torch"] = float(f"{float(((X - tor).abs().amax(-1) / scale).max()):.3e}")
        plan.imdct(X, w, y)
        yc = comp_imdct()
        torch.cuda.synchronize()
        row["max_rel_diff_imdct_vs_composition"] = float(
            f"{float(((y - yc).abs().amax(-1) / y.abs().amax(-1)).max()):.3e}")
        row["round_trip_max_rel_err"] = float(f"{float(((y - x).abs().amax(-1) / x.abs().amax(-1)).max()):.3e}")
        del ref, tor, yc
        nbytes = rows * (length + F * n) * rb
        for name, ts in t.items():
            ms = ts[len(ts) // 2]
            b = nbytes if name != "rfft" else rows * length * rb + V.numel() * 2 * rb
            row[name] = {"ms_per_call": round(ms, 4), "ms_min": round(ts[0], 4), "ms_max": round(ts[-1], 4),
                         "gb_per_s": round(b / (ms * 1e-3) / 1e9, 1)}
        row["algorithmic_bytes"] = nbytes
        m, mi = row["mdct"]["ms_per_call"], row["imdct"]["ms_per_call"]
        row["speedup_mdct_vs_composition"] = round(row["composition_mdct"]["ms_per_call"] / m, 3)
        row["speedup_mdct_vs_torch"] = round(row["torch_mdct"]["ms_per_call"] / m, 3)
        row["speedup_imdct_vs_composition"] = round(row["composition_imdct"]["ms_per_call"] / mi, 3)
        row["mdct_over_rfft"] = round(m / row["rfft"]["ms_per_call"], 3)
        row["imdct_over_rfft"] = round(mi / row["rfft"]["ms_per_call"], 3)
        results.append(row)

        def cell(name):
            ts = t[name]
            return f"{ts[len(ts) // 2]:.3f} ms [{ts[0]:.3f}, {ts[-1]:.3f}]"

        print(f"{prec} N={n} rows={rows} L={length} F={F} [{row['path']}]: mdct {cell('mdct')} "
              f"({row['mdct']['gb_per_s']} GB/s), composition {cell('composition_mdct')}, torch {cell('torch_mdct')}; "
              f"imdct {cell('imdct')} ({row['imdct']['gb_per_s']} GB/s), composition {cell('composition_imdct')}; "
              f"rfft alone {cell('rfft')}; diffs {row['max_rel_diff_mdct_vs_composition']:.1e} / "
              f"{row['max_rel_diff_mdct_vs_torch']:.1e} / {row['max_rel_diff_imdct_vs_composition']:.1e}, "
              f"round trip {row['round_trip_max_rel_err']:.1e}", flush=True)
        del x, y, X, u, V
        plan.close()
        torch.cuda.empty_cache()
    info["sm_clock_after"] = card()["sm_clock"]
    print(f"SM clock after the timed runs: {info['sm_clock_after']}")
    print(json.dumps({"card": info, "calls_per_round": args.calls, "rounds": args.rounds, "results": results}))


def _post_layout(P, n):
    """(y[2k], y[N-1-2k]) = (Re P, -Im P) as rows of N reals"""
    import torch
    y = torch.empty(P.shape[:-1] + (n,), dtype=P.real.dtype, device=P.device)
    y[..., ::2] = P.real
    y[..., 1::2] = -P.imag.flip(-1)
    return y


if __name__ == "__main__":
    main()

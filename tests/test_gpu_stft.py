"""Short-time Fourier transform of real rows (RealFft.stft / istft, fourier_b200_stft_* / fourier_b200_istft_*) on the
GPU: every fused size class and the half-length and full-length paths against float64 numpy framing + rfft and against
CPU float64 torch.stft, round trips against torch.istft, the zero rule where no window covers, leading shapes, hops
beyond N, the shortest legal rows, host against device memory bit for bit (one row above the 64 MB staging chunk), an
inverse long enough to need two scratch runs, a side stream, launch counts and refusals.  Outputs are NaN-filled before
each call, so an element the call never writes fails."""

import numpy as np
import pytest

import fourier_b200 as fb
from fourier_b200 import _lib
from helpers import per_transform_err

pytestmark = pytest.mark.gpu

TOL = {"f32": 2e-5, "f64": 1e-12}
REAL = {"f32": np.float32, "f64": np.float64}
SPEC = {"f32": np.complex64, "f64": np.complex128}
BOUNDARIES = (("none", False, "reflect"), ("zeros", True, "constant"), ("reflect", True, "reflect"))
FUSED = [("f32", n) for n in (128, 256, 512, 1024, 2048)] + [("f64", n) for n in (128, 256, 512)]


def torch_mod():
    import torch
    return torch


def tdt(prec, kind):
    torch = torch_mod()
    return getattr(torch, np.dtype((REAL if kind == "real" else SPEC)[prec]).name)


def plan(prec, n):
    return fb.create_rfft_f32(n) if prec == "f32" else fb.create_rfft_f64(n)


def reals(prec, shape, seed):
    return np.random.default_rng(seed).standard_normal(shape).astype(REAL[prec])


def window(prec, n, seed=5):
    return (0.5 + 0.5 * np.random.default_rng(seed).random(n)).astype(REAL[prec])


def hann(prec, n):
    return torch_mod().hann_window(n, dtype=torch_mod().float64).numpy().astype(REAL[prec])


def ref_stft(x, w, hop, center, pad_mode):
    """float64 numpy: pad, frames every hop, times the window, rfft; frame-major"""
    x = np.asarray(x, np.float64)
    n = len(w)
    if center:
        widths = [(0, 0)] * (x.ndim - 1) + [(n // 2, n // 2)]
        x = np.pad(x, widths, mode=pad_mode)
    frames = np.lib.stride_tricks.sliding_window_view(x, n, axis=-1)[..., ::hop, :]
    return np.fft.rfft(frames * np.asarray(w, np.float64), axis=-1)


def torch_stft(x, w, hop, center, pad_mode):
    torch = torch_mod()
    s = torch.stft(torch.from_numpy(np.asarray(x, np.float64)), len(w), hop, window=torch.from_numpy(np.asarray(w, np.float64)),
                   center=center, pad_mode=pad_mode, return_complex=True)
    return s.transpose(-1, -2).numpy()


def dev_stft(p, x, w, hop, center=True, pad_mode="reflect"):
    """device stft of numpy x -> (torch output, frames)"""
    torch = torch_mod()
    prec = p.real
    n = p.size()
    frames = p.stft_frames(x.shape[-1], hop, center)
    xd, wd = torch.from_numpy(x).cuda(), torch.from_numpy(w).cuda()
    out = torch.full(x.shape[:-1] + (frames, n // 2 + 1), complex(float("nan"), float("nan")), dtype=tdt(prec, "spec"),
                     device="cuda")
    p.stft(xd, wd, hop, out, center=center, pad_mode=pad_mode)
    torch.cuda.synchronize()
    return out, frames


def row_err(got, ref):
    """per row (all frames of one input row) max |got - ref| / max |ref|"""
    lead = int(np.prod(np.shape(ref)[:-2], dtype=np.int64)) or 1
    return per_transform_err(np.asarray(got).reshape(lead, -1), np.asarray(ref).reshape(lead, -1)).max()


def launches(p):
    return p.info()["last_launches"]


@pytest.mark.parametrize("prec,n", FUSED)
@pytest.mark.parametrize("boundary,center,pad_mode", BOUNDARIES)
def test_fused_size_classes(prec, n, boundary, center, pad_mode):
    p = plan(prec, n)
    assert p.info()["path_name"] == "real_fused"
    hop = n // 4
    x = reals(prec, (3, 3 * n + 17), n)
    w = window(prec, n)
    out, frames = dev_stft(p, x, w, hop, center, pad_mode)
    assert launches(p) == 1
    got = out.cpu().numpy()
    ref = ref_stft(x, w, hop, center, pad_mode)
    assert got.shape == ref.shape
    assert row_err(got, ref) < TOL[prec]
    assert row_err(got, torch_stft(x, w, hop, center, pad_mode)) < TOL[prec]


def test_real_half_whisper_shape():
    torch = torch_mod()
    p = plan("f32", 400)
    assert p.info()["path_name"] == "real_half"
    x = reals("f32", (2, 480000), 11)
    w = hann("f32", 400)
    out, frames = dev_stft(p, x, w, 160)
    assert frames == 3001
    n_stft = launches(p)
    got = out.cpu().numpy()
    assert row_err(got, ref_stft(x, w, 160, True, "reflect")) < TOL["f32"]
    assert row_err(got, torch_stft(x, w, 160, True, "reflect")) < TOL["f32"]
    # one chunk: the gather and the plan's rfft of all 6002 frames
    frames_in = torch.zeros(2 * frames, 400, dtype=torch.float32, device="cuda")
    spec = torch.empty(2 * frames, 201, dtype=torch.complex64, device="cuda")
    p.rfft(frames_in, spec)
    assert n_stft == 1 + launches(p)


def test_real_half_persistent_inner_plan():
    n = 1 << 21
    p = plan("f32", n)
    info = p.info()
    assert info["path_name"] == "real_half"
    x = reals("f32", (1, 4 * n + 5), 12)
    w = window("f32", n)
    out, frames = dev_stft(p, x, w, n // 2, True, "constant")
    assert frames == 9
    assert row_err(out.cpu().numpy(), ref_stft(x, w, n // 2, True, "constant")) < 1e-4


@pytest.mark.parametrize("prec", ("f32", "f64"))
@pytest.mark.parametrize("boundary,center,pad_mode", BOUNDARIES)
def test_real_full_odd_n(prec, boundary, center, pad_mode):
    p = plan(prec, 1009)
    assert p.info()["path_name"] == "real_full"
    x = reals(prec, (2, 5000), 13)
    w = window(prec, 1009)
    out, frames = dev_stft(p, x, w, 250, center, pad_mode)
    got = out.cpu().numpy()
    assert row_err(got, ref_stft(x, w, 250, center, pad_mode)) < TOL[prec]
    assert row_err(got, torch_stft(x, w, 250, center, pad_mode)) < TOL[prec]


def dev_istft(p, spec, w, hop, out_len, center=True):
    torch = torch_mod()
    y = torch.full(tuple(spec.shape[:-2]) + (out_len,), float("nan"), dtype=tdt(p.real, "real"), device="cuda")
    p.istft(spec, torch.from_numpy(w).cuda(), hop, y, center=center)
    torch.cuda.synchronize()
    return y


@pytest.mark.parametrize("prec,n", [("f32", 512), ("f64", 512), ("f32", 400), ("f64", 1009)])
@pytest.mark.parametrize("div", (4, 2))
def test_round_trip_matches_torch_istft(prec, n, div):
    torch = torch_mod()
    p = plan(prec, n)
    hop = n // div
    L = 7 * n + 33
    x = reals(prec, (2, L), 14)
    w = hann(prec, n)
    spec, frames = dev_stft(p, x, w, hop)
    y = dev_istft(p, spec, w, hop, L).cpu().numpy()
    assert np.abs(y - x).max() / np.abs(x).max() < 10 * TOL[prec]
    default = hop * (frames - 1) + n - 2 * (n // 2)
    yd = dev_istft(p, spec, w, hop, default).cpu().numpy()
    sc = spec.cpu().to(torch.complex128).transpose(-1, -2)
    wt = torch.from_numpy(w.astype(np.float64))
    t_len = torch.istft(sc, n, hop, window=wt, center=True, length=L).numpy()
    t_def = torch.istft(sc, n, hop, window=wt, center=True).numpy()
    assert t_def.shape[-1] == default
    assert np.abs(y - t_len).max() / np.abs(t_len).max() < 10 * TOL[prec]
    assert np.abs(yd - t_def).max() / np.abs(t_def).max() < 10 * TOL[prec]


def test_center_false_zero_rule():
    """Hann without center: position 0 has window 0 in every frame that covers it, and positions past the last frame
    are covered by none; both give exactly 0 (torch.istft raises there)."""
    n, hop = 512, 128
    p = plan("f64", n)
    x = reals("f64", (1, 4000), 15)
    w = hann("f64", n)
    spec, frames = dev_stft(p, x, w, hop, center=False)
    covered = hop * (frames - 1) + n
    y = dev_istft(p, spec, w, hop, covered + 40, center=False).cpu().numpy()[0]
    assert y[0] == 0.0
    assert np.all(y[covered:] == 0.0)
    assert np.abs(y[1:covered] - x[0, 1:covered]).max() < 1e-8


def test_leading_shapes_and_hop_beyond_n():
    p = plan("f32", 256)
    x = reals("f32", (2, 3, 1000), 16)
    w = window("f32", 256)
    out, frames = dev_stft(p, x, w, 300)
    assert tuple(out.shape) == (2, 3, frames, 129)
    assert row_err(out.cpu().numpy(), ref_stft(x, w, 300, True, "reflect")) < TOL["f32"]
    # gaps between frames: positions no frame covers are 0, the others are the input
    y = dev_istft(p, out, w, 300, 1000).cpu().numpy()
    t = np.arange(1000) + 128
    cov = (t % 300) < 256
    assert np.all(y[..., ~cov] == 0.0)
    assert np.abs(y[..., cov] - x[..., cov]).max() < 1e-4


@pytest.mark.parametrize("prec", ("f32", "f64"))
def test_shortest_legal_rows(prec):
    n = 512
    p = plan(prec, n)
    w = window(prec, n)
    for (boundary, center, pad_mode), L in zip(BOUNDARIES, (n, 1, n // 2 + 1)):
        for hop in (1, 37, n + 3):
            x = reals(prec, (2, L), 17 + L)
            out, frames = dev_stft(p, x, w, hop, center, pad_mode)
            assert row_err(out.cpu().numpy(), ref_stft(x, w, hop, center, pad_mode)) < TOL[prec], (boundary, hop)


@pytest.mark.parametrize("prec,n", [("f32", 512), ("f32", 400), ("f64", 1009)])
def test_host_memory_gives_the_same_bits(prec, n):
    p = plan(prec, n)
    hop = n // 4
    x = reals(prec, (3, 20 * n + 3), 18)
    w = hann(prec, n)
    dev, frames = dev_stft(p, x, w, hop)
    host = np.full((3, frames, n // 2 + 1), np.nan, SPEC[prec])
    p.stft(x, w, hop, host)
    assert np.array_equal(host.view(REAL[prec]), dev.cpu().numpy().view(REAL[prec]))
    yd = dev_istft(p, dev, w, hop, x.shape[-1]).cpu().numpy()
    yh = np.full(x.shape, np.nan, REAL[prec])
    p.istft(dev.cpu().numpy(), w, hop, yh)
    assert np.array_equal(yh, yd)


def test_host_row_above_the_staging_chunk():
    """rows of 17.5 M f32 samples (70 MB) and their 68 MB of spectra are staged one row at a time"""
    n, hop = 512, 512
    p = plan("f32", n)
    x = reals("f32", (2, 35 << 19), 19)
    w = hann("f32", n)
    dev, frames = dev_stft(p, x, w, hop)
    host = np.full((2, frames, n // 2 + 1), np.nan, np.complex64)
    p.stft(x, w, hop, host)
    assert np.array_equal(host.view(np.float32), dev.cpu().numpy().view(np.float32))
    yd = dev_istft(p, dev, w, hop, x.shape[-1]).cpu().numpy()
    yh = np.full(x.shape, np.nan, np.float32)
    p.istft(dev.cpu().numpy(), w, hop, yh)
    assert np.array_equal(yh, yd)


def test_inverse_in_two_scratch_runs():
    """f32 N = 2^21 at H = N/2: 70 frames of 8 MB do not fit the 512 MB scratch, so the row is inverted in two runs of
    frames; it must equal the frames inverted in one piece per run by the plan's irfft, overlap-added in float64."""
    torch = torch_mod()
    n = 1 << 21
    hop = n // 2
    p = plan("f32", n)
    L = hop * 69
    x = reals("f32", (1, L), 20)
    w = hann("f32", n)
    spec, frames = dev_stft(p, x, w, hop)
    assert frames == 70
    y = dev_istft(p, spec, w, hop, L)
    n_inv = launches(p)
    yn = y.cpu().numpy()
    assert np.abs(yn - x).max() / np.abs(x).max() < 1e-4
    # the runs: frames [0, 63) and [62, 70)
    parts = []
    run_launches = 0
    for gs, ge in ((0, 63), (62, 70)):
        v = torch.empty(ge - gs, n, dtype=torch.float32, device="cuda")
        p.irfft(spec[0, gs:ge].contiguous(), v)
        run_launches += launches(p) + 1
        parts.append((gs, v.double()))
    assert n_inv == run_launches
    wt = torch.from_numpy(w.astype(np.float64)).cuda()
    num = torch.zeros(hop * 69 + n, dtype=torch.float64, device="cuda")
    den = torch.zeros_like(num)
    for f in range(frames):
        gs, v = parts[0] if f < 63 else parts[1]
        num[f * hop:f * hop + n] += wt * v[f - gs]
        den[f * hop:f * hop + n] += wt * wt
    ref = torch.where(den >= 1e-11, num / den, torch.zeros_like(num))[n // 2:n // 2 + L].cpu().numpy()
    assert np.abs(yn - ref).max() / np.abs(ref).max() < 1e-5
    del spec, y, parts


def test_async_on_a_side_stream():
    torch = torch_mod()
    p = plan("f32", 512)
    x = reals("f32", (4, 9000), 21)
    w = hann("f32", 512)
    ref, frames = dev_stft(p, x, w, 128)
    yref = dev_istft(p, ref, w, 128, 9000)
    s = torch.cuda.Stream()
    xd, wd = torch.from_numpy(x).cuda(), torch.from_numpy(w).cuda()
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        out = torch.full((4, frames, 257), complex(float("nan"), float("nan")), dtype=torch.complex64, device="cuda")
        y = torch.full((4, 9000), float("nan"), dtype=torch.float32, device="cuda")
        p.stft(xd, wd, 128, out)
        p.istft(out, wd, 128, y)
    s.synchronize()
    assert torch.equal(torch.view_as_real(out), torch.view_as_real(ref))
    assert torch.equal(y, yref)


def test_launch_counts_fused():
    p = plan("f32", 512)
    x = reals("f32", (2, 5000), 22)
    w = hann("f32", 512)
    spec, frames = dev_stft(p, x, w, 128)
    assert launches(p) == 1
    dev_istft(p, spec, w, 128, 5000)
    assert launches(p) == 2   # the fused irfft and one overlap-add


def test_refusals():
    torch = torch_mod()
    p = plan("f32", 512)
    x = torch.zeros(2, 1000, device="cuda")
    w = torch.ones(512, device="cuda")
    frames = p.stft_frames(1000, 128)
    out = torch.empty(2, frames, 257, dtype=torch.complex64, device="cuda")
    with pytest.raises(ValueError, match="hop"):
        p.stft(x, w, 0, out)
    with pytest.raises(ValueError, match="last dimension"):
        p.stft(x, torch.ones(400, device="cuda"), 128, out)
    with pytest.raises(ValueError, match="output"):
        p.stft(x, w, 128, out[:, :-1])
    with pytest.raises(ValueError, match="pad_mode"):
        p.stft(x, w, 128, out, pad_mode="circular")
    with pytest.raises(ValueError, match="center=False"):
        p.stft(torch.zeros(2, 500, device="cuda"), w, 128, out, center=False)
    with pytest.raises(ValueError, match="reflect"):
        p.stft(torch.zeros(2, 256, device="cuda"), w, 128, out)
    with pytest.raises(ValueError, match="host or all be device"):
        p.stft(x, np.ones(512, np.float32), 128, out)
    with pytest.raises(ValueError, match="conj"):
        p.istft(out.conj(), w, 128, torch.empty(2, 1000, device="cuda"))
    with pytest.raises(ValueError, match="leading"):
        p.istft(out, w, 128, torch.empty(3, 1000, device="cuda"))
    # the C entry points check in_len against N themselves
    L = _lib.load()
    rc = L.fourier_b200_stft_float(p._plan, x.data_ptr(), 500, w.data_ptr(), 128, 0, out.data_ptr(), 0)
    assert rc == 1 and "in_len >= N" in _lib.last_error()
    rc = L.fourier_b200_stft_float(p._plan, x.data_ptr(), 256, w.data_ptr(), 128, 2, out.data_ptr(), 0)
    assert rc == 1 and "in_len > N/2" in _lib.last_error()
    rc = L.fourier_b200_stft_float(p._plan, x.data_ptr(), 1000, w.data_ptr(), 128, 1, x.data_ptr(), 2)
    assert rc == 1 and "overlap" in _lib.last_error()

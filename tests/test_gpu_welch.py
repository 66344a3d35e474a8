"""Welch power spectral density of real rows (RealFft.welch, fourier_b200_welch_*) on the GPU: every fused size class,
the half-length and full-length paths, against scipy.signal.welch in float64 on the same (rounded) inputs; a DC offset
of 1e4 that only a detrend in the time domain survives; rows of a periodic batch bit for bit against the same row run
alone; host against device memory bit for bit, a side stream, both scratch chunk loops, the plan's own stft, leading
shapes, batch 0, launch counts and refusals.  Every output is NaN-filled before the call, and a guard region behind it
must stay untouched."""

import numpy as np
import pytest

import fourier_b200 as fb
from fourier_b200 import _lib

pytestmark = pytest.mark.gpu

TOL = {"f32": 2e-5, "f64": 1e-12}
REAL = {"f32": np.float32, "f64": np.float64}
# (N, FFTs per CTA of its fused class)
FUSED = [("f32", 128, 32), ("f32", 256, 32), ("f32", 512, 16), ("f32", 1024, 16), ("f32", 2048, 8), ("f64", 128, 32),
         ("f64", 256, 32), ("f64", 512, 16)]
ARGS = (("constant", "density", 2.5), (False, "density", 1.0), ("constant", "spectrum", 1.0), (False, "spectrum", 2.5))
GUARD = 64


def torch_mod():
    import torch
    return torch


def tdt(prec):
    return getattr(torch_mod(), np.dtype(REAL[prec]).name)


def plan(prec, n):
    return fb.create_rfft_f32(n) if prec == "f32" else fb.create_rfft_f64(n)


def reals(prec, shape, seed, dc=0.0):
    return (dc + np.random.default_rng(seed).standard_normal(shape)).astype(REAL[prec])


def hann(prec, n):
    return torch_mod().hann_window(n, dtype=torch_mod().float64).numpy().astype(REAL[prec])


def ref_welch(x, w, hop, fs, scaling, detrend):
    """scipy.signal.welch in float64 where it takes the hop (hop <= N); the same definition in numpy beyond"""
    x = np.asarray(x, np.float64)
    w = np.asarray(w, np.float64)
    n = len(w)
    if hop <= n:
        from scipy.signal import welch
        return welch(x, fs, window=w, nperseg=n, noverlap=n - hop, detrend=detrend, scaling=scaling, axis=-1)[1]
    frames = np.lib.stride_tricks.sliding_window_view(x, n, axis=-1)[..., ::hop, :]
    if detrend == "constant":
        frames = frames - frames.mean(axis=-1, keepdims=True)
    p = (np.abs(np.fft.rfft(frames * w, axis=-1)) ** 2).mean(axis=-2)
    p *= 1.0 / (fs * (w * w).sum()) if scaling == "density" else 1.0 / w.sum() ** 2
    p[..., 1:(n + 1) // 2] *= 2
    return p


def dev_welch(p, x, w, hop, fs=1.0, scaling="density", detrend="constant"):
    """device welch of numpy x into a NaN-filled output followed by a guard region -> numpy output"""
    torch = torch_mod()
    shape = x.shape[:-1] + (p.size() // 2 + 1,)
    count = int(np.prod(shape, dtype=np.int64))
    buf = torch.full((count + GUARD,), float("nan"), dtype=tdt(p.real), device="cuda")
    buf[count:] = 12345.0
    out = buf[:count].view(shape)
    p.welch(torch.from_numpy(x).cuda(), torch.from_numpy(w).cuda(), hop, out, fs=fs, scaling=scaling, detrend=detrend)
    torch.cuda.synchronize()
    assert torch.all(buf[count:] == 12345.0), "a write past the output"
    return out.cpu().numpy()


def row_err(got, ref):
    """per row max |got - ref| / max |ref|; NaN counts as infinite"""
    g = np.asarray(got, np.float64).reshape(-1, np.shape(ref)[-1])
    r = np.asarray(ref, np.float64).reshape(g.shape)
    e = np.abs(g - r).max(axis=1) / np.maximum(np.abs(r).max(axis=1), 1e-300)
    return float(np.where(np.isnan(e), np.inf, e).max())


def launches(p):
    return p.info()["last_launches"]


def rfft_launches(p, rows):
    torch = torch_mod()
    p.rfft(torch.zeros(rows, p.size(), dtype=tdt(p.real), device="cuda"),
           torch.empty(rows, p.size() // 2 + 1, dtype=torch.complex64 if p.real == "f32" else torch.complex128,
                       device="cuda"))
    return launches(p)


def row_len(n, hop, frames):
    return n + (frames - 1) * hop + hop // 2


@pytest.mark.parametrize("prec,n,c", FUSED)
@pytest.mark.parametrize("detrend,scaling,fs", ARGS)
def test_fused_size_classes(prec, n, c, detrend, scaling, fs):
    """the emulator's hops and row lengths: F = 1, F < C, B-1, B, B+1 and 2B+3 (B = 4C) at hop N/4, F < C and B+1 at
    hops 1, N/2, N and N+3; one call per case, with the launch count of one or several items per row"""
    p = plan(prec, n)
    assert p.info()["path_name"] == "real_fused"
    w = hann(prec, n) + REAL[prec](0.25)
    b = 4 * c
    seed = 0
    for hop in (1, n // 4, n // 2, n, n + 3):
        for frames in ((1, c // 2 + 1, b - 1, b, b + 1, 2 * b + 3) if hop == n // 4 else (c // 2 + 1, b + 1)):
            seed += 1
            rows = c + 1 if frames == 1 else 3
            x = reals(prec, (rows, row_len(n, hop, frames)), seed, dc=0.5)
            got = dev_welch(p, x, w, hop, fs, scaling, detrend)
            assert launches(p) == (3 if frames > b else 2), (hop, frames)
            err = row_err(got, ref_welch(x, w, hop, fs, scaling, detrend))
            assert err < TOL[prec], (hop, frames, err)


@pytest.mark.parametrize("prec,n,path", (("f32", 400, "real_half"), ("f64", 400, "real_half"), ("f32", 4096, "real_half"),
                                         ("f32", 97, "real_full"), ("f64", 97, "real_full"), ("f32", 1001, "real_full")))
@pytest.mark.parametrize("detrend,scaling,fs", ARGS[:2])
def test_other_paths(prec, n, path, detrend, scaling, fs):
    p = plan(prec, n)
    assert p.info()["path_name"] == path
    w = hann(prec, n)
    for hop, frames in ((n // 4, 1), (n // 4, 50), (n // 2, 7), (n + 3, 3)):
        x = reals(prec, (3, row_len(n, hop, frames)), n + hop + frames, dc=0.5)
        got = dev_welch(p, x, w, hop, fs, scaling, detrend)
        err = row_err(got, ref_welch(x, w, hop, fs, scaling, detrend))
        assert err < TOL[prec], (hop, frames, err)


def test_dc_offset_needs_the_detrend_in_the_time_domain():
    """f32 N = 512, Hann, unit noise on a DC offset of 1e4, detrend constant: every bin k >= 4 within 1e-5 of scipy in
    float64 on the same f32 inputs.  Subtracting mu * rfft(w) from the spectrum instead fails this."""
    n, hop = 512, 256
    p = plan("f32", n)
    w = hann("f32", n)
    x = reals("f32", (4, n + 39 * hop), 77, dc=1e4)
    got = dev_welch(p, x, w, hop)
    ref = ref_welch(x, w, hop, 1.0, "density", "constant")
    rel = np.abs(got[:, 4:].astype(np.float64) - ref[:, 4:]) / ref[:, 4:]
    assert rel.max() <= 1e-5, rel.max()


@pytest.mark.parametrize("prec,n,hop,frames", (("f32", 512, 128, 5), ("f32", 512, 128, 131), ("f32", 128, 7, 1),
                                               ("f64", 256, 64, 300), ("f32", 400, 160, 40)))
def test_rows_of_a_periodic_batch_equal_the_row_alone(prec, n, hop, frames):
    """97 rows repeating 5 base rows, short rows packed several to a group and rows of many items: every row equals its
    base row run alone, bit for bit"""
    p = plan(prec, n)
    w = hann(prec, n)
    base = reals(prec, (5, row_len(n, hop, frames)), frames + n)
    x = base[np.arange(97) % 5]
    got = dev_welch(p, x, w, hop)
    alone = np.stack([dev_welch(p, base[i:i + 1], w, hop)[0] for i in range(5)])
    assert np.array_equal(got, alone[np.arange(97) % 5])
    assert row_err(alone, ref_welch(base, w, hop, 1.0, "density", "constant")) < TOL[prec]


@pytest.mark.parametrize("prec,n", (("f32", 512), ("f64", 512), ("f32", 400), ("f32", 97)))
def test_host_memory_gives_the_same_bits(prec, n):
    p = plan(prec, n)
    hop = n // 4
    x = reals(prec, (3, 20 * n + 3), 39, dc=1.0)
    w = hann(prec, n)
    dev = dev_welch(p, x, w, hop, 2.0, "spectrum")
    host = np.full((3, n // 2 + 1), np.nan, REAL[prec])
    p.welch(x, w, hop, host, fs=2.0, scaling="spectrum")
    assert np.array_equal(host, dev)


def test_host_row_above_the_staging_chunk():
    """rows of 17.5 M f32 samples (70 MB) are staged one row at a time"""
    n, hop = 512, 512
    p = plan("f32", n)
    x = reals("f32", (2, 35 << 19), 40)
    w = hann("f32", n)
    dev = dev_welch(p, x, w, hop)
    host = np.full((2, n // 2 + 1), np.nan, np.float32)
    p.welch(x, w, hop, host)
    assert launches(p) == 1 + 2 * 2   # the scale, then per staged row the fused kernel and the finish
    assert np.array_equal(host, dev)
    assert row_err(dev, ref_welch(x, w, hop, 1.0, "density", "constant")) < TOL["f32"]


def test_async_on_a_side_stream():
    torch = torch_mod()
    p = plan("f32", 512)
    x = reals("f32", (4, 9000), 41)
    w = hann("f32", 512)
    ref = dev_welch(p, x, w, 128)
    s = torch.cuda.Stream()
    xd, wd = torch.from_numpy(x).cuda(), torch.from_numpy(w).cuda()
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        out = torch.full((4, 257), float("nan"), dtype=torch.float32, device="cuda")
        p.welch(xd, wd, 128, out)
    s.synchronize()
    assert np.array_equal(out.cpu().numpy(), ref)


def test_real_half_two_scratch_chunks():
    """60 rows of 2998 frames at N = 400: frames and spectra of 3208 bytes each fill the 512 MB scratch after 167354
    frames, and the item of 12 frames that straddles the cut is continued in the second chunk"""
    p = plan("f32", 400)
    rows = 60
    x = reals("f32", (rows, 480000), 33, dc=0.5)
    w = hann("f32", 400)
    got = dev_welch(p, x, w, 160)
    n_welch = launches(p)
    frames = 1 + (480000 - 400) // 160
    chunk = (512 << 20) // (400 * 4 + 201 * 8)
    total = rows * frames
    assert chunk < total and (chunk % frames) % 12 != 0
    assert n_welch == 2 + (2 + rfft_launches(p, chunk)) + (2 + rfft_launches(p, total - chunk))
    for r in (0, chunk // frames, chunk // frames + 1, rows - 1):
        assert row_err(got[r:r + 1], ref_welch(x[r:r + 1], w, 160, 1.0, "density", "constant")) < TOL["f32"], r


@pytest.mark.parametrize("prec,n", (("f32", 512), ("f64", 256), ("f32", 400)))
def test_matches_the_plans_stft(prec, n):
    """detrend False: the plan's own stft(center=False), |S|^2, the mean over frames, one-sided and scaled"""
    torch = torch_mod()
    p = plan(prec, n)
    hop = n // 2
    x = reals(prec, (3, 40 * n + 5), 51)
    w = hann(prec, n)
    got = dev_welch(p, x, w, hop, 4.0, "density", False)
    frames = p.stft_frames(x.shape[-1], hop, center=False)
    S = torch.empty((3, frames, n // 2 + 1), dtype=torch.complex64 if prec == "f32" else torch.complex128,
                    device="cuda")
    p.stft(torch.from_numpy(x).cuda(), torch.from_numpy(w).cuda(), hop, S, center=False)
    pw = (S.abs().double() ** 2).mean(-2).cpu().numpy() / (4.0 * (w.astype(np.float64) ** 2).sum())
    pw[..., 1:(n + 1) // 2] *= 2
    assert row_err(got, pw) < TOL[prec]


def test_leading_shapes_and_batch_zero():
    torch = torch_mod()
    p = plan("f32", 256)
    w = hann("f32", 256)
    x = reals("f32", (2, 3, 1500), 61)
    got = dev_welch(p, x, w, 100)
    assert got.shape == (2, 3, 129)
    assert np.array_equal(got.reshape(6, 129), dev_welch(p, x.reshape(6, 1500), w, 100))
    out = torch.full((0, 129), float("nan"), device="cuda")
    p.welch(torch.empty((0, 1500), device="cuda"), torch.from_numpy(w).cuda(), 100, out)
    # the C entry point at batch 0 succeeds and launches nothing
    L = _lib.load()
    wd = torch.from_numpy(w).cuda()
    xd = torch.zeros(1500, device="cuda")
    o = torch.empty(129, device="cuda")
    assert L.fourier_b200_welch_float(p._plan, xd.data_ptr(), 1500, wd.data_ptr(), 100, 1, 0, 1.0, o.data_ptr(), 0) == 0
    assert launches(p) == 0


def test_refusals():
    torch = torch_mod()
    p = plan("f32", 512)
    x = torch.zeros(2, 1000, device="cuda")
    w = torch.ones(512, device="cuda")
    out = torch.empty(2, 257, device="cuda")
    with pytest.raises(ValueError, match="last dimension"):
        p.welch(x, w, 128, torch.empty(2, 256, device="cuda"))
    with pytest.raises(ValueError, match="leading"):
        p.welch(x, w, 128, torch.empty(3, 257, device="cuda"))
    with pytest.raises(ValueError, match="window"):
        p.welch(x, torch.ones(2, 512, device="cuda"), 128, out)
    with pytest.raises(TypeError, match="expected"):
        p.welch(x, w, 128, out.double())
    with pytest.raises(ValueError, match="at least N"):
        p.welch(torch.zeros(2, 500, device="cuda"), w, 128, out)
    with pytest.raises(ValueError, match="hop"):
        p.welch(x, w, 0, out)
    with pytest.raises(ValueError, match="scaling"):
        p.welch(x, w, 128, out, scaling="power")
    with pytest.raises(ValueError, match="detrend"):
        p.welch(x, w, 128, out, detrend="linear")
    with pytest.raises(ValueError, match="detrend"):
        p.welch(x, w, 128, out, detrend=True)
    for fs in (0.0, -1.0, float("inf"), float("nan")):
        with pytest.raises(ValueError, match="fs"):
            p.welch(x, w, 128, out, fs=fs)
    with pytest.raises(ValueError, match="host or all be device"):
        p.welch(x, w.cpu().numpy(), 128, out)
    with pytest.raises(ValueError, match="conj"):
        p.welch(x, w._neg_view(), 128, out)
    # the C entry points check the overlap and a mix of host and device memory themselves
    L = _lib.load()
    rc = L.fourier_b200_welch_float(p._plan, x.data_ptr(), 1000, w.data_ptr(), 128, 1, 0, 1.0, x.data_ptr(), 1)
    assert rc == 1 and "overlap" in _lib.last_error()
    host = np.zeros(257, np.float32)
    rc = L.fourier_b200_welch_float(p._plan, x.data_ptr(), 1000, w.data_ptr(), 128, 1, 0, 1.0, host.ctypes.data, 1)
    assert rc == 1 and "host or all be device" in _lib.last_error()

"""Mel spectrogram of real rows (RealFft.mel_spectrogram, fourier_b200_mel_spectrogram_*) on the GPU: every fused size
class, the half-length and full-length paths, against float64 numpy (frames -> rfft -> |.|^p -> @ filters.T) with
torchaudio's HTK and Slaney banks; torchaudio's MelSpectrogram itself; Whisper's shape, also over two scratch chunks;
the plan's own stft; banks that are not triangular; leading shapes, batch 0, host against device memory bit for bit,
a side stream, launch counts and refusals.  Every output is NaN-filled before the call, and a guard region behind it
must stay untouched."""

import numpy as np
import pytest

import fourier_b200 as fb
from fourier_b200 import _lib

pytestmark = pytest.mark.gpu

TOL = {"f32": 2e-5, "f64": 1e-12}
REAL = {"f32": np.float32, "f64": np.float64}
BOUNDARIES = (("none", False, "reflect"), ("zeros", True, "constant"), ("reflect", True, "reflect"))
FUSED = [("f32", n) for n in (128, 256, 512, 1024, 2048)] + [("f64", n) for n in (128, 256, 512)]
GUARD = 64


def torch_mod():
    import torch
    return torch


def tdt(prec):
    return getattr(torch_mod(), np.dtype(REAL[prec]).name)


def plan(prec, n):
    return fb.create_rfft_f32(n) if prec == "f32" else fb.create_rfft_f64(n)


def reals(prec, shape, seed):
    return np.random.default_rng(seed).standard_normal(shape).astype(REAL[prec])


def hann(prec, n):
    return torch_mod().hann_window(n, dtype=torch_mod().float64).numpy().astype(REAL[prec])


def bank(prec, n, n_mels, scale="htk", sr=16000):
    """torchaudio's triangular bank as (n_mels, N//2+1)"""
    import torchaudio
    fbk = torchaudio.functional.melscale_fbanks(n // 2 + 1, 0.0, sr / 2, n_mels, sr,
                                                norm="slaney" if scale == "slaney" else None, mel_scale=scale)
    return fbk.T.contiguous().double().numpy().astype(REAL[prec])


def ref_mel(x, w, hop, center, pad_mode, filters, power):
    """float64 numpy: pad, frames every hop, times the window, rfft, |.|^p, @ filters.T; frame-major"""
    x = np.asarray(x, np.float64)
    n = len(w)
    if center:
        x = np.pad(x, [(0, 0)] * (x.ndim - 1) + [(n // 2, n // 2)], mode=pad_mode)
    frames = np.lib.stride_tricks.sliding_window_view(x, n, axis=-1)[..., ::hop, :]
    mag = np.abs(np.fft.rfft(frames * np.asarray(w, np.float64), axis=-1)) ** power
    return mag @ np.asarray(filters, np.float64).T


def dev_mel(p, x, w, hop, filters, power=2, center=True, pad_mode="reflect"):
    """device mel of numpy x into a NaN-filled output followed by a guard region -> (numpy output, frames)"""
    torch = torch_mod()
    n_mels = filters.shape[0]
    frames = p.stft_frames(x.shape[-1], hop, center)
    shape = x.shape[:-1] + (frames, n_mels)
    count = int(np.prod(shape, dtype=np.int64))
    buf = torch.full((count + GUARD,), float("nan"), dtype=tdt(p.real), device="cuda")
    buf[count:] = 12345.0
    out = buf[:count].view(shape)
    p.mel_spectrogram(torch.from_numpy(x).cuda(), torch.from_numpy(w).cuda(), hop, torch.from_numpy(filters).cuda(), out,
                      power=power, center=center, pad_mode=pad_mode)
    torch.cuda.synchronize()
    assert torch.all(buf[count:] == 12345.0), "a write past the output"
    return out.cpu().numpy(), frames


def row_err(got, ref):
    """per input row (all its frames and mels) max |got - ref| / max |ref|; NaN counts as infinite"""
    lead = int(np.prod(np.shape(ref)[:-2], dtype=np.int64)) or 1
    g = np.asarray(got, np.float64).reshape(lead, -1)
    r = np.asarray(ref, np.float64).reshape(lead, -1)
    e = np.abs(g - r).max(axis=1) / np.maximum(np.abs(r).max(axis=1), 1e-300)
    return float(np.where(np.isnan(e), np.inf, e).max())


def launches(p):
    return p.info()["last_launches"]


@pytest.mark.parametrize("prec,n", FUSED)
@pytest.mark.parametrize("boundary,center,pad_mode", BOUNDARIES)
@pytest.mark.parametrize("power,scale", ((2, "htk"), (1, "slaney"), (2, "slaney"), (1, "htk")))
def test_fused_size_classes(prec, n, boundary, center, pad_mode, power, scale):
    p = plan(prec, n)
    assert p.info()["path_name"] == "real_fused"
    hop = n // 4
    x = reals(prec, (3, 3 * n + 17), n)
    w = hann(prec, n)
    f = bank(prec, n, 40, scale)
    got, frames = dev_mel(p, x, w, hop, f, power, center, pad_mode)
    assert launches(p) == 2
    ref = ref_mel(x, w, hop, center, pad_mode, f, power)
    assert got.shape == ref.shape
    assert row_err(got, ref) < TOL[prec]


@pytest.mark.parametrize("n_fft,hop,n_mels,path", ((400, 200, 128, "real_half"), (512, 128, 80, "real_fused")))
def test_torchaudio_mel_spectrogram(n_fft, hop, n_mels, path):
    """the module at its defaults (N = 400: 4 all-zero mel rows) and at N = 512, in float64 on the CPU, with the
    module's own window and bank"""
    import torch
    import torchaudio
    m = torchaudio.transforms.MelSpectrogram(sample_rate=16000, n_fft=n_fft, hop_length=hop, n_mels=n_mels).double()
    window = m.spectrogram.window.numpy()
    filters = m.mel_scale.fb.T.contiguous().numpy()
    if n_fft == 400:
        assert (np.abs(filters).sum(axis=1) == 0).sum() == 4
    x = reals("f64", (2, 16000), 31)
    want = m(torch.from_numpy(x)).transpose(-1, -2).numpy()
    p = plan("f64", n_fft)
    assert p.info()["path_name"] == path
    got, _ = dev_mel(p, x, window, hop, filters)
    assert got.shape == want.shape
    assert row_err(got, want) < 1e-12
    assert np.all(got[..., np.abs(filters).sum(axis=1) == 0] == 0.0)


def rfft_launches(p, rows):
    torch = torch_mod()
    p.rfft(torch.zeros(rows, p.size(), dtype=tdt(p.real), device="cuda"),
           torch.empty(rows, p.size() // 2 + 1, dtype=torch.complex64 if p.real == "f32" else torch.complex128,
                       device="cuda"))
    return launches(p)


def test_whisper_shape():
    p = plan("f32", 400)
    assert p.info()["path_name"] == "real_half"
    x = reals("f32", (2, 480000), 32)
    w = hann("f32", 400)
    f = bank("f32", 400, 80, "slaney")
    got, frames = dev_mel(p, x, w, 160, f)
    assert frames == 3001
    n_mel = launches(p)
    assert row_err(got, ref_mel(x, w, 160, True, "reflect", f, 2)) < TOL["f32"]
    assert n_mel == 1 + 2 + rfft_launches(p, 2 * frames)   # bands; one chunk: gather, rfft, mels


def test_whisper_shape_two_scratch_chunks():
    """60 rows of 3001 frames: frames and spectra of 3208 bytes each fill the 512 MB scratch after 167354 frames"""
    p = plan("f32", 400)
    rows = 60
    x = reals("f32", (rows, 480000), 33)
    w = hann("f32", 400)
    f = bank("f32", 400, 80, "slaney")
    got, frames = dev_mel(p, x, w, 160, f)
    n_mel = launches(p)
    chunk = (512 << 20) // (400 * 4 + 201 * 8)
    total = rows * frames
    assert chunk < total
    assert n_mel == 1 + (2 + rfft_launches(p, chunk)) + (2 + rfft_launches(p, total - chunk))
    for r in (0, chunk // frames, chunk // frames + 1, rows - 1):
        assert row_err(got[r:r + 1], ref_mel(x[r:r + 1], w, 160, True, "reflect", f, 2)) < TOL["f32"], r


@pytest.mark.parametrize("prec", ("f32", "f64"))
@pytest.mark.parametrize("boundary,center,pad_mode", BOUNDARIES)
def test_real_full_odd_n(prec, boundary, center, pad_mode):
    p = plan(prec, 401)
    assert p.info()["path_name"] == "real_full"
    x = reals(prec, (2, 5000), 34)
    w = hann(prec, 401)
    f = bank(prec, 401, 64, "htk")
    for power in (1, 2):
        got, _ = dev_mel(p, x, w, 100, f, power, center, pad_mode)
        assert row_err(got, ref_mel(x, w, 100, center, pad_mode, f, power)) < TOL[prec], power


@pytest.mark.parametrize("prec,n", [("f32", 512), ("f32", 400), ("f64", 512), ("f64", 401)])
def test_equals_power_of_the_plans_stft(prec, n):
    torch = torch_mod()
    p = plan(prec, n)
    x = reals(prec, (2, 7000), 35)
    w = hann(prec, n)
    f = bank(prec, n, 80, "slaney")
    frames = p.stft_frames(7000, n // 4)
    S = torch.empty(2, frames, n // 2 + 1, dtype=torch.complex64 if prec == "f32" else torch.complex128, device="cuda")
    p.stft(torch.from_numpy(x).cuda(), torch.from_numpy(w).cuda(), n // 4, S)
    mag = np.abs(S.cpu().numpy().astype(np.complex128))
    for power in (1, 2):
        got, _ = dev_mel(p, x, w, n // 4, f, power)
        assert row_err(got, (mag ** power) @ f.astype(np.float64).T) < TOL[prec], power


def odd_banks(prec, n, seed):
    """dense random; zero rows, single weights at bins 0 and N/2 and negative bands (N/2+6 rows); one row"""
    rng = np.random.default_rng(seed)
    bins = n // 2 + 1
    dense = rng.standard_normal((7, bins))
    special = np.zeros((bins + 5, bins))
    for m in range(bins + 5):
        kind = m % 5
        if kind == 1:
            special[m, 0] = 1.5
        elif kind == 2:
            special[m, bins - 1] = 0.75
        elif kind == 3:
            lo = int(rng.integers(0, bins))
            special[m, lo:lo + 9] = -rng.random(min(9, bins - lo))
        elif kind == 4:
            special[m, m % bins] = 0.5
    one = rng.random((1, bins))
    return [(name, b.astype(REAL[prec])) for name, b in (("dense", dense), ("special", special), ("one", one))]


@pytest.mark.parametrize("prec,n", [("f32", 512), ("f32", 400), ("f64", 256), ("f64", 401)])
def test_banks_that_are_not_triangular(prec, n):
    p = plan(prec, n)
    x = reals(prec, (3, 3000), 36)
    w = hann(prec, n)
    for name, f in odd_banks(prec, n, 37):
        for power in (1, 2):
            got, _ = dev_mel(p, x, w, 97, f, power)
            assert row_err(got, ref_mel(x, w, 97, True, "reflect", f, power)) < TOL[prec], (name, power)
            zero = np.abs(f).sum(axis=1) == 0
            assert np.all(got[..., zero] == 0.0), name


def test_leading_shapes_and_batch_zero():
    torch = torch_mod()
    p = plan("f32", 256)
    x = reals("f32", (2, 3, 1000), 38)
    w = hann("f32", 256)
    f = bank("f32", 256, 32)
    got, frames = dev_mel(p, x, w, 300, f)
    assert got.shape == (2, 3, frames, 32)
    assert row_err(got, ref_mel(x, w, 300, True, "reflect", f, 2)) < TOL["f32"]
    wd, fd = torch.from_numpy(w).cuda(), torch.from_numpy(f).cuda()
    p.mel_spectrogram(torch.zeros(0, 1000, device="cuda"), wd, 300, fd, torch.empty(0, frames, 32, device="cuda"))
    # the C entry point at batch 0: succeeds and launches nothing
    xd, out = torch.zeros(1, 1000, device="cuda"), torch.full((1, frames, 32), float("nan"), device="cuda")
    rc = _lib.load().fourier_b200_mel_spectrogram_float(p._plan, xd.data_ptr(), 1000, wd.data_ptr(), 300, 2, 2,
                                                         fd.data_ptr(), 32, out.data_ptr(), 0)
    assert rc == 0 and launches(p) == 0
    assert torch.isnan(out).all()


@pytest.mark.parametrize("prec,n", [("f32", 512), ("f32", 400), ("f64", 401)])
def test_host_memory_gives_the_same_bits(prec, n):
    p = plan(prec, n)
    hop = n // 4
    x = reals(prec, (3, 20 * n + 3), 39)
    w = hann(prec, n)
    f = bank(prec, n, 80, "slaney")
    dev, frames = dev_mel(p, x, w, hop, f)
    host = np.full((3, frames, 80), np.nan, REAL[prec])
    p.mel_spectrogram(x, w, hop, f, host)
    assert np.array_equal(host, dev)


def test_host_row_above_the_staging_chunk():
    """rows of 17.5 M f32 samples (70 MB) are staged one row at a time"""
    n, hop = 512, 512
    p = plan("f32", n)
    x = reals("f32", (2, 35 << 19), 40)
    w = hann("f32", n)
    f = bank("f32", n, 80)
    dev, frames = dev_mel(p, x, w, hop, f)
    host = np.full((2, frames, 80), np.nan, np.float32)
    p.mel_spectrogram(x, w, hop, f, host)
    assert np.array_equal(host, dev)


def test_async_on_a_side_stream():
    torch = torch_mod()
    p = plan("f32", 512)
    x = reals("f32", (4, 9000), 41)
    w = hann("f32", 512)
    f = bank("f32", 512, 80)
    ref, frames = dev_mel(p, x, w, 128, f)
    s = torch.cuda.Stream()
    xd, wd, fd = torch.from_numpy(x).cuda(), torch.from_numpy(w).cuda(), torch.from_numpy(f).cuda()
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        out = torch.full((4, frames, 80), float("nan"), dtype=torch.float32, device="cuda")
        p.mel_spectrogram(xd, wd, 128, fd, out)
    s.synchronize()
    assert np.array_equal(out.cpu().numpy(), ref)


def test_refusals():
    torch = torch_mod()
    p = plan("f32", 512)
    x = torch.zeros(2, 1000, device="cuda")
    w = torch.ones(512, device="cuda")
    f = torch.ones(80, 257, device="cuda")
    frames = p.stft_frames(1000, 128)
    out = torch.empty(2, frames, 80, device="cuda")
    with pytest.raises(ValueError, match="last dimension"):
        p.mel_spectrogram(x, w, 128, torch.ones(80, 256, device="cuda"), out)
    with pytest.raises(ValueError, match="filters must have shape"):
        p.mel_spectrogram(x, w, 128, torch.ones(257, device="cuda"), out)
    with pytest.raises(TypeError, match="expected"):
        p.mel_spectrogram(x, w, 128, f.double(), out)
    with pytest.raises(ValueError, match="power"):
        p.mel_spectrogram(x, w, 128, f, out, power=3)
    with pytest.raises(ValueError, match="host or all be device"):
        p.mel_spectrogram(x, w, 128, f.cpu().numpy(), out)
    with pytest.raises(ValueError, match="output"):
        p.mel_spectrogram(x, w, 128, f, out[:, :-1])
    with pytest.raises(ValueError, match="last dimension"):
        p.mel_spectrogram(x, w, 128, f, torch.empty(2, frames, 79, device="cuda"))
    with pytest.raises(ValueError, match="hop"):
        p.mel_spectrogram(x, w, 0, f, out)
    # the C entry points check in_len against N and the overlap themselves
    L = _lib.load()
    rc = L.fourier_b200_mel_spectrogram_float(p._plan, x.data_ptr(), 500, w.data_ptr(), 128, 0, 2, f.data_ptr(), 80,
                                              out.data_ptr(), 0)
    assert rc == 1 and "in_len >= N" in _lib.last_error()
    rc = L.fourier_b200_mel_spectrogram_float(p._plan, x.data_ptr(), 1000, w.data_ptr(), 128, 1, 2, f.data_ptr(), 80,
                                              f.data_ptr(), 1)
    assert rc == 1 and "overlap" in _lib.last_error()

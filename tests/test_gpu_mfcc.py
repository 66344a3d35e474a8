"""MFCC and log-mel spectrogram of real rows (RealFft.mfcc, fourier_b200_mfcc_*) on the GPU: every fused size class, the
half-length and full-length paths and the chunked route of a fused plan (n_mels = N/2), against a float64 numpy
restatement of the definition (mel -> log -> group clamp -> projection); torchaudio's MFCC (both log_mels settings, and
the grouping rule on (3, 2, L) input); Whisper's log-mel; a clamp that binds; a group alone against the same group in a
larger batch, host against device memory (also a row above the staging chunk with the clamp on) and a side stream bit
for bit; leading shapes, batch 0, launch counts and refusals.  Every output is NaN-filled before the call, and a guard
region behind it must stay untouched."""
import math

import numpy as np
import pytest

from fourier_b200 import _lib
from test_gpu_mel import (FUSED, GUARD, REAL, TOL, bank, hann, launches, plan, reals, ref_mel, rfft_launches, row_err,
                          tdt, torch_mod)

pytestmark = pytest.mark.gpu

TEN_LN10 = 10.0 / math.log(10.0)
WHISPER_SCALE = 1.0 / (4.0 * math.log(10.0))


def dct_matrix(prec, n_mels, n_out):
    """librosa's orthonormal DCT-II matrix, (n_mels, n_out) = torchaudio's create_dct(n_out, n_mels, 'ortho')"""
    m = np.arange(n_mels)[:, None]
    j = np.arange(n_out)[None, :]
    d = np.cos(np.pi / n_mels * (m + 0.5) * j) * math.sqrt(2.0 / n_mels)
    d[:, 0] /= math.sqrt(2.0)
    return d.astype(REAL[prec])


def ref_mfcc(x, w, hop, filters, dct, power=2, center=True, pad_mode="reflect", log_scale=TEN_LN10, log_floor=1e-10,
             log_offset=0.0, top_db=80.0, top_db_rows=1, bias=0.0):
    """float64 numpy restatement of the definition: frame-major (..., F, n_out)"""
    mel = ref_mel(x, w, hop, center, pad_mode, filters, power)
    lm = log_scale * np.log(np.maximum(mel + log_offset, log_floor))
    if top_db is not None:
        g = lm.reshape((-1, top_db_rows) + lm.shape[-2:])
        theta = g.max(axis=(1, 2, 3), keepdims=True) - top_db
        lm = np.maximum(g, theta).reshape(lm.shape)
    return (lm if dct is None else lm @ np.asarray(dct, np.float64)) + bias


def dev_mfcc(p, x, w, hop, filters, dct, **kw):
    """device MFCC of numpy x into a NaN-filled output followed by a guard region -> (numpy output, frames)"""
    torch = torch_mod()
    center = kw.get("center", True)
    n_out = filters.shape[0] if dct is None else dct.shape[1]
    frames = p.stft_frames(x.shape[-1], hop, center)
    shape = x.shape[:-1] + (frames, n_out)
    count = int(np.prod(shape, dtype=np.int64))
    buf = torch.full((count + GUARD,), float("nan"), dtype=tdt(p.real), device="cuda")
    buf[count:] = 12345.0
    out = buf[:count].view(shape)
    p.mfcc(torch.from_numpy(x).cuda(), torch.from_numpy(w).cuda(), hop, torch.from_numpy(filters).cuda(),
           None if dct is None else torch.from_numpy(dct).cuda(), out, **kw)
    torch.cuda.synchronize()
    assert torch.all(buf[count:] == 12345.0), "a write past the output"
    return out.cpu().numpy(), frames


def check(p, x, w, hop, f, d, tol, **kw):
    got, frames = dev_mfcc(p, x, w, hop, f, d, **kw)
    ref = ref_mfcc(x, w, hop, f, d, **kw)
    assert got.shape == ref.shape
    err = row_err(got, ref)
    assert err < tol, err
    return got, frames


@pytest.mark.parametrize("prec,n", FUSED)
@pytest.mark.parametrize("top_db", (80.0, None))
@pytest.mark.parametrize("n_out", (13, None))
def test_fused_size_classes(prec, n, top_db, n_out):
    p = plan(prec, n)
    assert p.info()["path_name"] == "real_fused"
    x = reals(prec, (4, 3 * n + 17), n)
    w = hann(prec, n)
    f = bank(prec, n, 40)
    d = None if n_out is None else dct_matrix(prec, 40, n_out)
    check(p, x, w, n // 4, f, d, TOL[prec], top_db=top_db, top_db_rows=2, bias=1.5 if n_out is None else 0.0)
    assert launches(p) == (3 if top_db is not None else 2)


@pytest.mark.parametrize("prec,n,path", [("f32", 400, "real_half"), ("f64", 400, "real_half"), ("f32", 401, "real_full"),
                                         ("f64", 401, "real_full")])
@pytest.mark.parametrize("top_db", (80.0, None))
def test_chunked_paths(prec, n, path, top_db):
    p = plan(prec, n)
    assert p.info()["path_name"] == path
    x = reals(prec, (2, 5000), 51)
    w = hann(prec, n)
    f = bank(prec, n, 64)
    for d in (dct_matrix(prec, 64, 20), None):
        for power, center in ((2, True), (1, False)):
            check(p, x, w, 100, f, d, TOL[prec], power=power, center=center, top_db=top_db)
    mel = np.empty((2, p.stft_frames(5000, 100), 64), REAL[prec])
    p.mel_spectrogram(x, w, 100, f, mel)
    n_mel = launches(p)   # bands; one chunk: gather, rfft, mels
    dev_mfcc(p, x, w, 100, f, None, top_db=top_db)
    assert launches(p) == (2 * n_mel + 1 if top_db is not None else n_mel + 1)


@pytest.mark.parametrize("prec,n", [("f32", 512), ("f64", 256)])
def test_mel_count_at_the_fused_limit(prec, n):
    """n_mels = N/2 - 1 runs the fused kernel, n_mels = N/2 the chunked route of the same plan"""
    p = plan(prec, n)
    x = reals(prec, (2, 4 * n), 52)
    w = hann(prec, n)
    for n_mels, fused in ((n // 2 - 1, True), (n // 2, False)):
        f = bank(prec, n, n_mels)
        d = dct_matrix(prec, n_mels, 30)
        check(p, x, w, n // 4, f, d, TOL[prec])
        frames = p.stft_frames(4 * n, n // 4)
        assert launches(p) == (3 if fused else 1 + 2 * (3 + rfft_launches(p, 2 * frames))), n_mels


@pytest.mark.parametrize("n_fft,path", ((400, "real_half"), (512, "real_fused")))
@pytest.mark.parametrize("shape,rows", (((2, 16000), 2), ((3, 2, 16000), 2)))
def test_torchaudio_mfcc(n_fft, path, shape, rows):
    """torchaudio's MFCC in float64 on the CPU at its defaults (log_mels False, top_db 80 over each item's channels)
    and with log_mels True, with the module's own window, bank and DCT matrix"""
    import torch
    import torchaudio
    x = reals("f64", shape, 53)
    p = plan("f64", n_fft)
    assert p.info()["path_name"] == path
    for log_mels in (False, True):
        m = torchaudio.transforms.MFCC(sample_rate=16000, log_mels=log_mels,
                                       melkwargs={"n_fft": n_fft, "hop_length": n_fft // 2}).double()
        want = m(torch.from_numpy(x)).transpose(-1, -2).numpy()
        window = m.MelSpectrogram.spectrogram.window.numpy()
        filters = m.MelSpectrogram.mel_scale.fb.T.contiguous().numpy()
        dct = m.dct_mat.contiguous().numpy()
        if log_mels:
            kw = dict(log_scale=1.0, log_floor=np.finfo(np.float64).tiny, log_offset=1e-6, top_db=None)
        else:
            kw = dict(top_db_rows=rows)
        got, _ = dev_mfcc(p, x, window, n_fft // 2, filters, dct, **kw)
        assert got.shape == want.shape
        assert row_err(got, want) < 1e-12, log_mels


def test_whisper_log_mel():
    """Whisper's log10 -> max(., max - 8) -> (. + 4) / 4 on a 30 s clip; Whisper drops the last frame first, so the
    two agree on frames 0 .. F-2 while the maximum lies elsewhere"""
    p = plan("f32", 400)
    assert p.info()["path_name"] == "real_half"
    t = np.arange(480000) / 16000.0
    x = (np.sin(2 * np.pi * (200 + 50 * t) * t) * np.exp(-((t - 15) / 4) ** 2) +
         1e-4 * reals("f32", 480000, 54)).astype(np.float32)[None]
    w = hann("f32", 400)
    f = bank("f32", 400, 80, "slaney")
    got, frames = dev_mfcc(p, x, w, 160, f, None, log_scale=WHISPER_SCALE, top_db=2.0, bias=1.0)
    assert frames == 3001
    mel = ref_mel(x, w, 160, True, "reflect", f, 2)[..., :-1, :]
    log_spec = np.log10(np.maximum(mel, 1e-10))
    log_spec = np.maximum(log_spec, log_spec.max() - 8.0)
    want = (log_spec + 4.0) / 4.0
    # 1e-4 rather than 2e-5: the clamp keeps bins down to 80 dB below the clip's peak, where the f32 spectrum's own
    # rounding is a larger part of the power and the log shows it (3.4e-5 measured)
    assert row_err(got[..., :-1, :], want) < 1e-4


@pytest.mark.parametrize("prec,n", [("f32", 512), ("f64", 512), ("f32", 400)])
def test_clamp_that_binds(prec, n):
    """rows loud for their first half and 120 dB quieter for the rest: every entry the reference clamps (by more than
    1 dB, so that rounding cannot move it across) equals the row minimum bit for bit, and that minimum is within one
    ulp of the row's maximum - top_db"""
    p = plan(prec, n)
    x = reals(prec, (2, 40 * n), 55)
    x[:, 20 * n:] *= 1e-6
    w = hann(prec, n)
    f = bank(prec, n, 64)
    got, _ = check(p, x, w, n // 4, f, None, TOL[prec])
    lm = TEN_LN10 * np.log(np.maximum(ref_mel(x, w, n // 4, True, "reflect", f, 2), 1e-10))
    for b in range(2):
        theta = lm[b].max() - 80.0
        clamped = lm[b] < theta - 1.0
        assert clamped.sum() > lm[b].size // 4
        lo, hi = got[b].min(), float(got[b].max())
        assert np.all(got[b][clamped] == lo)
        assert abs(float(lo) - (hi - 80.0)) <= float(np.spacing(REAL[prec](abs(hi - 80.0)))), (lo, hi)


@pytest.mark.parametrize("prec,n", [("f32", 512), ("f32", 400)])
def test_group_alone_equals_group_in_a_batch(prec, n):
    p = plan(prec, n)
    x = reals(prec, (6, 9000), 56)
    x[3] *= 1e-3
    w = hann(prec, n)
    f = bank(prec, n, 80)
    d = dct_matrix(prec, 80, 40)
    full, _ = dev_mfcc(p, x, w, 128, f, d, top_db_rows=2)
    alone, _ = dev_mfcc(p, np.ascontiguousarray(x[2:4]), w, 128, f, d, top_db_rows=2)
    assert np.array_equal(full[2:4], alone)


@pytest.mark.parametrize("prec,n", [("f32", 512), ("f32", 400), ("f64", 401)])
def test_host_memory_gives_the_same_bits(prec, n):
    p = plan(prec, n)
    x = reals(prec, (4, 20 * n + 3), 57)
    w = hann(prec, n)
    f = bank(prec, n, 80, "slaney")
    d = dct_matrix(prec, 80, 13)
    for dd, top_db in ((d, 80.0), (None, None)):
        dev, frames = dev_mfcc(p, x, w, n // 4, f, dd, top_db=top_db, top_db_rows=2)
        host = np.full(dev.shape, np.nan, REAL[prec])
        p.mfcc(x, w, n // 4, f, dd, host, top_db=top_db, top_db_rows=2)
        assert np.array_equal(host, dev), top_db


def test_host_row_above_the_staging_chunk():
    """rows of 17.5 M f32 samples (70 MB) are staged one row at a time, so a clamp group of two rows is cut"""
    n, hop = 512, 512
    p = plan("f32", n)
    x = reals("f32", (2, 35 << 19), 58)
    x[1] *= 1e-3
    w = hann("f32", n)
    f = bank("f32", n, 80)
    d = dct_matrix("f32", 80, 13)
    dev, _ = dev_mfcc(p, x, w, hop, f, d, top_db_rows=2)
    host = np.full(dev.shape, np.nan, np.float32)
    p.mfcc(x, w, hop, f, d, host, top_db_rows=2)
    assert np.array_equal(host, dev)


def test_async_on_a_side_stream():
    torch = torch_mod()
    p = plan("f32", 512)
    x = reals("f32", (4, 9000), 59)
    w = hann("f32", 512)
    f = bank("f32", 512, 80)
    d = dct_matrix("f32", 80, 40)
    ref, frames = dev_mfcc(p, x, w, 128, f, d, top_db_rows=4)
    s = torch.cuda.Stream()
    xd, wd, fd, dd = (torch.from_numpy(a).cuda() for a in (x, w, f, d))
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        out = torch.full((4, frames, 40), float("nan"), dtype=torch.float32, device="cuda")
        p.mfcc(xd, wd, 128, fd, dd, out, top_db_rows=4)
    s.synchronize()
    assert np.array_equal(out.cpu().numpy(), ref)


def test_leading_shapes_and_batch_zero():
    torch = torch_mod()
    p = plan("f32", 256)
    x = reals("f32", (2, 3, 1000), 60)
    w = hann("f32", 256)
    f = bank("f32", 256, 32)
    d = dct_matrix("f32", 32, 12)
    got, frames = check(p, x, w, 300, f, d, TOL["f32"], top_db_rows=3)
    assert got.shape == (2, 3, frames, 12)
    wd, fd, dd = torch.from_numpy(w).cuda(), torch.from_numpy(f).cuda(), torch.from_numpy(d).cuda()
    p.mfcc(torch.zeros(0, 1000, device="cuda"), wd, 300, fd, dd, torch.empty(0, frames, 12, device="cuda"))
    # the C entry point at batch 0: succeeds and launches nothing
    xd, out = torch.zeros(1, 1000, device="cuda"), torch.full((1, frames, 12), float("nan"), device="cuda")
    rc = _lib.load().fourier_b200_mfcc_float(p._plan, xd.data_ptr(), 1000, wd.data_ptr(), 300, 2, 2, fd.data_ptr(), 32,
                                             0.0, 1e-10, TEN_LN10, 80.0, 1, dd.data_ptr(), 12, 0.0, out.data_ptr(), 0)
    assert rc == 0 and launches(p) == 0
    assert torch.isnan(out).all()


def test_refusals():
    torch = torch_mod()
    p = plan("f32", 512)
    x = torch.zeros(2, 1000, device="cuda")
    w = torch.ones(512, device="cuda")
    f = torch.ones(80, 257, device="cuda")
    d = torch.ones(80, 13, device="cuda")
    frames = p.stft_frames(1000, 128)
    out = torch.empty(2, frames, 13, device="cuda")
    with pytest.raises(ValueError, match="dct must have shape"):
        p.mfcc(x, w, 128, f, torch.ones(79, 13, device="cuda"), out)
    with pytest.raises(ValueError, match="last dimension must be 80"):
        p.mfcc(x, w, 128, f, None, out)
    with pytest.raises(ValueError, match="top_db_rows"):
        p.mfcc(x, w, 128, f, d, out, top_db_rows=3)
    p.mfcc(x, w, 128, f, d, out, top_db=None, top_db_rows=3)   # no clamp: any batch
    for kw, word in ((dict(top_db=-1.0), "top_db"), (dict(log_floor=0.0), "log_floor"),
                     (dict(log_scale=-1.0), "log_scale"), (dict(bias=math.nan), "bias"),
                     (dict(log_offset=math.inf), "log_offset"), (dict(power=3), "power")):
        with pytest.raises(ValueError, match=word):
            p.mfcc(x, w, 128, f, d, out, **kw)
    with pytest.raises(ValueError, match="host or all be device"):
        p.mfcc(x, w, 128, f, d.cpu().numpy(), out)
    # the C entry points check in_len against N, the overlaps and mixed memory themselves
    L = _lib.load()

    def call(xp=x.data_ptr(), in_len=1000, boundary=2, fp=f.data_ptr(), dp=d.data_ptr(), op=out.data_ptr(), batch=2):
        return L.fourier_b200_mfcc_float(p._plan, xp, in_len, w.data_ptr(), 128, boundary, 2, fp, 80, 0.0, 1e-10,
                                         TEN_LN10, 80.0, 1, dp, 13, 0.0, op, batch)

    assert call(in_len=500, boundary=0) == 1 and "in_len >= N" in _lib.last_error()
    assert call(in_len=256, boundary=2) == 1 and "in_len > N/2" in _lib.last_error()
    for kw in (dict(op=x.data_ptr()), dict(op=f.data_ptr()), dict(op=d.data_ptr()), dict(op=w.data_ptr())):
        assert call(**kw) == 1 and "overlap" in _lib.last_error(), kw
    host_d = np.ones((80, 13), np.float32)
    assert call(dp=host_d.ctypes.data) == 1 and "host or all be device" in _lib.last_error()

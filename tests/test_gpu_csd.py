"""Cross-spectral density and coherence of real rows (RealFft.csd / coherence, fourier_b200_csd_* / _coherence_*) on the
GPU: every fused size class, the half-length and full-length paths, against scipy.signal.csd and coherence in float64
on the same (rounded) inputs; csd(x, x) against the plan's welch; the coherence of x with 3x and of a zero row; a DC
offset of 1e4; rows of a periodic batch and a broadcast y bit for bit against the rows run alone; host against device
memory bit for bit, a row above the staging chunk, a side stream, two scratch chunks, leading shapes, batch 0 and
refusals.  Every output is NaN-filled before the call, and a guard region behind it must stay untouched."""

import numpy as np
import pytest

import fourier_b200 as fb
from fourier_b200 import _lib

pytestmark = pytest.mark.gpu

TOL = {"f32": 2e-5, "f64": 1e-12}
REAL = {"f32": np.float32, "f64": np.float64}
# (N, FFTs per CTA of its fused class; a round runs half as many frame pairs)
FUSED = [("f32", 128, 32), ("f32", 256, 32), ("f32", 512, 16), ("f32", 1024, 16), ("f32", 2048, 8), ("f64", 128, 32),
         ("f64", 256, 32), ("f64", 512, 16)]
GUARD = 64


def torch_mod():
    import torch
    return torch


def tdt(prec, cplx=False):
    torch = torch_mod()
    if cplx:
        return torch.complex64 if prec == "f32" else torch.complex128
    return torch.float32 if prec == "f32" else torch.float64


def plan(prec, n):
    return fb.create_rfft_f32(n) if prec == "f32" else fb.create_rfft_f64(n)


def reals(prec, shape, seed, dc=0.0):
    return (dc + np.random.default_rng(seed).standard_normal(shape)).astype(REAL[prec])


def partner(prec, x, seed):
    """broadband y for x: a first-order filter of x plus independent noise, so no bin's coherence is near 0/0"""
    from scipy.signal import lfilter
    x64 = np.asarray(x, np.float64)
    noise = np.random.default_rng(seed).standard_normal(x.shape)
    return (lfilter([1.0, 0.5], [1.0, -0.3], x64, axis=-1) + 0.7 * noise).astype(REAL[prec])


def hann(prec, n):
    return torch_mod().hann_window(n, dtype=torch_mod().float64).numpy().astype(REAL[prec])


def frames_of(x, n, hop, detrend):
    f = np.lib.stride_tricks.sliding_window_view(np.asarray(x, np.float64), n, axis=-1)[..., ::hop, :]
    return f - f.mean(axis=-1, keepdims=True) if detrend == "constant" else f


def ref_csd(x, y, w, hop, fs=1.0, scaling="density", detrend="constant"):
    """scipy.signal.csd in float64 where it takes the hop (hop <= N); the same definition in numpy beyond"""
    w = np.asarray(w, np.float64)
    n = len(w)
    if hop <= n:
        from scipy.signal import csd
        return csd(np.asarray(x, np.float64), np.asarray(y, np.float64), fs, window=w, nperseg=n, noverlap=n - hop,
                   detrend=detrend, scaling=scaling, axis=-1)[1]
    X = np.fft.rfft(frames_of(x, n, hop, detrend) * w, axis=-1)
    Y = np.fft.rfft(frames_of(y, n, hop, detrend) * w, axis=-1)
    p = (np.conj(X) * Y).mean(axis=-2)
    p *= 1.0 / (fs * (w * w).sum()) if scaling == "density" else 1.0 / w.sum() ** 2
    p[..., 1:(n + 1) // 2] *= 2
    return p


def ref_coherence(x, y, w, hop, detrend="constant"):
    w = np.asarray(w, np.float64)
    n = len(w)
    if hop <= n:
        from scipy.signal import coherence
        return coherence(np.asarray(x, np.float64), np.asarray(y, np.float64), 1.0, window=w, nperseg=n,
                         noverlap=n - hop, detrend=detrend, axis=-1)[1]
    X = np.fft.rfft(frames_of(x, n, hop, detrend) * w, axis=-1)
    Y = np.fft.rfft(frames_of(y, n, hop, detrend) * w, axis=-1)
    return np.abs((np.conj(X) * Y).sum(-2)) ** 2 / ((np.abs(X) ** 2).sum(-2) * (np.abs(Y) ** 2).sum(-2))


def dev_call(p, kind, x, y, w, hop, **kw):
    """device csd or coherence of numpy x, y into a NaN-filled output followed by a guard region -> numpy output"""
    torch = torch_mod()
    shape = x.shape[:-1] + (p.size() // 2 + 1,)
    count = int(np.prod(shape, dtype=np.int64))
    buf = torch.full((count + GUARD,), float("nan"), dtype=tdt(p.real, kind == "csd"), device="cuda")
    buf[count:] = 12345.0
    out = buf[:count].view(shape)
    getattr(p, kind)(torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda(), torch.from_numpy(w).cuda(), hop, out, **kw)
    torch.cuda.synchronize()
    assert torch.all(buf[count:] == 12345.0), "a write past the output"
    return out.cpu().numpy()


def row_err(got, ref):
    """per row max |got - ref| / max |ref|; NaN counts as infinite"""
    g = np.asarray(got).reshape(-1, np.shape(ref)[-1])
    r = np.asarray(ref).reshape(g.shape)
    e = np.abs(g - r).max(axis=1) / np.maximum(np.abs(r).max(axis=1), 1e-300)
    return float(np.where(np.isnan(e), np.inf, e).max())


def abs_err(got, ref):
    e = np.abs(np.asarray(got, np.float64) - np.asarray(ref, np.float64))
    return float(np.where(np.isnan(e), np.inf, e).max())


def launches(p):
    return p.info()["last_launches"]


def rfft_launches(p, rows):
    torch = torch_mod()
    p.rfft(torch.zeros(rows, p.size(), dtype=tdt(p.real), device="cuda"),
           torch.empty(rows, p.size() // 2 + 1, dtype=tdt(p.real, True), device="cuda"))
    return launches(p)


def row_len(n, hop, frames):
    return n + (frames - 1) * hop + hop // 2


@pytest.mark.parametrize("prec,n,c", FUSED)
def test_fused_size_classes(prec, n, c):
    """F = 1, F < C/2, B-1, B, B+1 and 2B+3 (B = 4 C/2) at hop N/4, F < C/2 and B+1 at hops 1, N and N+3; y_rows 1
    and one y per row; both outputs, both detrends, both scalings; the launch count of one or several items per row"""
    p = plan(prec, n)
    assert p.info()["path_name"] == "real_fused"
    w = hann(prec, n) + REAL[prec](0.25)
    pairs = c // 2
    b = 4 * pairs
    seed = 0
    for hop in (1, n // 4, n, n + 3):
        for frames in ((1, pairs // 2 + 1, b - 1, b, b + 1, 2 * b + 3) if hop == n // 4 else (pairs // 2 + 1, b + 1)):
            seed += 1
            rows = pairs + 1 if frames == 1 else 3
            x = reals(prec, (rows, row_len(n, hop, frames)), seed, dc=0.5)
            for y in (partner(prec, x[0], seed + 100), partner(prec, x, seed + 200)):
                detrend, scaling, fs = (("constant", "density", 2.5) if y.ndim == 1 else (False, "spectrum", 1.0))
                got = dev_call(p, "csd", x, y, w, hop, fs=fs, scaling=scaling, detrend=detrend)
                assert launches(p) == (3 if frames > b else 2), (hop, frames)
                err = row_err(got, ref_csd(x, y, w, hop, fs, scaling, detrend))
                assert err < TOL[prec], ("csd", hop, frames, y.ndim, err)
                got = dev_call(p, "coherence", x, y, w, hop, detrend=detrend)
                assert launches(p) == (2 if frames > b else 1), (hop, frames)
                err = abs_err(got, ref_coherence(x, y, w, hop, detrend))
                assert err < TOL[prec], ("coherence", hop, frames, y.ndim, err)


@pytest.mark.parametrize("prec,n,path", (("f32", 400, "real_half"), ("f64", 400, "real_half"), ("f32", 4096, "real_half"),
                                         ("f32", 97, "real_full"), ("f64", 97, "real_full")))
def test_other_paths(prec, n, path):
    p = plan(prec, n)
    assert p.info()["path_name"] == path
    w = hann(prec, n)
    for hop, frames in ((n // 4, 1), (n // 4, 50), (n // 2, 7), (n + 3, 3)):
        x = reals(prec, (3, row_len(n, hop, frames)), n + hop + frames, dc=0.5)
        for y, detrend in ((partner(prec, x[0], 5), "constant"), (partner(prec, x, 6), False)):
            got = dev_call(p, "csd", x, y, w, hop, fs=3.0, detrend=detrend)
            assert row_err(got, ref_csd(x, y, w, hop, 3.0, "density", detrend)) < TOL[prec], (hop, frames)
            got = dev_call(p, "coherence", x, y, w, hop, detrend=detrend)
            assert abs_err(got, ref_coherence(x, y, w, hop, detrend)) < TOL[prec], (hop, frames)


@pytest.mark.parametrize("prec,n", (("f32", 512), ("f64", 256), ("f32", 400), ("f32", 97)))
def test_csd_of_x_with_itself_is_welch(prec, n):
    """Re csd(x, x) matches welch(x), Im is within the bound of 0, and exactly +0 at bins 0 and N/2"""
    torch = torch_mod()
    p = plan(prec, n)
    hop = n // 2
    x = reals(prec, (3, 30 * n + 7), 71, dc=0.3)
    w = hann(prec, n)
    got = dev_call(p, "csd", x, x, w, hop, fs=2.0)
    P = torch.empty((3, n // 2 + 1), dtype=tdt(prec), device="cuda")
    p.welch(torch.from_numpy(x).cuda(), torch.from_numpy(w).cuda(), hop, P, fs=2.0)
    P = P.cpu().numpy().astype(np.float64)
    assert row_err(got.real, P) < TOL[prec]
    assert (np.abs(got.imag).max(axis=1) / P.max(axis=1)).max() < TOL[prec]
    edges = [0] + ([n // 2] if n % 2 == 0 else [])
    for k in edges:
        assert np.all(got.imag[:, k] == 0) and not np.any(np.signbit(got.imag[:, k])), k


@pytest.mark.parametrize("prec,n", (("f32", 512), ("f64", 512), ("f32", 400)))
def test_coherence_special_cases(prec, n):
    """coherence(x, 3x) is 1; a zero row gives NaN at every bin, as scipy does"""
    p = plan(prec, n)
    w = hann(prec, n)
    x = reals(prec, (2, 20 * n), 72)
    got = dev_call(p, "coherence", x, (3 * x).astype(REAL[prec]), w, n // 4)
    assert abs_err(got, np.ones_like(got)) < TOL[prec] * 5
    x[1] = 0
    got = dev_call(p, "coherence", x, partner(prec, x, 3), w, n // 4)
    assert np.all(np.isnan(got[1])) and not np.any(np.isnan(got[0]))


def test_dc_offset_needs_the_detrend_in_the_time_domain():
    """f32 N = 512, Hann, unit noise on a DC offset of 1e4 in x and y, detrend constant: every bin k >= 4 of the csd
    within 1e-5 of scipy in float64 on the same f32 inputs, relative to that bin's |Pxy|"""
    n, hop = 512, 256
    p = plan("f32", n)
    w = hann("f32", n)
    x = reals("f32", (4, n + 39 * hop), 77, dc=1e4)
    y = (partner("f32", x - np.float32(1e4), 78) + np.float32(1e4)).astype(np.float32)
    got = dev_call(p, "csd", x, y, w, hop)
    ref = ref_csd(x, y, w, hop)
    rel = np.abs(got[:, 4:] - ref[:, 4:]) / np.abs(ref[:, 4:])
    assert rel.max() <= 1e-5, rel.max()


@pytest.mark.parametrize("prec,n,hop,frames", (("f32", 512, 128, 5), ("f32", 512, 128, 131), ("f32", 128, 7, 1),
                                               ("f64", 256, 64, 300), ("f32", 400, 160, 40)))
@pytest.mark.parametrize("kind", ("csd", "coherence"))
def test_rows_of_a_periodic_batch_equal_the_row_alone(prec, n, hop, frames, kind):
    """97 rows repeating 5 base pairs, and y_rows = 1 against the same y repeated per row: bit for bit"""
    p = plan(prec, n)
    w = hann(prec, n)
    base = reals(prec, (5, row_len(n, hop, frames)), frames + n)
    ybase = partner(prec, base, frames)
    x, y = base[np.arange(97) % 5], ybase[np.arange(97) % 5]
    got = dev_call(p, kind, x, y, w, hop)
    alone = np.concatenate([dev_call(p, kind, base[i:i + 1], ybase[i:i + 1], w, hop) for i in range(5)])
    assert np.array_equal(got, alone[np.arange(97) % 5], equal_nan=True)
    one = dev_call(p, kind, x, ybase[0], w, hop)
    rep = dev_call(p, kind, x, np.ascontiguousarray(np.broadcast_to(ybase[0], x.shape)), w, hop)
    assert np.array_equal(one, rep, equal_nan=True)


@pytest.mark.parametrize("prec,n", (("f32", 512), ("f64", 512), ("f32", 400), ("f32", 97)))
@pytest.mark.parametrize("kind", ("csd", "coherence"))
def test_host_memory_gives_the_same_bits(prec, n, kind):
    """numpy and pinned torch buffers against device buffers, with a y of 2 rows broadcast over 3 x 2 rows"""
    torch = torch_mod()
    p = plan(prec, n)
    hop = n // 4
    x = reals(prec, (3, 2, 20 * n + 3), 39, dc=1.0)
    y = partner(prec, x[0], 40)
    w = hann(prec, n)
    kw = dict(fs=2.0, scaling="spectrum") if kind == "csd" else {}
    dev = dev_call(p, kind, x, y, w, hop, **kw)
    host = np.full(dev.shape, np.nan, dev.dtype)
    getattr(p, kind)(x, y, w, hop, host, **kw)
    assert np.array_equal(host, dev)
    pinned = torch.full(dev.shape, float("nan"), dtype=tdt(prec, kind == "csd")).pin_memory()
    getattr(p, kind)(torch.from_numpy(x).pin_memory(), torch.from_numpy(y).pin_memory(),
                     torch.from_numpy(w).pin_memory(), hop, pinned, **kw)
    assert np.array_equal(pinned.numpy(), dev)


def test_host_row_above_the_staging_chunk():
    """rows of 17.5 M f32 samples (70 MB) are staged one row at a time, with their y row beside them"""
    n, hop = 512, 512
    p = plan("f32", n)
    x = reals("f32", (2, 35 << 19), 40)
    y = partner("f32", x, 41)
    w = hann("f32", n)
    dev = dev_call(p, "csd", x, y, w, hop)
    host = np.full((2, n // 2 + 1), np.nan, np.complex64)
    p.csd(x, y, w, hop, host)
    assert launches(p) == 1 + 2 * 2   # the scale, then per staged row the fused kernel and the finish
    assert np.array_equal(host, dev)
    assert row_err(dev, ref_csd(x, y, w, hop)) < TOL["f32"]


def test_async_on_a_side_stream():
    torch = torch_mod()
    p = plan("f32", 512)
    x = reals("f32", (4, 9000), 41)
    y = partner("f32", x, 42)
    w = hann("f32", 512)
    ref = dev_call(p, "csd", x, y, w, 128)
    s = torch.cuda.Stream()
    xd, yd, wd = torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda(), torch.from_numpy(w).cuda()
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        out = torch.full((4, 257), float("nan"), dtype=torch.complex64, device="cuda")
        p.csd(xd, yd, wd, 128, out)
    s.synchronize()
    assert np.array_equal(out.cpu().numpy(), ref)


def test_real_half_two_scratch_chunks():
    """60 rows of 2998 frame pairs at N = 400: two frames and two spectra of 3208 bytes each per pair fill the 512 MB
    scratch after 83676 pairs, and the item of 12 frames that straddles the cut is continued in the second chunk"""
    p = plan("f32", 400)
    rows = 60
    x = reals("f32", (rows, 480000), 33, dc=0.5)
    y = partner("f32", x[0], 34)
    w = hann("f32", 400)
    got = dev_call(p, "csd", x, y, w, 160)
    frames = 1 + (480000 - 400) // 160
    chunk = (512 << 20) // (2 * (400 * 4 + 201 * 8))
    assert chunk < rows * frames and (chunk % frames) % 12 != 0
    n = launches(p)
    total = rows * frames
    # the scale; per scratch chunk the gather, the plan's rfft of its frames of x and y, and the accumulate; the finish
    nqs = [min(chunk, total - q0) for q0 in range(0, total, chunk)]
    assert n == 1 + sum(2 + rfft_launches(p, 2 * nq) for nq in nqs) + 1
    for r in (0, chunk // frames, chunk // frames + 1, rows - 1):
        assert row_err(got[r:r + 1], ref_csd(x[r:r + 1], y, w, 160)) < TOL["f32"], r


def test_leading_shapes_and_batch_zero():
    torch = torch_mod()
    p = plan("f32", 256)
    w = hann("f32", 256)
    x = reals("f32", (2, 3, 1500), 61)
    y = partner("f32", x[0], 62)
    got = dev_call(p, "csd", x, y, w, 100)
    assert got.shape == (2, 3, 129)
    assert np.array_equal(got.reshape(6, 129), dev_call(p, "csd", x.reshape(6, 1500), np.tile(y, (2, 1)), w, 100))
    out = torch.full((0, 129), float("nan"), dtype=torch.complex64, device="cuda")
    p.csd(torch.empty((0, 1500), device="cuda"), torch.empty((0, 1500), device="cuda"), torch.from_numpy(w).cuda(), 100,
          out)
    p.coherence(torch.empty((0, 1500), device="cuda"), torch.empty((1500,), device="cuda"), torch.from_numpy(w).cuda(),
                100, torch.empty((0, 129), device="cuda"))
    # the C entry points at batch 0 succeed and launch nothing
    L = _lib.load()
    wd = torch.from_numpy(w).cuda()
    xd = torch.zeros(1500, device="cuda")
    o = torch.empty(129, dtype=torch.complex64, device="cuda")
    assert L.fourier_b200_csd_float(p._plan, xd.data_ptr(), xd.data_ptr(), 1, 1500, wd.data_ptr(), 100, 1, 0, 1.0,
                                    o.data_ptr(), 0) == 0
    assert launches(p) == 0
    assert L.fourier_b200_coherence_float(p._plan, xd.data_ptr(), xd.data_ptr(), 1, 1500, wd.data_ptr(), 100, 1,
                                          o.data_ptr(), 0) == 0
    assert launches(p) == 0


def test_refusals():
    torch = torch_mod()
    p = plan("f32", 512)
    x = torch.zeros(2, 1000, device="cuda")
    y = torch.zeros(2, 1000, device="cuda")
    w = torch.ones(512, device="cuda")
    out = torch.empty(2, 257, dtype=torch.complex64, device="cuda")
    coh = torch.empty(2, 257, device="cuda")
    with pytest.raises(ValueError, match="last dimension"):
        p.csd(x, y, w, 128, torch.empty(2, 256, dtype=torch.complex64, device="cuda"))
    with pytest.raises(ValueError, match="leading"):
        p.csd(x, y, w, 128, torch.empty(3, 257, dtype=torch.complex64, device="cuda"))
    with pytest.raises(ValueError, match="trailing part"):
        p.csd(x, torch.zeros(3, 1000, device="cuda"), w, 128, out)
    with pytest.raises(ValueError, match="samples of the x rows"):
        p.coherence(x, torch.zeros(2, 999, device="cuda"), w, 128, coh)
    with pytest.raises(TypeError, match="expected"):
        p.csd(x, y, w, 128, coh)
    with pytest.raises(TypeError, match="expected"):
        p.coherence(x, y, w, 128, out)
    with pytest.raises(ValueError, match="at least N"):
        p.csd(torch.zeros(2, 500, device="cuda"), torch.zeros(2, 500, device="cuda"), w, 128, out)
    with pytest.raises(ValueError, match="hop"):
        p.coherence(x, y, w, 0, coh)
    with pytest.raises(ValueError, match="scaling"):
        p.csd(x, y, w, 128, out, scaling="power")
    with pytest.raises(ValueError, match="detrend"):
        p.coherence(x, y, w, 128, coh, detrend="linear")
    for fs in (0.0, -1.0, float("inf"), float("nan")):
        with pytest.raises(ValueError, match="fs"):
            p.csd(x, y, w, 128, out, fs=fs)
    with pytest.raises(ValueError, match="host or all be device"):
        p.csd(x, y.cpu().numpy(), w, 128, out)
    with pytest.raises(ValueError, match="conj"):
        p.coherence(x, y._neg_view(), w, 128, coh)
    # the C entry points check the overlaps and a mix of host and device memory themselves; y == x is allowed
    L = _lib.load()
    big = torch.zeros(4 * 1000, device="cuda")
    for o in (x, y, w):
        rc = L.fourier_b200_csd_float(p._plan, x.data_ptr(), y.data_ptr(), 2, 1000, w.data_ptr(), 128, 1, 0, 1.0,
                                      o.data_ptr(), 2)
        assert rc == 1 and "overlap" in _lib.last_error()
        rc = L.fourier_b200_coherence_float(p._plan, x.data_ptr(), y.data_ptr(), 2, 1000, w.data_ptr(), 128, 1,
                                            o.data_ptr(), 2)
        assert rc == 1 and "overlap" in _lib.last_error()
    assert L.fourier_b200_csd_float(p._plan, x.data_ptr(), x.data_ptr(), 2, 1000, w.data_ptr(), 128, 1, 0, 1.0,
                                    big.data_ptr(), 2) == 0
    host = np.zeros(2 * 257, np.complex64)
    rc = L.fourier_b200_csd_float(p._plan, x.data_ptr(), y.data_ptr(), 2, 1000, w.data_ptr(), 128, 1, 0, 1.0,
                                  host.ctypes.data, 1)
    assert rc == 1 and "host or all be device" in _lib.last_error()
    with pytest.raises(ValueError, match="in_len|at least N"):
        p.csd(torch.zeros(2, 100, device="cuda"), torch.zeros(2, 100, device="cuda"), w, 128, out)

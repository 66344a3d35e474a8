"""Type-IV DCT, MDCT and IMDCT of real rows (RealFft.dct4 / mdct / imdct, fourier_b200_dct4_* / mdct_* / imdct_*) on the
GPU: every fused size class (f32 N = 128 .. 2048, f64 N = 128 .. 512) and the half-length path (f32 N = 480, 960 and
4096, f64 N = 96 and 1024), with the plan's path asserted, against scipy.fft.dct(type=4) and the MDCT fold in float64
on the same (rounded) inputs; the round trip imdct(mdct(x)) = x with a sine window in all three norms; periodic batches
against their base rows bit for bit, past one sweep of the fused grid and over two scratch chunks of real_half; an
imdct row long enough for two scratch runs; host against device memory; a side stream, launch counts and refusals.
Every output is NaN-filled before the call, and a guard region behind it must stay untouched."""

import numpy as np
import pytest

import fourier_b200 as fb
from fourier_b200 import _lib

pytestmark = pytest.mark.gpu

TOL = {"f32": 2e-5, "f64": 1e-12}
REAL = {"f32": np.float32, "f64": np.float64}
NORMS = ("backward", "ortho", "forward")
SWAP = {"backward": "forward", "forward": "backward", "ortho": "ortho"}
# (N, FFTs per CTA of its fused class)
FUSED = [("f32", 128, 32), ("f32", 256, 32), ("f32", 512, 16), ("f32", 1024, 16), ("f32", 2048, 8), ("f64", 128, 32),
         ("f64", 256, 32), ("f64", 512, 16)]
HALF = [("f32", 480), ("f32", 960), ("f32", 4096), ("f64", 96), ("f64", 1024)]
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


def sine(prec, n):
    return np.sin(np.pi * (np.arange(2 * n) + 0.5) / (2 * n)).astype(REAL[prec])


def ref_dct4(x, norm):
    from scipy.fft import dct
    return dct(np.asarray(x, np.float64), type=4, norm=norm, axis=-1)


def frames_of(n, length, center):
    return -(-length // n) + 1 if center else 1 + (length - 2 * n) // n


def ref_mdct(x, w, n, center, norm):
    """the frames, the window and the fold u = (-c_rev - d, a - b_rev) in float64, then scipy's DCT-IV"""
    x = np.asarray(x, np.float64)
    length = x.shape[-1]
    pad, F = (n if center else 0), frames_of(n, length, center)
    xp = np.zeros(x.shape[:-1] + ((F + 1) * n,))
    xp[..., pad:pad + length] = x[..., :(F + 1) * n - pad]
    fr = np.stack([xp[..., f * n:f * n + 2 * n] for f in range(F)], axis=-2) * np.asarray(w, np.float64)
    a, b, c, d = np.split(fr, 4, axis=-1)
    return ref_dct4(np.concatenate([-c[..., ::-1] - d, a - b[..., ::-1]], axis=-1), norm)


def ref_imdct(X, w, n, center, norm, out_len):
    v = ref_dct4(X, SWAP[norm])
    h = n // 2
    fr = np.concatenate([v[..., h:], -v[..., ::-1], -v[..., :h]], axis=-1) * np.asarray(w, np.float64)
    F = X.shape[-2]
    y = np.zeros(X.shape[:-2] + ((F + 1) * n + out_len + n,))
    for f in range(F):
        y[..., f * n:f * n + 2 * n] += fr[..., f, :]
    pad = n if center else 0
    return y[..., pad:pad + out_len]


def nan_out(prec, shape):
    """a NaN-filled device output followed by a guard region -> (output view, whole buffer, count)"""
    torch = torch_mod()
    count = int(np.prod(shape, dtype=np.int64))
    buf = torch.full((count + GUARD,), float("nan"), dtype=tdt(prec), device="cuda")
    buf[count:] = 12345.0
    return buf[:count].view(shape), buf, count


def finish(buf, count, out):
    torch = torch_mod()
    torch.cuda.synchronize()
    assert torch.all(buf[count:] == 12345.0), "a write past the output"
    got = out.cpu().numpy()
    assert not np.isnan(got).any(), "an output was not written"
    return got


def dev_dct4(p, x, norm):
    torch = torch_mod()
    out, buf, count = nan_out(p.real, x.shape)
    p.dct4(torch.from_numpy(x).cuda(), out, norm=norm)
    return finish(buf, count, out)


def dev_mdct(p, x, w, center, norm):
    torch = torch_mod()
    n = p.size()
    out, buf, count = nan_out(p.real, x.shape[:-1] + (p.mdct_frames(x.shape[-1], center), n))
    p.mdct(torch.from_numpy(x).cuda(), torch.from_numpy(w).cuda(), out, center=center, norm=norm)
    return finish(buf, count, out)


def dev_imdct(p, X, w, center, norm, out_len):
    torch = torch_mod()
    out, buf, count = nan_out(p.real, X.shape[:-2] + (out_len,))
    p.imdct(torch.from_numpy(X).cuda(), torch.from_numpy(w).cuda(), out, center=center, norm=norm)
    return finish(buf, count, out)


def row_err(got, ref):
    """worst over rows of max |got - ref| / max |ref|; NaN counts as infinite"""
    g = np.asarray(got, np.float64).reshape(-1, np.shape(ref)[-1])
    r = np.asarray(ref, np.float64).reshape(g.shape)
    e = np.abs(g - r).max(axis=1) / np.maximum(np.abs(r).max(axis=1), 1e-300)
    return float(np.where(np.isnan(e), np.inf, e).max())


def launches(p):
    return p.info()["last_launches"]


def inner_launches(prec, m, rows):
    """launches of the complex plan of length m on `rows` rows in place, as the half-length path runs it"""
    torch = torch_mod()
    c = fb.create_fft_f32(m) if prec == "f32" else fb.create_fft_f64(m)
    ct = torch.complex64 if prec == "f32" else torch.complex128
    c.fft_in_place(torch.zeros(rows, m, dtype=ct, device="cuda"))
    torch.cuda.synchronize()
    return c.info()["last_launches"]


@pytest.mark.parametrize("prec,n,c", FUSED)
@pytest.mark.parametrize("norm", NORMS)
def test_fused_dct4(prec, n, c, norm):
    """3 C + 5 rows (a partial group) in one launch, against scipy"""
    p = plan(prec, n)
    assert p.info()["path_name"] == "real_fused"
    x = reals(prec, (3 * c + 5, n), n)
    got = dev_dct4(p, x, norm)
    assert launches(p) == 1
    assert row_err(got, ref_dct4(x, norm)) < TOL[prec]


@pytest.mark.parametrize("prec,n,c", FUSED)
@pytest.mark.parametrize("center", (True, False))
def test_fused_mdct_and_imdct(prec, n, c, center):
    """rows of 2N + 1, 4N and 5N + 17 samples (and 1 with center), one launch for the mdct and two for the imdct, in
    every norm"""
    p = plan(prec, n)
    assert p.info()["path_name"] == "real_fused"
    w = sine(prec, n)
    for length in ([1] if center else []) + [2 * n + 1, 4 * n, 5 * n + 17]:
        x = reals(prec, (3, length), length)
        F = frames_of(n, length, center)
        for norm in NORMS:
            X = dev_mdct(p, x, w, center, norm)
            assert X.shape == (3, F, n)
            assert launches(p) == 1
            assert row_err(X, ref_mdct(x, w, n, center, norm)) < TOL[prec], (length, norm)
            out_len = length if center else (F + 1) * n
            y = dev_imdct(p, X, w, center, norm, out_len)
            assert launches(p) == 2
            assert row_err(y, ref_imdct(X, w, n, center, norm, out_len)) < TOL[prec], (length, norm)


@pytest.mark.parametrize("prec,n", HALF)
def test_real_half(prec, n):
    p = plan(prec, n)
    assert p.info()["path_name"] == "real_half"
    w = sine(prec, n)
    x = reals(prec, (5, n), n)
    inner = inner_launches(prec, n // 2, 5)
    for norm in NORMS:
        assert row_err(dev_dct4(p, x, norm), ref_dct4(x, norm)) < TOL[prec], norm
        assert launches(p) == 2 + inner
    for center in (True, False):
        length = 3 * n + n // 2 + 1
        s = reals(prec, (2, length), n + center)
        F = frames_of(n, length, center)
        for norm in NORMS:
            X = dev_mdct(p, s, w, center, norm)
            assert launches(p) == 2 + inner_launches(prec, n // 2, 2 * F)
            assert row_err(X, ref_mdct(s, w, n, center, norm)) < TOL[prec], (center, norm)
            out_len = length if center else (F + 1) * n
            y = dev_imdct(p, X, w, center, norm, out_len)
            assert launches(p) == 3 + inner_launches(prec, n // 2, 2 * F)
            assert row_err(y, ref_imdct(X, w, n, center, norm, out_len)) < TOL[prec], (center, norm)


@pytest.mark.parametrize("prec,n", (("f32", 1024), ("f32", 256), ("f32", 960), ("f64", 512), ("f64", 96)))
@pytest.mark.parametrize("norm", NORMS)
def test_round_trip_with_a_sine_window(prec, n, norm):
    """with center, out_len = L and a Princen-Bradley window the imdct gives x back, L not a multiple of N"""
    p = plan(prec, n)
    w = sine(prec, n)
    x = reals(prec, (4, 7 * n + 13), 3 * n)
    y = dev_imdct(p, dev_mdct(p, x, w, True, norm), w, True, norm, x.shape[-1])
    assert row_err(y, x) < 4 * TOL[prec]


def test_dct4_inverse_is_the_swapped_norm():
    p = plan("f32", 512)
    x = reals("f32", (6, 512), 9)
    for norm in NORMS:
        back = dev_dct4(p, dev_dct4(p, x, norm), SWAP[norm])
        assert row_err(back, x) < 4 * TOL["f32"], norm


@pytest.mark.parametrize("prec,n,rows", (("f32", 1024, 7 * 2500 + 3), ("f64", 512, 7 * 1300 + 3),
                                         ("f32", 4096, 7 * 4830 + 3)))
def test_periodic_dct4_rows_match_their_base_row(prec, n, rows):
    """past one sweep of the fused grid (f32 N = 1024: 1056 groups of 16 rows; f64 N = 512: 528 groups of 16), and over
    two 512 MB scratch chunks of real_half (f32 N = 4096: 32768 rows per chunk); in place gives the same bits"""
    torch = torch_mod()
    p = plan(prec, n)
    base = reals(prec, (7, n), n + rows)
    x = np.concatenate([base] * (rows // 7) + [base[:rows % 7]])
    got = dev_dct4(p, x, "ortho")
    calls = launches(p)
    alone = dev_dct4(p, base, "ortho")
    for r in range(7):
        assert np.array_equal(got[r::7], np.broadcast_to(alone[r], got[r::7].shape)), r
    if p.info()["path_name"] == "real_half":
        chunk = (512 << 20) // (n * np.dtype(REAL[prec]).itemsize)
        assert rows > chunk
        assert calls == (2 + inner_launches(prec, n // 2, chunk)) + (2 + inner_launches(prec, n // 2, rows - chunk))
    xd = torch.from_numpy(x).cuda()
    p.dct4(xd, xd, norm="ortho")
    torch.cuda.synchronize()
    assert np.array_equal(xd.cpu().numpy(), got)


@pytest.mark.parametrize("prec,n,length,rows", (("f32", 1024, 6 * 1024 + 7, 2200), ("f32", 4096, 64 * 4096, 520)))
def test_periodic_mdct_rows_match_their_base_row(prec, n, length, rows):
    """f32 N = 1024: 17600 frames, past one sweep of the fused grid; f32 N = 4096 (real_half): 33800 frames, over two
    scratch chunks of 32768 frames"""
    p = plan(prec, n)
    w = sine(prec, n)
    base = reals(prec, (3, length), n)
    x = np.concatenate([base] * (rows // 3) + [base[:rows % 3]])
    got = dev_mdct(p, x, w, True, "backward")
    alone = dev_mdct(p, base, w, True, "backward")
    for r in range(3):
        assert np.array_equal(got[r::3], np.broadcast_to(alone[r], got[r::3].shape)), r


def test_imdct_row_over_two_scratch_runs():
    """one f32 N = 1024 row of 140001 frames: a scratch of 131072 frames cuts it into two runs; the round trip gives x
    back, and the outputs on both sides of the cut equal those of shorter calls bit for bit"""
    n = 1024
    p = plan("f32", n)
    w = sine("f32", n)
    x = reals("f32", (1, 140000 * n + 5), 12)
    X = dev_mdct(p, x, w, True, "ortho")
    F = X.shape[1]
    y = dev_imdct(p, X, w, True, "ortho", x.shape[-1])
    runs = 2
    assert launches(p) == 2 * runs
    assert row_err(y, x) < 4 * TOL["f32"]
    # outputs of the first run, and around the cut, from calls on fewer frames that cover them the same way
    head = dev_imdct(p, np.ascontiguousarray(X[:, :1000]), w, True, "ortho", 998 * n)
    assert np.array_equal(head, y[:, :998 * n])
    f0 = 131000
    part = dev_imdct(p, np.ascontiguousarray(X[:, f0:f0 + 2000]), w, False, "ortho", 2000 * n)
    t0 = f0 * n - n   # output i of the part is padded position i + f0 N of the row, output i + f0 N - N
    assert np.array_equal(part[:, n:1999 * n], y[:, t0 + n:t0 + 1999 * n])
    assert F == 140002


@pytest.mark.parametrize("prec,n", (("f32", 1024), ("f64", 96)))
def test_host_memory_gives_the_same_bits(prec, n):
    p = plan(prec, n)
    w = sine(prec, n)
    x = reals(prec, (5, 5 * n + 3), 17)
    X = dev_mdct(p, x, w, True, "ortho")
    Xh = np.full_like(X, np.nan)
    p.mdct(x, w, Xh, center=True, norm="ortho")
    assert np.array_equal(Xh, X)
    y = dev_imdct(p, X, w, True, "ortho", x.shape[-1])
    yh = np.full((5, x.shape[-1]), np.nan, REAL[prec])
    p.imdct(Xh, w, yh, center=True, norm="ortho")
    assert np.array_equal(yh, y)
    r = reals(prec, (9, n), 18)
    d = dev_dct4(p, r, "forward")
    dh = np.full_like(r, np.nan)
    p.dct4(r, dh, norm="forward")
    assert np.array_equal(dh, d)
    p.dct4(r, r, norm="forward")
    assert np.array_equal(r, d)


def test_async_on_a_side_stream():
    torch = torch_mod()
    n = 1024
    p = plan("f32", n)
    w = sine("f32", n)
    x = reals("f32", (20, 9 * n), 41)
    ref = dev_mdct(p, x, w, True, "backward")
    s = torch.cuda.Stream()
    xd, wd = torch.from_numpy(x).cuda(), torch.from_numpy(w).cuda()
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        out = torch.full(ref.shape, float("nan"), dtype=torch.float32, device="cuda")
        p.mdct(xd, wd, out)
        y = torch.full((20, 9 * n), float("nan"), dtype=torch.float32, device="cuda")
        p.imdct(out, wd, y)
    s.synchronize()
    assert np.array_equal(out.cpu().numpy(), ref)
    assert np.array_equal(y.cpu().numpy(), dev_imdct(p, ref, w, True, "backward", 9 * n))


def test_leading_shapes_and_batch_zero():
    torch = torch_mod()
    n = 256
    p = plan("f32", n)
    w = sine("f32", n)
    x = reals("f32", (2, 3, 4 * n), 61)
    X = dev_mdct(p, x, w, True, "ortho")
    assert X.shape == (2, 3, 5, n)
    assert np.array_equal(X.reshape(6, 5, n), dev_mdct(p, x.reshape(6, 4 * n), w, True, "ortho"))
    p.mdct(torch.empty((0, 4 * n), device="cuda"), torch.from_numpy(w).cuda(), torch.empty((0, 5, n), device="cuda"))
    L = _lib.load()
    xd = torch.zeros(4 * n, device="cuda")
    wd = torch.from_numpy(w).cuda()
    out = torch.zeros(5 * n, device="cuda")
    assert L.fourier_b200_mdct_float(p._plan, xd.data_ptr(), 4 * n, wd.data_ptr(), 1, 0, out.data_ptr(), 0) == 0
    assert launches(p) == 0
    assert L.fourier_b200_imdct_float(p._plan, xd.data_ptr(), 2, wd.data_ptr(), 1, 0, out.data_ptr(), 7, 0) == 0
    assert L.fourier_b200_dct4_float(p._plan, xd.data_ptr(), xd.data_ptr(), 0, 0) == 0
    assert launches(p) == 0


def test_refusals():
    torch = torch_mod()
    n = 512
    p = plan("f32", n)
    x = torch.zeros(4, 3 * n, device="cuda")
    w = torch.zeros(2 * n, device="cuda")
    out = torch.empty(4, 4, n, device="cuda")
    with pytest.raises(ValueError, match="shape"):
        p.mdct(x, w, torch.empty(4, 5, n, device="cuda"))
    with pytest.raises(ValueError, match="last dimension"):
        p.mdct(x, w, torch.empty(4, 4, n + 1, device="cuda"))
    with pytest.raises(ValueError, match="last dimension must be 1024"):
        p.mdct(x, torch.zeros(n, device="cuda"), out)
    with pytest.raises(ValueError, match="at least 2N"):
        p.mdct(torch.zeros(4, n, device="cuda"), w, out, center=False)
    with pytest.raises(ValueError, match="leading shapes"):
        p.imdct(out, w, torch.empty(3, 3 * n, device="cuda"))
    with pytest.raises(ValueError, match="F >= 1"):
        p.imdct(torch.empty(4, 0, n, device="cuda"), w, torch.empty(4, 3 * n, device="cuda"))
    with pytest.raises(ValueError, match="norm"):
        p.dct4(x[:, :n].contiguous(), torch.empty(4, n, device="cuda"), norm="none")
    with pytest.raises(ValueError, match="host or all be device"):
        p.mdct(x, w.cpu().numpy(), out)
    with pytest.raises(ValueError, match="shapes differ"):
        p.dct4(torch.zeros(4, n, device="cuda"), torch.empty(3, n, device="cuda"))
    # odd N: refused by Python and by the C entry points
    odd = plan("f32", 97)
    assert odd.info()["path_name"] == "real_full"
    with pytest.raises(ValueError, match="even plan length"):
        odd.dct4(torch.zeros(2, 97, device="cuda"), torch.empty(2, 97, device="cuda"))
    L = _lib.load()
    buf = torch.zeros(8 * 97, device="cuda")
    rc = L.fourier_b200_dct4_float(odd._plan, buf.data_ptr(), buf.data_ptr(), 2, 0)
    assert rc == 1 and "even plan length" in _lib.last_error()
    rc = L.fourier_b200_mdct_float(odd._plan, buf.data_ptr(), 97, buf.data_ptr(), 1, 0, buf.data_ptr(), 1)
    assert rc == 1 and "even plan length" in _lib.last_error()
    rc = L.fourier_b200_imdct_float(odd._plan, buf.data_ptr(), 1, buf.data_ptr(), 1, 0, buf.data_ptr(), 5, 1)
    assert rc == 1 and "even plan length" in _lib.last_error()
    # the C entry points check overlaps, a mix of host and device memory and the alignment themselves
    flat = torch.zeros(5 * n, device="cuda")
    rc = L.fourier_b200_dct4_float(p._plan, flat.data_ptr(), flat.data_ptr() + n * 4, 4, 0)
    assert rc == 1 and "overlap" in _lib.last_error()
    big = torch.zeros(40 * n, device="cuda")
    rc = L.fourier_b200_mdct_float(p._plan, big.data_ptr(), 4 * n, w.data_ptr(), 1, 0, big.data_ptr() + 8 * n, 1)
    assert rc == 1 and "overlap" in _lib.last_error()
    rc = L.fourier_b200_mdct_float(p._plan, x.data_ptr(), 3 * n, big.data_ptr(), 1, 0, big.data_ptr() + 4 * n, 1)
    assert rc == 1 and "overlap" in _lib.last_error()
    rc = L.fourier_b200_imdct_float(p._plan, big.data_ptr(), 4, w.data_ptr(), 1, 0, big.data_ptr() + 2 * n * 4, 100, 1)
    assert rc == 1 and "overlap" in _lib.last_error()
    rc = L.fourier_b200_mdct_float(p._plan, x.data_ptr(), n, w.data_ptr(), 0, 0, out.data_ptr(), 1)
    assert rc == 1 and "2N" in _lib.last_error()
    host = np.zeros((4, n), np.float32)
    rc = L.fourier_b200_dct4_float(p._plan, flat.data_ptr(), host.ctypes.data, 4, 0)
    assert rc == 1 and "host or both be device" in _lib.last_error()
    rc = L.fourier_b200_dct4_async_float(p._plan, flat.data_ptr() + 4, flat.data_ptr() + 4, 4, 0, None)
    assert rc == 716, rc
    assert "16-byte aligned" in _lib.last_error()

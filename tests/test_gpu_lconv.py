"""Linear convolution of real rows by overlap-save (RealFft.convolve_linear, fourier_b200_linear_convolve_real_*) on the
GPU: every path against a direct linear convolution (np.convolve in long double, or scipy's fftconvolve in float64 for
long rows), every mode, short and multi-segment rows, several spectra, exact properties (host memory, rows alone,
streams, complete and contained stores), agreement with zero padding + convolve, 64-bit offsets, launch counts and
refusals.  Taps have magnitudes in [0.5, 1): a row of one output (L = 1, mode same) is a single tap times x[0], and the
per-row error is measured against the row's largest output."""

import numpy as np
import pytest

import fourier_b200 as fb
from fourier_b200 import _lib
from helpers import per_transform_err

pytestmark = pytest.mark.gpu

TOL = {"f32": 1e-5, "f64": 1e-12}
REAL = {"f32": np.float32, "f64": np.float64}
SPEC = {"f32": np.complex64, "f64": np.complex128}
MODES = ("full", "same", "valid")


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


def taps(shape, k, seed):
    rng = np.random.default_rng(seed)
    return rng.choice([-1.0, 1.0], tuple(shape) + (k,)) * rng.uniform(0.5, 1.0, tuple(shape) + (k,))


def spectra(prec, h, n):
    """rfft of the taps zero-padded to n, in the plan's precision"""
    return np.fft.rfft(h, n=n, axis=-1).astype(SPEC[prec])


def out_len(mode, l, k):
    return {"full": l + k - 1, "same": l, "valid": l - k + 1}[mode]


def offset(mode, k):
    return {"full": 0, "same": (k - 1) // 2, "valid": k - 1}[mode]


def truth(x, h, mode):
    """the outputs [o, o + out_len) of the full linear convolution of every row of x (..., L) with h (..., K), h
    broadcast as convolve_linear broadcasts the spectra: np.convolve in long double, or scipy's fftconvolve in float64
    when L * K is large"""
    lead, l, k = x.shape[:-1], x.shape[-1], h.shape[-1]
    xs = x.reshape(-1, l)
    hs = np.broadcast_to(h, lead + (k,)).reshape(-1, k)
    if l * k <= 200_000:
        full = np.stack([np.convolve(xs[b].astype(np.longdouble), hs[b].astype(np.longdouble))
                         for b in range(xs.shape[0])])
    else:
        from scipy.signal import fftconvolve
        full = fftconvolve(xs.astype(np.float64), hs.astype(np.float64), axes=-1)
    o = offset(mode, k)
    return full[:, o:o + out_len(mode, l, k)].reshape(lead + (-1,))


def run(p, x, H, k, mode, host=False):
    """convolve_linear on device buffers (or host arrays) -> numpy result"""
    torch = torch_mod()
    shape = x.shape[:-1] + (out_len(mode, x.shape[-1], k),)
    if host:
        y = np.full(shape, np.nan, x.dtype)
        p.convolve_linear(np.ascontiguousarray(x), np.ascontiguousarray(H), k, y, mode)
        return y
    xd = torch.from_numpy(np.ascontiguousarray(x)).cuda()
    Hd = torch.from_numpy(np.ascontiguousarray(H)).cuda()
    y = torch.full(shape, float("nan"), dtype=xd.dtype, device="cuda")
    p.convolve_linear(xd, Hd, k, y, mode)
    torch.cuda.synchronize()
    return y.cpu().numpy()


def check(prec, p, n, l, k, mode, batch, rows, seed):
    """batch rows of l samples, rows spectra (0: one for all rows) -> worst per-row error"""
    x = reals(prec, (batch, l), seed)
    hshape = () if rows == 0 else (rows,)
    h = taps(hshape, k, seed + 1)
    xs = x if rows in (0, batch) else x.reshape(batch // rows, rows, l)
    y = run(p, xs, spectra(prec, h, n), k, mode)
    err = per_transform_err(y, truth(xs, h, mode))
    assert err.max() < TOL[prec], (prec, n, l, k, mode, batch, rows, err.max())
    return float(err.max())


@pytest.mark.parametrize("prec", ["f32", "f64"])
def test_every_size_up_to_256(prec):
    worst = {}
    for n in range(1, 257):
        p = plan(prec, n)
        for i, (k, l) in enumerate([(1, 1), (max(1, n // 3), 3 * (n - max(1, n // 3) + 1) + 7), (n, n + 2),
                                    ((n + 1) // 2, 1)]):
            mode = MODES[(n + i) % 3]
            if mode == "valid" and l < k:
                mode = "full"
            err = check(prec, p, n, l, k, mode, 3, 3 if i % 2 else 0, seed=n + i)
            name = p.info()["path_name"]
            worst[name] = max(worst.get(name, 0.0), err)
        p.close()
    print(f"{prec} N=1..256 worst per path: {worst}")
    assert set(worst) == {"real_fused", "real_half", "real_full"}


FUSED = [("f32", n) for n in (128, 256, 512, 1024, 2048)] + [("f64", n) for n in (128, 256, 512)]


@pytest.mark.parametrize("prec,n", FUSED)
def test_fused_sizes(prec, n):
    p = plan(prec, n)
    assert p.info()["path_name"] == "real_fused"
    worst = 0.0
    for k in (1, 17, n // 2 + 1, n):
        s = n - k + 1
        for mode in MODES:
            l = (k if mode == "valid" else 0) + 2 * s + 5
            for batch in (1, 3, 17, 1026):
                worst = max(worst, check(prec, p, n, l, k, mode, batch, 3 if batch % 3 == 0 else 0, seed=k + batch))
    p.close()
    print(f"fused {prec} N={n}: worst per-row error {worst:.3e}")


def test_half_and_full_paths():
    """real_half on persistent inner plans and real_full on fused Bluestein, multi-segment rows"""
    cases = [("f32", 1 << 21, 3000, "full", 3 * ((1 << 21) - 2999) + 7, 2, "real_half"),
             ("f64", 1 << 17, 1000, "same", 5 * ((1 << 17) - 999) + 3, 3, "real_half"),
             ("f32", 1009, 100, "valid", 5000, 4, "real_full"), ("f64", 1009, 333, "full", 2000, 3, "real_full")]
    for prec, n, k, mode, l, batch, path in cases:
        p = plan(prec, n)
        assert p.info()["path_name"] == path, (prec, n, p.info())
        err = check(prec, p, n, l, k, mode, batch, batch, seed=n)
        print(f"{path} {prec} N={n} K={k} {mode} L={l}: worst {err:.3e}, inner {p.info()['inner_path_name']}")
        p.close()


def circular_launches(p, prec, n, rows):
    torch = torch_mod()
    x = torch.zeros((rows, n), dtype=tdt(prec, "real"), device="cuda")
    p.convolve(x, torch.zeros((n // 2 + 1,), dtype=tdt(prec, "spec"), device="cuda"), x)
    torch.cuda.synchronize()
    return p.info()["last_launches"]


def test_two_scratch_chunks():
    """f32 N = 2^21 keeps 64 segments per 512 MB scratch chunk: 65 segments take two chunks"""
    torch = torch_mod()
    n, k = 1 << 21, (1 << 21) - 1000
    s = n - k + 1
    l = k - 1 + 64 * s + 500   # valid: ceil((l - k + 1) / s) = 65 segments
    p = plan("f32", n)
    x = reals("f32", (1, l), 5)
    h = taps((), k, 6)
    y = run(p, x, spectra("f32", h, n), k, "valid")
    launches = p.info()["last_launches"]
    err = per_transform_err(y, truth(x, h, "valid"))
    assert err.max() < TOL["f32"], err.max()
    assert launches == 2 + circular_launches(p, "f32", n, 64) + 2 + circular_launches(p, "f32", n, 1), launches
    p.close()
    torch.cuda.empty_cache()


def test_long_rows():
    p = plan("f32", 2048)
    err = check("f32", p, 2048, 1 << 22, 129, "full", 8, 0, seed=9)
    print(f"8 rows of 2^22 f32, N=2048, K=129: worst {err:.3e}")
    p.close()


def test_broadcasting():
    for prec, n in (("f32", 512), ("f64", 4096)):
        p = plan(prec, n)
        k, l = 77, 3000
        xs = reals(prec, (4, 3, l), 11)
        h = taps((3,), k, 12)
        err = per_transform_err(run(p, xs, spectra(prec, h, n), k, "same"), truth(xs, h, "same"))
        assert err.max() < TOL[prec], err.max()
        h = taps((4, 3), k, 13)   # F = batch
        err = per_transform_err(run(p, xs, spectra(prec, h, n), k, "full"), truth(xs, h, "full"))
        assert err.max() < TOL[prec], err.max()
        p.close()


def lconv_c(p, x, l, H, rows, k, mode, y, batch, stream=None):
    L = _lib.load()
    t = p._t
    if isinstance(x, np.ndarray):
        return getattr(L, f"fourier_b200_linear_convolve_real_{t}")(p._plan, x.ctypes.data, l, H.ctypes.data, rows, k,
                                                                   mode, y.ctypes.data, batch)
    torch = torch_mod()
    s = torch.cuda.current_stream().cuda_stream if stream is None else stream
    return getattr(L, f"fourier_b200_linear_convolve_real_async_{t}")(p._plan, x.data_ptr(), l, H.data_ptr(), rows, k,
                                                                     mode, y.data_ptr(), batch, s)


EXACT = [("f32", 2048, 129), ("f64", 512, 65), ("f32", 4096, 300), ("f32", 1009, 50)]


@pytest.mark.parametrize("prec,n,k", EXACT)
def test_exact_properties(prec, n, k):
    """Host memory == device memory, a row alone == the same row of the batch (spectrum row b mod F), a side stream ==
    the current stream, all bit for bit; NaN-poisoned outputs completely written, 16-byte guard bands untouched, the
    input and the spectrum unchanged.  F = 3 spectrum rows, a batch of 7 rows of odd length, every mode."""
    torch = torch_mod()
    p = plan(prec, n)
    batch, rows = 7, 3
    l = 3 * (n - k + 1) + 7
    x = reals(prec, (batch, l), 41)
    h = taps((rows,), k, 42)
    H = spectra(prec, h, n)
    xd, Hd = torch.from_numpy(x).cuda(), torch.from_numpy(H).cuda()
    guard = 16 // np.dtype(REAL[prec]).itemsize
    for code, mode in enumerate(MODES):
        ol = out_len(mode, l, k)
        buf = torch.full((batch * ol + 2 * guard,), float("nan"), dtype=xd.dtype, device="cuda")
        g0 = buf.cpu().numpy().copy()
        y = buf[guard:guard + batch * ol]
        assert lconv_c(p, xd, l, Hd, rows, k, code, y, batch) == 0, _lib.last_error()
        torch.cuda.synchronize()
        b = buf.cpu().numpy()
        assert np.array_equal(b[:guard].view(np.uint8), g0[:guard].view(np.uint8)), mode
        assert np.array_equal(b[-guard:].view(np.uint8), g0[-guard:].view(np.uint8)), mode
        ref = b[guard:guard + batch * ol].reshape(batch, ol)
        assert not np.isnan(ref).any(), mode
        assert torch.equal(xd.cpu(), torch.from_numpy(x)) and torch.equal(Hd.cpu(), torch.from_numpy(H))
        yh = np.full((batch, ol), np.nan, x.dtype)
        assert lconv_c(p, x, l, H, rows, k, code, yh, batch) == 0, _lib.last_error()
        assert np.array_equal(yh.view(np.uint8), ref.view(np.uint8)), ("host", mode)
        for r in range(batch):
            alone = torch.empty((1, ol), dtype=xd.dtype, device="cuda")
            p.convolve_linear(xd[r:r + 1].clone(), Hd[r % rows].clone(), k, alone, mode)
            torch.cuda.synchronize()
            assert np.array_equal(alone.cpu().numpy()[0].view(np.uint8), ref[r].view(np.uint8)), ("alone", mode, r)
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            ys = torch.full((batch, ol), float("nan"), dtype=xd.dtype, device="cuda")
            assert lconv_c(p, xd, l, Hd, rows, k, code, ys, batch, stream=s.cuda_stream) == 0
        s.synchronize()
        assert np.array_equal(ys.cpu().numpy().view(np.uint8), ref.view(np.uint8)), ("stream", mode)
        err = per_transform_err(ref, truth(x, h[np.arange(batch) % rows], mode))
        assert err.max() < TOL[prec], (mode, err.max())
    p.close()


def test_host_row_larger_than_the_staging_chunk():
    """one f32 row of 2^24 + 1000 samples (more than 64 MB): runs of segments staged with their input window"""
    torch = torch_mod()
    n, k, l = 2048, 129, (1 << 24) + 1000
    p = plan("f32", n)
    x = reals("f32", (2, l), 21)
    h = taps((2,), k, 22)
    H = spectra("f32", h, n)
    for mode in ("full", "valid"):
        yh = np.full((2, out_len(mode, l, k)), np.nan, np.float32)
        p.convolve_linear(x, H, k, yh, mode)
        yd = torch.empty(yh.shape, dtype=torch.float32, device="cuda")
        p.convolve_linear(torch.from_numpy(x).cuda(), torch.from_numpy(H).cuda(), k, yd, mode)
        torch.cuda.synchronize()
        assert np.array_equal(yh.view(np.uint8), yd.cpu().numpy().view(np.uint8)), mode
    err = per_transform_err(yh, truth(x, h, "valid"))
    assert err.max() < TOL["f32"], err.max()
    p.close()


@pytest.mark.parametrize("prec,n", [("f32", 2048), ("f64", 512), ("f32", 6000), ("f64", 1009)])
def test_agrees_with_zero_padding_and_convolve(prec, n):
    torch = torch_mod()
    p = plan(prec, n)
    k = n // 4
    l = n - k + 1   # l + k - 1 = n
    x = reals(prec, (5, l), 81)
    h = taps((5,), k, 82)
    H = spectra(prec, h, n)
    y = run(p, x, H, k, "full")
    xp = np.zeros((5, n), REAL[prec])
    xp[:, :l] = x
    yc = torch.from_numpy(xp).cuda()
    p.convolve(yc, torch.from_numpy(H).cuda(), yc)
    torch.cuda.synchronize()
    err = per_transform_err(y, yc.cpu().numpy().astype(np.longdouble))
    assert err.max() < TOL[prec], err.max()
    p.close()


def test_64_bit_offsets():
    """one f32 row of 2^31 + 1001 samples; the last 512 outputs against a direct long-double dot product"""
    torch = torch_mod()
    free, _ = torch.cuda.mem_get_info()
    if free < 24 * (1 << 30):
        pytest.skip(f"needs 24 GB of free device memory, {free / 2**30:.1f} GB free")
    n, k, l = 2048, 129, (1 << 31) + 1001
    p = plan("f32", n)
    g = torch.Generator(device="cuda").manual_seed(3)
    x = torch.randn((1, l), dtype=torch.float32, device="cuda", generator=g)
    h = taps((), k, 4)
    y = torch.empty((1, l + k - 1), dtype=torch.float32, device="cuda")
    p.convolve_linear(x, torch.from_numpy(spectra("f32", h, n)).cuda(), k, y, "full")
    torch.cuda.synchronize()
    tail = x[0, l - 512 - k:].cpu().numpy().astype(np.longdouble)
    full = np.convolve(tail, h.astype(np.longdouble))   # full[j] is output t0 + j wherever j >= k - 1
    # output t of the row is sum_m x[t - m] h[m]; the last 512 outputs are t = l + k - 1 - 512 .. l + k - 2
    t0 = l - 512 - k
    want = np.array([full[t - t0] for t in range(l + k - 1 - 512, l + k - 1)])
    got = y[0, -512:].cpu().numpy()
    err = np.abs(got - want).max() / np.abs(want).max()
    assert err < TOL["f32"], err
    del x, y
    p.close()
    torch.cuda.empty_cache()


def test_launch_counts():
    torch = torch_mod()
    for prec, n in FUSED:
        p = plan(prec, n)
        x = torch.from_numpy(reals(prec, (3, 5 * n), 1)).cuda()
        y = torch.empty((3, 5 * n + 9), dtype=x.dtype, device="cuda")
        p.convolve_linear(x, torch.from_numpy(spectra(prec, taps((), 10, 2), n)).cuda(), 10, y)
        assert p.info()["last_launches"] == 1, (prec, n)
        p.close()
    for prec, n, k in (("f32", 4096, 100), ("f32", 1 << 21, 3000), ("f64", 1 << 13, 9), ("f32", 1009, 30)):
        p = plan(prec, n)
        l = 3 * n
        x = torch.from_numpy(reals(prec, (2, l), 1)).cuda()
        y = torch.empty((2, l + k - 1), dtype=x.dtype, device="cuda")
        p.convolve_linear(x, torch.from_numpy(spectra(prec, taps((), k, 2), n)).cuda(), k, y)
        torch.cuda.synchronize()
        got = p.info()["last_launches"]
        segments = 2 * -(-(l + k - 1) // (n - k + 1))
        assert got == 2 + circular_launches(p, prec, n, segments), (prec, n, got)
        p.close()


def test_errors_are_refused_with_a_message():
    torch = torch_mod()
    L = _lib.load()
    n, k, l = 2048, 33, 5000
    for prec, t in (("f32", "float"), ("f64", "double")):
        p = plan(prec, n)
        esz = np.dtype(REAL[prec]).itemsize
        x = torch.zeros((4, l), dtype=tdt(prec, "real"), device="cuda")
        y = torch.zeros((4, l + k - 1), dtype=tdt(prec, "real"), device="cuda")
        H = torch.zeros((2, n // 2 + 1), dtype=tdt(prec, "spec"), device="cuda")
        sync = getattr(L, f"fourier_b200_linear_convolve_real_{t}")
        asyn = getattr(L, f"fourier_b200_linear_convolve_real_async_{t}")
        xp, yp, hp = x.data_ptr(), y.data_ptr(), H.data_ptr()
        cases = [
            ("taps > N", lambda: sync(p._plan, xp, l, hp, 2, n + 1, 0, yp, 4), 1, "taps"),
            ("taps > N, batch 0", lambda: asyn(p._plan, xp, l, hp, 2, n + 1, 0, yp, 0, None), 1, "taps"),
            ("identical in / out", lambda: sync(p._plan, xp, l, hp, 2, k, 1, xp, 4), 1, "overlap"),
            ("overlapping in / out", lambda: asyn(p._plan, xp, l, hp, 2, k, 0, xp + 64, 1, None), 1, "overlap"),
            ("spectrum overlaps out", lambda: asyn(p._plan, xp, l, yp + 256, 1, k, 0, yp, 4, None), 1, "spectrum"),
            ("host/device mix", lambda: sync(p._plan, xp, l, np.zeros((2, n // 2 + 1), SPEC[prec]).ctypes.data, 2, k, 0,
                                             yp, 4), 1, "host"),
            ("misaligned in", lambda: asyn(p._plan, xp + esz, l, hp, 2, k, 0, yp, 2, None), 716, "aligned"),
            ("misaligned out", lambda: sync(p._plan, xp, l, hp, 2, k, 0, yp + 8, 2), 716, "aligned"),
            ("misaligned spectrum", lambda: sync(p._plan, xp, l, hp + 8, 1, k, 0, yp, 2), 716, "aligned"),
        ]
        for name, call, code, word in cases:
            rc = call()
            assert rc == code, (name, rc)
            assert word in _lib.last_error(), (name, _lib.last_error())
        assert sync(p._plan, xp, l, hp, 2, k, 0, yp, 0) == 0   # batch 0
        assert p.info()["last_launches"] == 0
        Hc = torch.complex(torch.randn(n // 2 + 1, dtype=x.dtype, device="cuda"),
                           torch.randn(n // 2 + 1, dtype=x.dtype, device="cuda"))
        with pytest.raises(ValueError, match="resolve_conj"):
            p.convolve_linear(x, Hc.conj(), k, y)
        with pytest.raises(ValueError, match=str(l + k - 1)):
            p.convolve_linear(x, H, k, y[:, :-1].contiguous())
        with pytest.raises(ValueError, match=str(l)):
            p.convolve_linear(x, H, k, y, "same")
        with pytest.raises(ValueError, match="mode"):
            p.convolve_linear(x, H, k, y, "circular")
        with pytest.raises(ValueError, match="taps"):
            p.convolve_linear(x, H, n + 1, y)
        with pytest.raises(ValueError, match="valid"):
            p.convolve_linear(x[:, :10].contiguous(), H, k, y, "valid")
        with pytest.raises(TypeError):
            p.convolve_linear(x.to(torch.float16), H, k, y)
        with pytest.raises(TypeError):
            p.convolve_linear(x, H.real.contiguous(), k, y)
        with pytest.raises(ValueError):
            p.convolve_linear(x, torch.zeros((3, n // 2 + 1), dtype=H.dtype, device="cuda"), k, y)
        with pytest.raises(ValueError):
            p.convolve_linear(x[:3], H, k, y)
        with pytest.raises(ValueError):
            p.convolve_linear(x, H.cpu().numpy(), k, y)
        with pytest.raises(ValueError):
            p.convolve_linear(x[:, ::2], H, k, y[:, :l // 2 + k - 1])
        torch.cuda.synchronize()
        p.close()

"""Convolution of real rows, y = irfft(rfft(x) * H) (RealFft.convolve, fourier_b200_convolve_real_*), on the GPU: every
path against numpy in long double with one, three and one spectrum per row and with (B, C, N) inputs filtered per
channel, exact properties (in place, host memory, rows alone, streams), stray and missing stores, agreement with the
three-call composition, linear convolution by zero-padding, launch counts and refusals."""

import numpy as np
import pytest

import fourier_b200 as fb
from fourier_b200 import _lib
from helpers import per_transform_err

pytestmark = pytest.mark.gpu

TOL = {"f32": 1e-5, "f64": 1e-12}
REAL = {"f32": np.float32, "f64": np.float64}
SPEC = {"f32": np.complex64, "f64": np.complex128}


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


def spectra(prec, shape, n, seed):
    """Random bins (not the rfft of anything in particular), random imaginary parts in bins 0 and N/2 included."""
    rng = np.random.default_rng(seed)
    b = n // 2 + 1
    return (rng.standard_normal(tuple(shape) + (b,)) + 1j * rng.standard_normal(tuple(shape) + (b,))).astype(SPEC[prec])


def truth(x, H, n):
    """irfft(rfft(x) * H) in long double, H broadcast over x's leading shape as convolve does."""
    X = np.fft.rfft(np.asarray(x).astype(np.longdouble), axis=-1)
    return np.fft.irfft(X * np.asarray(H).astype(np.clongdouble), n=n, axis=-1)


def conv_c(p, x, H, rows, y, batch):
    """the C entry point with an explicit spectrum_rows: device tensors (async on torch's stream, then synchronised)
    or numpy arrays (the synchronous call)"""
    L = _lib.load()
    t = p._t
    if isinstance(x, np.ndarray):
        rc = getattr(L, f"fourier_b200_convolve_real_{t}")(p._plan, x.ctypes.data, H.ctypes.data, rows, y.ctypes.data,
                                                           batch)
    else:
        torch = torch_mod()
        rc = getattr(L, f"fourier_b200_convolve_real_async_{t}")(p._plan, x.data_ptr(), H.data_ptr(), rows,
                                                                 y.data_ptr(), batch,
                                                                 torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
    assert rc == 0, _lib.last_error()


def run(p, x, H, out=None):
    """convolve on device buffers -> numpy result"""
    torch = torch_mod()
    xd = torch.from_numpy(np.ascontiguousarray(x)).cuda()
    Hd = torch.from_numpy(np.ascontiguousarray(H)).cuda()
    y = torch.empty_like(xd) if out is None else out
    p.convolve(xd, Hd, y)
    torch.cuda.synchronize()
    return y.cpu().numpy()


def check(prec, n, batch, seed, shapes=None):
    """x of shape (batch, n) against F = 1, 3 (when batch allows) and batch spectra, and (B, C, N) with C filters;
    -> (worst error, plan info)."""
    p = plan(prec, n)
    x = reals(prec, (batch, n), seed)
    worst = 0.0
    cases = [((), x), ((batch,), x)]
    if batch % 3 == 0:
        cases.append(((3,), x.reshape(batch // 3, 3, n)))
    for hs, xs in cases + (shapes or []):
        H = spectra(prec, hs, n, seed + 1)
        err = per_transform_err(run(p, xs, H), truth(xs, H, n))
        assert err.max() < TOL[prec], (prec, n, xs.shape, hs, np.nonzero(err >= TOL[prec])[0][:8], err.max())
        worst = max(worst, err.max())
    info = p.info()
    p.close()
    return worst, info


@pytest.mark.parametrize("prec", ["f32", "f64"])
def test_every_size_up_to_256(prec):
    worst = {}
    for n in range(1, 257):
        err, info = check(prec, n, 6, seed=n)
        worst[info["path_name"]] = max(worst.get(info["path_name"], 0.0), err)
    print(f"{prec} N=1..256 worst per path: {worst}")
    assert set(worst) == {"real_fused", "real_half", "real_full"}


FUSED = [("f32", n) for n in (128, 256, 512, 1024, 2048)] + [("f64", n) for n in (128, 256, 512)]


@pytest.mark.parametrize("prec,n", FUSED)
def test_fused_sizes(prec, n):
    worst = 0.0
    for batch in (1, 3, 17, 1026):
        err, info = check(prec, n, batch, seed=batch)
        assert info["path_name"] == "real_fused"
        worst = max(worst, err)
    # (B, C, N) with one filter per channel, C not dividing the rows per CTA
    xs = reals(prec, (37, 7, n), 3)
    H = spectra(prec, (7,), n, 4)
    p = plan(prec, n)
    err = per_transform_err(run(p, xs, H), truth(xs, H, n))
    p.close()
    assert err.max() < TOL[prec], err.max()
    print(f"fused {prec} N={n}: worst per-row error {max(worst, err.max()):.3e}")


# half-length path: the inner plans of these sizes reach every complex path listed below
HALF = [("f32", 64, 3), ("f32", 4096, 3), ("f32", 1 << 21, 3), ("f32", 1 << 22, 3), ("f32", 2018, 3),
        ("f32", 4036, 3), ("f32", 200006, 3), ("f32", 1536, 3),
        ("f64", 1 << 13, 3), ("f64", 1 << 17, 3), ("f64", 1 << 18, 3), ("f64", 2018, 3), ("f64", 200006, 3)]


def test_half_path_over_every_inner_path():
    inner, kernels, worst = set(), [], {}
    for prec, n, batch in HALF:
        xs = reals(prec, (2, 3, n), n + 7)
        err, info = check(prec, n, batch, seed=n, shapes=[((3,), xs)])
        assert info["path_name"] == "real_half" and info["inner_size"] == n // 2, (prec, n, info)
        inner.add(info["inner_path_name"])
        p = plan(prec, n)
        kernels.append(p.kernel_name())
        p.close()
        key = (prec, info["inner_path_name"])
        worst[key] = max(worst.get(key, 0.0), err)
    print(f"half path worst per inner path: {worst}")
    assert {"onchip_cta", "twopass", "threepass", "bluestein_fused", "bluestein"} <= inner, inner
    assert any("fused_twopass_kernel" in k for k in kernels) and any("twopass::tile_kernel" in k for k in kernels)


@pytest.mark.parametrize("prec,n", [("f32", 1009), ("f32", 2187), ("f64", 1009), ("f64", 2187)])
def test_odd_sizes(prec, n):
    xs = reals(prec, (4, 3, n), 5)
    err, info = check(prec, n, 6, seed=n, shapes=[((3,), xs)])
    assert info["path_name"] == "real_full" and info["inner_size"] == n
    print(f"full path {prec} N={n}: worst {err:.3e}")


EXACT = [("f32", 2048), ("f32", 256), ("f64", 512), ("f32", 4096), ("f64", 1 << 13), ("f32", 1 << 21), ("f32", 1009),
         ("f64", 2187), ("f32", 2)]


@pytest.mark.parametrize("prec,n", EXACT)
def test_exact_properties(prec, n):
    """In place == out of place, host memory == device memory, a row alone == the same row in the batch, all bit for
    bit; F = 3 spectrum rows with a batch of 7 (through the C entry points: the Python shapes cannot say that)."""
    torch = torch_mod()
    p = plan(prec, n)
    batch, rows = 7, 3
    x = reals(prec, (batch, n), 41)
    H = spectra(prec, (rows,), n, 42)
    xd = torch.from_numpy(x).cuda()
    Hd = torch.from_numpy(H).cuda()
    y = torch.empty_like(xd)
    conv_c(p, xd, Hd, rows, y, batch)
    yi = xd.clone()
    conv_c(p, yi, Hd, rows, yi, batch)
    ref = y.cpu().numpy()
    assert np.array_equal(yi.cpu().numpy().view(np.uint8), ref.view(np.uint8)), "in place"
    yh = np.empty_like(x)
    conv_c(p, x, H, rows, yh, batch)
    assert np.array_equal(yh.view(np.uint8), ref.view(np.uint8)), "host"
    for b in range(batch):
        alone = torch.empty_like(xd[:1])
        p.convolve(xd[b:b + 1].clone(), Hd[b % rows:b % rows + 1].clone(), alone)   # a fresh allocation: odd f32
        torch.cuda.synchronize()                                                    # spectrum rows are misaligned
        assert np.array_equal(alone.cpu().numpy()[0].view(np.uint8), ref[b].view(np.uint8)), ("alone", b)
    err = per_transform_err(ref, truth(x, H[np.arange(batch) % rows], n))
    assert err.max() < TOL[prec], err.max()
    p.close()


@pytest.mark.parametrize("prec,n", [("f32", 2048), ("f64", 512), ("f32", 4096), ("f32", 1 << 21), ("f32", 1009)])
def test_non_default_stream_gives_the_same_bits(prec, n):
    torch = torch_mod()
    p = plan(prec, n)
    x = torch.from_numpy(reals(prec, (3, 2, n), 51)).cuda()
    H = torch.from_numpy(spectra(prec, (2,), n, 52)).cuda()
    y0 = torch.empty_like(x)
    p.convolve(x, H, y0)
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        y1 = torch.full_like(y0, float("nan"))
        p.convolve(x, H, y1)
    s.synchronize()
    assert torch.equal(y0.view(torch.uint8), y1.view(torch.uint8))
    p.close()


@pytest.mark.parametrize("prec,n", [("f32", 2048), ("f32", 256), ("f64", 512), ("f32", 4096), ("f64", 1 << 13),
                                    ("f32", 1 << 21), ("f32", 1009), ("f64", 2187)])
def test_no_stray_or_missing_stores(prec, n):
    """Output NaN-poisoned with guard rows after it; a decoy call on other input first; every sample stored, the guard
    rows keep their exact NaN bits, the input and the spectrum are unchanged.  F = 3 spectrum rows, batch 7."""
    torch = torch_mod()
    p = plan(prec, n)
    batch, guard, rows = 7, 2, 3
    x = torch.from_numpy(reals(prec, (batch, n), 61)).cuda()
    H = torch.from_numpy(spectra(prec, (rows,), n, 62)).cuda()
    x0, H0 = x.clone(), H.clone()
    decoy = torch.empty((batch + guard, n), dtype=tdt(prec, "real"), device="cuda")
    conv_c(p, torch.ones_like(x), H, rows, decoy, batch)
    out = torch.full((batch + guard, n), float("nan"), dtype=tdt(prec, "real"), device="cuda")
    g = out[batch:].cpu().numpy().copy()
    conv_c(p, x, H, rows, out, batch)
    o = out.cpu().numpy()
    assert not np.isnan(o[:batch]).any()
    assert np.array_equal(o[batch:].view(np.uint8), g.view(np.uint8))
    assert torch.equal(x.view(torch.uint8), x0.view(torch.uint8))
    assert torch.equal(H.view(torch.uint8), H0.view(torch.uint8))
    p.close()


@pytest.mark.parametrize("prec,n", [("f32", 2048), ("f64", 512), ("f32", 4096), ("f64", 1 << 13), ("f32", 1009)])
def test_agrees_with_the_three_call_composition(prec, n):
    torch = torch_mod()
    p = plan(prec, n)
    x = torch.from_numpy(reals(prec, (4, 3, n), 71)).cuda()
    H = torch.from_numpy(spectra(prec, (3,), n, 72)).cuda()
    y = torch.empty_like(x)
    p.convolve(x, H, y)
    X = torch.empty((4, 3, n // 2 + 1), dtype=tdt(prec, "spec"), device="cuda")
    p.rfft(x, X)
    y3 = torch.empty_like(x)
    p.irfft(X * H, y3)
    torch.cuda.synchronize()
    err = per_transform_err(y.cpu().numpy(), y3.cpu().numpy().astype(np.longdouble))
    assert err.max() < TOL[prec], err.max()
    p.close()


@pytest.mark.parametrize("prec,n", [("f32", 2048), ("f64", 512), ("f32", 6000), ("f64", 1009)])
def test_zero_padding_gives_linear_convolution(prec, n):
    """Rows of length len(x) and taps of length len(h), zero-padded to n >= len(x) + len(h) - 1: np.convolve, full."""
    torch = torch_mod()
    lx, lh = n // 2 + 3, n // 2 - 3
    assert lx + lh - 1 <= n
    rng = np.random.default_rng(81)
    x = rng.standard_normal((5, lx))
    h = rng.standard_normal((5, lh))
    xp = np.zeros((5, n), REAL[prec])
    hp = np.zeros((5, n), REAL[prec])
    xp[:, :lx] = x
    hp[:, :lh] = h
    p = plan(prec, n)
    Hd = torch.empty((5, n // 2 + 1), dtype=tdt(prec, "spec"), device="cuda")
    p.rfft(torch.from_numpy(hp).cuda(), Hd)
    y = run(p, xp, Hd.cpu().numpy())
    ref = np.stack([np.convolve(xp[b, :lx].astype(np.longdouble), hp[b, :lh].astype(np.longdouble)) for b in range(5)])
    err = per_transform_err(y[:, :lx + lh - 1], ref)
    assert err.max() < TOL[prec], err.max()
    tail = np.abs(y[:, lx + lh - 1:]).max() / np.abs(ref).max() if n > lx + lh - 1 else 0.0
    assert tail < TOL[prec], tail
    p.close()


def inner_launches(prec, m, batch):
    """launches of the complex plan of length m: Fft out of place, then UnscaledIfft in place, as convolve runs it"""
    torch = torch_mod()
    c = fb.create_fft_f32(m) if prec == "f32" else fb.create_fft_f64(m)
    z = torch.zeros((batch, m), dtype=tdt(prec, "spec"), device="cuda")
    w = torch.empty_like(z)
    c.transform(z, w, 0)
    torch.cuda.synchronize()
    total = c.info()["last_launches"]
    c.transform(w, w, 2)
    torch.cuda.synchronize()
    total += c.info()["last_launches"]
    c.close()
    return total


def test_launch_counts():
    torch = torch_mod()
    for prec, n in FUSED:
        p = plan(prec, n)
        x = torch.from_numpy(reals(prec, (9, n), 1)).cuda()
        p.convolve(x, torch.from_numpy(spectra(prec, (), n, 2)).cuda(), x)
        assert p.info()["last_launches"] == 1, (prec, n)
        assert p.kernel_name() == "onchip::onchip_real_kernel"
        p.close()
    for prec, n in (("f32", 4096), ("f32", 1 << 21), ("f64", 1 << 13), ("f32", 64), ("f32", 2018)):
        p = plan(prec, n)
        x = torch.from_numpy(reals(prec, (3, n), 1)).cuda()
        p.convolve(x, torch.from_numpy(spectra(prec, (), n, 2)).cuda(), torch.empty_like(x))
        torch.cuda.synchronize()
        assert p.info()["last_launches"] == inner_launches(prec, n // 2, 3) + 1, (prec, n)
        p.close()
    for prec, n in (("f32", 1009), ("f64", 2187)):
        p = plan(prec, n)
        x = torch.from_numpy(reals(prec, (3, n), 1)).cuda()
        p.convolve(x, torch.from_numpy(spectra(prec, (), n, 2)).cuda(), torch.empty_like(x))
        torch.cuda.synchronize()
        assert p.info()["last_launches"] == 3 + inner_launches(prec, n, 3), (prec, n)
        p.close()


def test_errors_are_refused_with_a_message():
    torch = torch_mod()
    L = _lib.load()
    n = 2048
    for prec, t in (("f32", "float"), ("f64", "double")):
        p = plan(prec, n)
        esz = np.dtype(REAL[prec]).itemsize
        x = torch.zeros((4, n), dtype=tdt(prec, "real"), device="cuda")
        y = torch.zeros((4, n), dtype=tdt(prec, "real"), device="cuda")
        H = torch.zeros((2, n // 2 + 1), dtype=tdt(prec, "spec"), device="cuda")
        sync = getattr(L, f"fourier_b200_convolve_real_{t}")
        asyn = getattr(L, f"fourier_b200_convolve_real_async_{t}")
        xp, yp, hp = x.data_ptr(), y.data_ptr(), H.data_ptr()
        cases = [
            ("null plan", lambda: sync(None, xp, hp, 2, yp, 4), 1, "null"),
            ("null in", lambda: asyn(p._plan, None, hp, 2, yp, 4, None), 1, "null"),
            ("null spectrum", lambda: sync(p._plan, xp, None, 2, yp, 4), 1, "null"),
            ("null out", lambda: sync(p._plan, xp, hp, 2, None, 4), 1, "null"),
            ("no rows", lambda: asyn(p._plan, xp, hp, 0, yp, 4, None), 1, "spectrum_rows"),
            ("partial overlap", lambda: sync(p._plan, xp, hp, 2, xp + 64, 2), 1, "overlap"),
            ("partial overlap async", lambda: asyn(p._plan, xp + 64, hp, 2, xp, 2, None), 1, "overlap"),
            ("spectrum overlaps out", lambda: asyn(p._plan, xp, yp + 256, 1, yp, 4, None), 1, "spectrum"),
            ("host/device mix", lambda: sync(p._plan, xp, np.zeros((2, n // 2 + 1), SPEC[prec]).ctypes.data, 2, yp, 4),
             1, "host"),
            ("misaligned in", lambda: asyn(p._plan, xp + esz, hp, 2, yp, 2, None), 716, "aligned"),
            ("misaligned out", lambda: sync(p._plan, xp, hp, 2, yp + 8, 2), 716, "aligned"),
            ("misaligned spectrum", lambda: sync(p._plan, xp, hp + 8, 1, yp, 2), 716, "aligned"),
        ]
        for name, call, code, word in cases:
            rc = call()
            assert rc == code, (name, rc)
            assert word in _lib.last_error(), (name, _lib.last_error())
        assert sync(p._plan, xp, hp, 2, yp, 0) == 0   # batch 0
        assert p.info()["last_launches"] == 0
        torch.cuda.synchronize()
        Hc = torch.complex(torch.randn(n // 2 + 1, dtype=x.dtype, device="cuda"),
                           torch.randn(n // 2 + 1, dtype=x.dtype, device="cuda"))
        with pytest.raises(ValueError, match="resolve_conj"):
            p.convolve(x, Hc.conj(), y)
        p.convolve(x, Hc.conj().resolve_conj(), y)
        xn = torch.complex(x, x).conj().imag   # a real view with the neg bit set
        assert xn.is_neg()
        with pytest.raises(ValueError, match="resolve_conj"):
            p.convolve(xn, H, y)
        with pytest.raises(TypeError):
            p.convolve(x.to(torch.float16), H, y)
        with pytest.raises(TypeError):
            p.convolve(x, H.real.contiguous(), y)
        with pytest.raises(ValueError):
            p.convolve(x, H, y[:3])
        with pytest.raises(ValueError):
            p.convolve(x, torch.zeros((3, n // 2 + 1), dtype=H.dtype, device="cuda"), y)   # 3 is not a trailing part
        with pytest.raises(ValueError):
            p.convolve(x, torch.zeros((5, 4, n // 2 + 1), dtype=H.dtype, device="cuda"), y)   # longer than the input's
        with pytest.raises(ValueError):
            p.convolve(x, H[:, :-1].contiguous(), y)
        with pytest.raises(ValueError):
            p.convolve(x, H.cpu().numpy(), y)   # host spectrum with device rows
        with pytest.raises(ValueError):
            p.convolve(x[:, ::2], H, y[:, ::2])
        p.close()

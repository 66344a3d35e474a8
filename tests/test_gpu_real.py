"""Real-input transforms (RealFft, fourier_b200_rfft_*) on the GPU: every path against numpy's rfft / irfft in long
double, exact properties (zero imaginary parts, batch independence, host == device), stray and missing stores, launch
counts, argument errors and streams."""

import numpy as np
import pytest

import fourier_b200 as fb
from fourier_b200 import _lib
from helpers import per_transform_err

pytestmark = pytest.mark.gpu

TOL = {"f32": 1e-5, "f64": 1e-12}
REAL = {"f32": np.float32, "f64": np.float64}
SPEC = {"f32": np.complex64, "f64": np.complex128}
FORWARD = (0, 3)
INVERSE = (1, 2, 4)


def torch_mod():
    import torch
    return torch


def plan(prec, n):
    return fb.create_rfft_f32(n) if prec == "f32" else fb.create_rfft_f64(n)


def scale_code(y, code, n):
    """Scale of Transform `code` relative to the real length n, in long double, applied to the unscaled forward (rfft)
    or unscaled inverse (n * irfft) transform y."""
    n = np.longdouble(n)
    if code == 1:
        return y / n
    if code in (3, 4):
        return y / np.sqrt(n)
    return y


def truth_rfft(x, code):
    x = np.asarray(x).astype(np.longdouble)
    return scale_code(np.fft.rfft(x, axis=-1), code, x.shape[-1])


def truth_irfft(X, n, code):
    X = np.asarray(X).astype(np.clongdouble)
    return scale_code(np.fft.irfft(X, n=n, axis=-1) * np.longdouble(n), code, n)


def real_input(prec, batch, n, seed):
    return np.random.default_rng(seed).standard_normal((batch, n)).astype(REAL[prec])


def spec_input(prec, batch, n, seed):
    """Random bins, Hermitian or not, with random imaginary parts in bins 0 and N/2 as well."""
    rng = np.random.default_rng(seed)
    b = n // 2 + 1
    return (rng.standard_normal((batch, b)) + 1j * rng.standard_normal((batch, b))).astype(SPEC[prec])


def run_forward(p, prec, x, code):
    torch = torch_mod()
    xd = torch.from_numpy(x).cuda()
    y = torch.empty(x.shape[:-1] + (x.shape[-1] // 2 + 1,), dtype=getattr(torch, np.dtype(SPEC[prec]).name),
                    device="cuda")
    p.rfft(xd, y, code)
    torch.cuda.synchronize()
    return y.cpu().numpy()


def run_inverse(p, prec, X, n, code):
    torch = torch_mod()
    Xd = torch.from_numpy(X).cuda()
    y = torch.empty(X.shape[:-1] + (n,), dtype=getattr(torch, np.dtype(REAL[prec]).name), device="cuda")
    p.irfft(Xd, y, code)
    torch.cuda.synchronize()
    return y.cpu().numpy()


def check_both(prec, n, batch, codes_f=(0,), codes_i=(1,), seed=0):
    """-> worst per-transform error over the forward and inverse codes."""
    p = plan(prec, n)
    worst = 0.0
    x = real_input(prec, batch, n, seed)
    ref = truth_rfft(x, 0)
    for code in codes_f:
        err = per_transform_err(run_forward(p, prec, x, code), scale_code(ref, code, n))
        assert err.max() < TOL[prec], (prec, n, batch, code, np.nonzero(err >= TOL[prec])[0][:8], err.max())
        worst = max(worst, err.max())
    X = spec_input(prec, batch, n, seed + 1)
    ref = truth_irfft(X, n, 2)
    for code in codes_i:
        err = per_transform_err(run_inverse(p, prec, X, n, code), scale_code(ref, code, n))
        assert err.max() < TOL[prec], (prec, n, batch, code, np.nonzero(err >= TOL[prec])[0][:8], err.max())
        worst = max(worst, err.max())
    info = p.info()
    p.close()
    return worst, info


@pytest.mark.parametrize("prec", ["f32", "f64"])
def test_every_size_up_to_256(prec):
    worst = {}
    for n in range(1, 257):
        err, info = check_both(prec, n, 3, seed=n)
        worst[info["path_name"]] = max(worst.get(info["path_name"], 0.0), err)
    print(f"{prec} N=1..256 worst per path: {worst}")
    assert set(worst) == {"real_fused", "real_half", "real_full"}


FUSED = [("f32", n) for n in (128, 256, 512, 1024, 2048)] + [("f64", n) for n in (128, 256, 512)]


@pytest.mark.parametrize("prec,n", FUSED)
def test_fused_sizes_all_codes(prec, n):
    p = plan(prec, n)
    assert p.info()["path_name"] == "real_fused" and p.info()["inner_size"] == 0
    worst = 0.0
    for batch in (1, 3, 17, 1000, 4099):
        x = real_input(prec, batch, n, batch)
        X = spec_input(prec, batch, n, batch + 1)
        ref_f = np.fft.rfft(x.astype(np.longdouble), axis=-1)
        ref_i = np.fft.irfft(X.astype(np.clongdouble), n=n, axis=-1) * np.longdouble(n)
        for code in FORWARD:
            err = per_transform_err(run_forward(p, prec, x, code), scale_code(ref_f, code, n))
            assert err.max() < TOL[prec], (batch, code, np.nonzero(err >= TOL[prec])[0][:8])
            worst = max(worst, err.max())
        for code in INVERSE:
            err = per_transform_err(run_inverse(p, prec, X, n, code), scale_code(ref_i, code, n))
            assert err.max() < TOL[prec], (batch, code, np.nonzero(err >= TOL[prec])[0][:8])
            worst = max(worst, err.max())
    print(f"fused {prec} N={n}: worst per-transform error {worst:.3e}")


# half-length path: the inner plans of these sizes reach every complex path listed below
HALF = [("f32", 64, 3), ("f32", 4096, 3), ("f32", 1 << 21, 3), ("f32", 1 << 22, 2), ("f32", 2018, 3),
        ("f32", 4036, 3), ("f32", 200006, 3), ("f32", 1536, 3),
        ("f64", 1 << 13, 3), ("f64", 1 << 17, 3), ("f64", 1 << 18, 2), ("f64", 2018, 3), ("f64", 200006, 2)]


def test_half_path_over_every_inner_path():
    inner, kernels, worst = set(), [], {}
    for prec, n, batch in HALF:
        err, info = check_both(prec, n, batch, codes_f=FORWARD, codes_i=INVERSE, seed=n)
        assert info["path_name"] == "real_half" and info["inner_size"] == n // 2, (prec, n, info)
        inner.add(info["inner_path_name"])
        p = plan(prec, n)
        kernels.append(p.kernel_name())
        p.close()
        worst[(prec, info["inner_path_name"])] = max(worst.get((prec, info["inner_path_name"]), 0.0), err)
    print(f"half path worst per inner path: {worst}")
    assert {"onchip_cta", "twopass", "threepass", "bluestein_fused", "bluestein"} <= inner, inner
    assert any("fused_twopass_kernel" in k for k in kernels) and any("twopass::tile_kernel" in k for k in kernels)
    assert all(k.startswith("real::untangle_kernel") for k in kernels)


@pytest.mark.parametrize("prec,n", [("f32", 1009), ("f32", 2187), ("f64", 1009), ("f64", 2187)])
def test_odd_sizes(prec, n):
    err, info = check_both(prec, n, 3, codes_f=FORWARD, codes_i=INVERSE, seed=n)
    assert info["path_name"] == "real_full" and info["inner_size"] == n
    print(f"full path {prec} N={n}: worst {err:.3e}")


@pytest.mark.parametrize("prec,n,batch,chunk", [("f32", 1 << 21, 67, 64), ("f64", 1 << 17, 515, 512)])
def test_batches_crossing_a_scratch_chunk(prec, n, batch, chunk):
    """Every row bit-identical to the same row alone; rows around the chunk boundary against long double; the launch
    count is that of the inner plan on each chunk plus one untangle / tangle launch per chunk."""
    torch = torch_mod()
    p = plan(prec, n)
    cplx = fb.create_fft_f32(n // 2) if prec == "f32" else fb.create_fft_f64(n // 2)
    x = real_input(prec, batch, n, 5)
    X = spec_input(prec, batch, n, 6)
    for direction in ("forward", "inverse"):
        if direction == "forward":
            src, code = torch.from_numpy(x).cuda(), 0
            dst = torch.empty((batch, n // 2 + 1), dtype=getattr(torch, np.dtype(SPEC[prec]).name), device="cuda")
            call = p.rfft
        else:
            src, code = torch.from_numpy(X).cuda(), 1
            dst = torch.empty((batch, n), dtype=getattr(torch, np.dtype(REAL[prec]).name), device="cuda")
            call = p.irfft
        call(src, dst, code)
        torch.cuda.synchronize()
        launches = p.info()["last_launches"]
        full = dst.cpu().numpy()
        for b in range(batch):
            alone = torch.empty_like(dst[:1])
            call(src[b:b + 1].clone(), alone, code)   # a fresh allocation: odd f32 spectrum rows are not 16-byte aligned
            torch.cuda.synchronize()
            assert np.array_equal(alone.cpu().numpy()[0].view(np.uint8), full[b].view(np.uint8)), (direction, b)
        rows = [0, chunk - 1, chunk, batch - 1]
        ref = truth_rfft(x[rows], code) if direction == "forward" else truth_irfft(X[rows], n, code)
        err = per_transform_err(full[rows], ref)
        assert err.max() < TOL[prec], (direction, err)
        # inner launches per chunk
        expect = 0
        for nb in (chunk, batch - chunk):
            z = torch.zeros((nb, n // 2), dtype=getattr(torch, np.dtype(SPEC[prec]).name), device="cuda")
            cplx.transform(z, torch.empty_like(z), 0 if direction == "forward" else 2)
            torch.cuda.synchronize()
            expect += cplx.info()["last_launches"] + 1
        assert launches == expect, (direction, launches, expect)
        print(f"{prec} N={n} batch={batch} {direction}: boundary rows worst {err.max():.3e}, {launches} launches")
    cplx.close()
    p.close()


EXACT = [("f32", 2048), ("f32", 4096), ("f32", 1009), ("f64", 512), ("f64", 1 << 13), ("f64", 2187), ("f32", 2)]


@pytest.mark.parametrize("prec,n", EXACT)
def test_exact_properties(prec, n):
    torch = torch_mod()
    p = plan(prec, n)
    batch = 5
    x = real_input(prec, batch, n, 11)
    for code in FORWARD:
        y = run_forward(p, prec, x, code)
        edges = [0] + ([n // 2] if n % 2 == 0 else [])
        for k in edges:
            im = y[:, k].imag
            assert np.all(im == 0) and not np.any(np.signbit(im)), (code, k, im)
        # batch independence: every row as the same transform alone
        for b in range(batch):
            assert np.array_equal(run_forward(p, prec, x[b:b + 1], code)[0].view(np.uint8), y[b].view(np.uint8))
        # host buffers give the device bits
        yh = np.empty_like(y)
        p.rfft(x, yh, code)
        assert np.array_equal(yh.view(np.uint8), y.view(np.uint8))
        # round trip
        pair = {0: 1, 3: 4}[code]
        back = run_inverse(p, prec, y, n, pair)
        assert per_transform_err(back, x.astype(np.longdouble)).max() < TOL[prec]
    X = spec_input(prec, batch, n, 12)
    for code in INVERSE:
        y = run_inverse(p, prec, X, n, code)
        X2 = X.copy()
        X2[:, 0] = X2[:, 0].real + 1j * np.random.default_rng(code).standard_normal(batch)
        if n % 2 == 0:
            X2[:, n // 2] = X2[:, n // 2].real + 1j * np.random.default_rng(code + 9).standard_normal(batch)
        assert np.array_equal(run_inverse(p, prec, X2, n, code).view(np.uint8), y.view(np.uint8)), code
        for b in range(batch):
            assert np.array_equal(run_inverse(p, prec, X[b:b + 1], n, code)[0].view(np.uint8), y[b].view(np.uint8))
        yh = np.empty_like(y)
        p.irfft(X, yh, code)
        assert np.array_equal(yh.view(np.uint8), y.view(np.uint8))
    p.close()
    torch.cuda.synchronize()


@pytest.mark.parametrize("prec,n", [("f32", 2048), ("f32", 256), ("f32", 4096), ("f32", 1009), ("f64", 512),
                                    ("f64", 1 << 13), ("f64", 2187), ("f32", 1 << 21)])
def test_no_stray_or_missing_stores(prec, n):
    """Outputs NaN-poisoned with one guard row; a decoy call on other input first; every in-range element is stored and
    the guard row keeps its exact NaN bits."""
    torch = torch_mod()
    p = plan(prec, n)
    batch = 7
    rdt = getattr(torch, np.dtype(REAL[prec]).name)
    sdt = getattr(torch, np.dtype(SPEC[prec]).name)
    x = torch.from_numpy(real_input(prec, batch, n, 21)).cuda()
    X = torch.from_numpy(spec_input(prec, batch, n, 22)).cuda()
    decoy_out = torch.empty((batch + 1, n // 2 + 1), dtype=sdt, device="cuda")
    p.rfft(torch.ones_like(x), decoy_out[:batch], 0)
    out = torch.full((batch + 1, n // 2 + 1), complex(float("nan"), float("nan")), dtype=sdt, device="cuda")
    guard = out[batch].cpu().numpy().copy()
    p.rfft(x, out[:batch], 0)
    o = out.cpu().numpy()
    assert not np.isnan(o[:batch].view(REAL[prec])).any()
    assert np.array_equal(o[batch].view(np.uint8), guard.view(np.uint8))

    decoy_r = torch.empty((batch + 1, n), dtype=rdt, device="cuda")
    p.irfft(torch.ones_like(X), decoy_r[:batch], 1)
    outr = torch.full((batch + 1, n), float("nan"), dtype=rdt, device="cuda")
    guard = outr[batch].cpu().numpy().copy()
    p.irfft(X, outr[:batch], 1)
    o = outr.cpu().numpy()
    assert not np.isnan(o[:batch]).any()
    assert np.array_equal(o[batch].view(np.uint8), guard.view(np.uint8))
    p.close()


def test_launch_counts_and_kernel_names():
    torch = torch_mod()
    for prec, n in FUSED:
        p = plan(prec, n)
        x = torch.from_numpy(real_input(prec, 9, n, 1)).cuda()
        y = torch.empty((9, n // 2 + 1), dtype=getattr(torch, np.dtype(SPEC[prec]).name), device="cuda")
        p.rfft(x, y, 0)
        assert p.info()["last_launches"] == 1
        p.irfft(y, x, 1)
        assert p.info()["last_launches"] == 1
        assert p.kernel_name() == "onchip::onchip_real_kernel"
        p.close()
    for prec, n in (("f32", 4096), ("f32", 1 << 21), ("f64", 1 << 13), ("f32", 64)):
        p = plan(prec, n)
        c = fb.create_fft_f32(n // 2) if prec == "f32" else fb.create_fft_f64(n // 2)
        sdt = getattr(torch, np.dtype(SPEC[prec]).name)
        x = torch.from_numpy(real_input(prec, 3, n, 1)).cuda()
        y = torch.empty((3, n // 2 + 1), dtype=sdt, device="cuda")
        z = torch.zeros((3, n // 2), dtype=sdt, device="cuda")
        p.rfft(x, y, 0)
        c.transform(z, torch.empty_like(z), 0)
        torch.cuda.synchronize()
        assert p.info()["last_launches"] == c.info()["last_launches"] + 1
        p.irfft(y, x, 1)
        c.transform(z, torch.empty_like(z), 2)
        torch.cuda.synchronize()
        assert p.info()["last_launches"] == c.info()["last_launches"] + 1
        assert p.kernel_name().startswith("real::untangle_kernel") and c.kernel_name() in p.kernel_name()
        assert (p.info()["n1"], p.info()["n2"]) == (c.info()["n1"], c.info()["n2"])
        c.close()
        p.close()
    p = fb.create_rfft_f64(1009)
    assert p.kernel_name().startswith("real::widen_kernel")
    p.close()


def test_errors_are_refused_with_a_message():
    torch = torch_mod()
    L = _lib.load()
    n = 2048
    for prec, t in (("f32", "float"), ("f64", "double")):
        p = plan(prec, n)
        esz = np.dtype(REAL[prec]).itemsize
        x = torch.zeros((4, n), dtype=getattr(torch, np.dtype(REAL[prec]).name), device="cuda")
        y = torch.zeros((4, n // 2 + 1), dtype=getattr(torch, np.dtype(SPEC[prec]).name), device="cuda")
        fwd = getattr(L, f"fourier_b200_rfft_forward_{t}")
        fwd_a = getattr(L, f"fourier_b200_rfft_forward_async_{t}")
        inv = getattr(L, f"fourier_b200_rfft_inverse_{t}")
        inv_a = getattr(L, f"fourier_b200_rfft_inverse_async_{t}")
        cases = [
            ("forward code to inverse", lambda: inv(p._plan, y.data_ptr(), x.data_ptr(), 2, 0), "inverse"),
            ("inverse code to forward", lambda: fwd(p._plan, x.data_ptr(), y.data_ptr(), 2, 1), "forward"),
            ("code 7", lambda: fwd_a(p._plan, x.data_ptr(), y.data_ptr(), 2, 7, None), "unknown"),
            ("code 7 inverse", lambda: inv_a(p._plan, y.data_ptr(), x.data_ptr(), 2, 7, None), "unknown"),
            ("misaligned", lambda: fwd_a(p._plan, x.data_ptr() + esz, y.data_ptr(), 2, 0, None), "aligned"),
            ("misaligned out", lambda: inv(p._plan, y.data_ptr(), x.data_ptr() + 8, 2, 1), "aligned"),
            ("overlap", lambda: fwd(p._plan, x.data_ptr(), x.data_ptr() + 64, 2, 0), "overlap"),
            ("overlap async", lambda: inv_a(p._plan, y.data_ptr(), y.data_ptr(), 1, 1, None), "overlap"),
            ("host/device mix", lambda: fwd(p._plan, np.zeros((2, n), REAL[prec]).ctypes.data, y.data_ptr(), 2, 0),
             "host"),
            ("null plan", lambda: fwd(None, x.data_ptr(), y.data_ptr(), 2, 0), "null"),
        ]
        for name, call, word in cases:
            rc = call()
            assert rc != 0, name
            assert word in _lib.last_error(), (name, _lib.last_error())
        assert fwd(p._plan, x.data_ptr(), y.data_ptr(), 0, 0) == 0   # batch 0
        assert p.info()["last_launches"] == 0
        torch.cuda.synchronize()
        with pytest.raises(TypeError):
            p.rfft(x.to(torch.float16), y)
        with pytest.raises(TypeError):
            p.rfft(y, y)
        with pytest.raises(ValueError):
            p.rfft(x[:, :n - 2].contiguous(), y)
        with pytest.raises(ValueError):
            p.rfft(x, y[:3])
        with pytest.raises(ValueError):
            p.irfft(y, x[:, ::2])
        with pytest.raises(TypeError):
            p.irfft(x, x)
        with pytest.raises(TypeError):
            p.rfft(np.zeros((2, n), np.float16), np.zeros((2, n // 2 + 1), SPEC[prec]))
        with pytest.raises(ValueError):
            p.rfft(x, np.zeros((4, n // 2 + 1), SPEC[prec]))
        p.close()
    assert fb.create_rfft_f32(2048).size() == 2048
    with pytest.raises(RuntimeError):
        fb.create_rfft_f32(0)


@pytest.mark.parametrize("prec,n", [("f32", 2048), ("f32", 1 << 20), ("f64", 1009)])
def test_non_default_stream_gives_the_same_bits(prec, n):
    torch = torch_mod()
    p = plan(prec, n)
    x = torch.from_numpy(real_input(prec, 6, n, 31)).cuda()
    y0 = torch.empty((6, n // 2 + 1), dtype=getattr(torch, np.dtype(SPEC[prec]).name), device="cuda")
    p.rfft(x, y0, 0)
    r0 = torch.empty_like(x)
    p.irfft(y0, r0, 1)
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        y1 = torch.full_like(y0, complex(float("nan"), float("nan")))
        r1 = torch.full_like(r0, float("nan"))
        p.rfft(x, y1, 0)
        p.irfft(y1, r1, 1)
    s.synchronize()
    assert torch.equal(y0.view(torch.uint8), y1.view(torch.uint8))
    assert torch.equal(r0.view(torch.uint8), r1.view(torch.uint8))
    p.close()

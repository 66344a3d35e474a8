"""Analytic signal and envelope of real rows (RealFft.hilbert / envelope, fourier_b200_hilbert_*) on the GPU: every fused
size class with both outputs, the half-length path (N = 2, 4, 64, 400, 4096 and f32 2^21 on the persistent two-pass
kernel) and the full-length path (N = 1, 3, 97 and a Bluestein 1009), against scipy.signal.hilbert in float64 on the same
(rounded) inputs; the real part equal to the input bit for bit; the envelope against abs of scipy's and of this library's
analytic signal; the envelope in place against out of place, rows of a periodic batch against the row alone, and host
against device memory, all bit for bit; a side stream, two scratch chunks on both other paths with their launch counts,
one launch on the fused path, leading shapes, batch 0 and refusals.  Every output is NaN-filled before the call, and a
guard region behind it must stay untouched."""

import numpy as np
import pytest

import fourier_b200 as fb
from fourier_b200 import _lib

pytestmark = pytest.mark.gpu

TOL = {"f32": 2e-5, "f64": 1e-12}
REAL = {"f32": np.float32, "f64": np.float64}
CPLX = {"f32": np.complex64, "f64": np.complex128}
# (N, FFTs per CTA of its fused class)
FUSED = [("f32", 128, 32), ("f32", 256, 32), ("f32", 512, 16), ("f32", 1024, 16), ("f32", 2048, 8), ("f64", 128, 32),
         ("f64", 256, 32), ("f64", 512, 16)]
GUARD = 64


def torch_mod():
    import torch
    return torch


def plan(prec, n):
    return fb.create_rfft_f32(n) if prec == "f32" else fb.create_rfft_f64(n)


def reals(prec, shape, seed):
    return np.random.default_rng(seed).standard_normal(shape).astype(REAL[prec])


def ref_hilbert(x):
    from scipy.signal import hilbert
    return hilbert(np.asarray(x, np.float64), axis=-1)


def dev_run(p, x, envelope=False):
    """device hilbert (or envelope) of numpy x into a NaN-filled output followed by a guard region -> numpy output"""
    torch = torch_mod()
    count = int(np.prod(x.shape, dtype=np.int64))
    dt = getattr(torch, np.dtype(REAL[p.real] if envelope else CPLX[p.real]).name)
    buf = torch.full((count + GUARD,), float("nan"), dtype=dt, device="cuda")
    buf[count:] = 12345.0
    out = buf[:count].view(x.shape)
    (p.envelope if envelope else p.hilbert)(torch.from_numpy(x).cuda(), out)
    torch.cuda.synchronize()
    assert torch.all(buf[count:] == 12345.0), "a write past the output"
    return out.cpu().numpy()


def row_err(got, ref):
    """worst over rows of max |got - ref| / max |ref|; NaN counts as infinite"""
    g = np.asarray(got).reshape(-1, np.shape(ref)[-1]).astype(np.complex128)
    r = np.asarray(ref).reshape(g.shape).astype(np.complex128)
    e = np.abs(g - r).max(axis=1) / np.maximum(np.abs(r).max(axis=1), 1e-300)
    return float(np.where(np.isnan(e), np.inf, e).max())


def ulps(a, b):
    """|a - b| in units of the last place of b (both of one real dtype)"""
    return np.abs(a.astype(np.float64) - b.astype(np.float64)) / np.spacing(np.abs(b))


def launches(p):
    return p.info()["last_launches"]


def inner_launches(prec, m, rows, half):
    """launches of the complex plan of length m on `rows` rows as the other paths run it: a forward, out of place from
    the input rows into the scratch at half length, in place at full length, then an unscaled inverse in place"""
    torch = torch_mod()
    c = fb.create_fft_f32(m) if prec == "f32" else fb.create_fft_f64(m)
    ct = torch.complex64 if prec == "f32" else torch.complex128
    x = torch.zeros(rows, m, dtype=ct, device="cuda")
    y = torch.empty_like(x)
    if half:
        c.transform(x, y, fb.Transform.Fft)
    else:
        c.transform_in_place(y, fb.Transform.Fft)
    torch.cuda.synchronize()
    total = c.info()["last_launches"]
    c.transform_in_place(y, fb.Transform.UnscaledIfft)
    torch.cuda.synchronize()
    return total + c.info()["last_launches"]


def check_both(p, x, prec):
    """analytic and envelope of x against scipy; the real part exact; the envelope against abs of both analytic signals"""
    z = dev_run(p, x)
    ref = ref_hilbert(x)
    assert row_err(z, ref) < TOL[prec]
    assert np.array_equal(z.real, x)
    env = dev_run(p, x, envelope=True)
    assert row_err(env, np.abs(ref)) < TOL[prec]
    assert ulps(env, np.abs(z)).max() <= 4
    return z, env


@pytest.mark.parametrize("prec,n,c", FUSED)
def test_fused_size_classes(prec, n, c):
    """3 C + 5 rows (a partial group) in one launch per output, against scipy"""
    p = plan(prec, n)
    assert p.info()["path_name"] == "real_fused"
    x = reals(prec, (3 * c + 5, n), n)
    dev_run(p, x)
    assert launches(p) == 1
    dev_run(p, x, envelope=True)
    assert launches(p) == 1
    check_both(p, x, prec)


@pytest.mark.parametrize("prec", ("f32", "f64"))
@pytest.mark.parametrize("n", (2, 4, 64, 400, 4096))
def test_real_half(prec, n):
    p = plan(prec, n)
    assert p.info()["path_name"] == "real_half"
    x = reals(prec, (7, n), n + 1)
    check_both(p, x, prec)
    assert launches(p) == 2 + inner_launches(prec, n // 2, 7, True)


def test_real_half_on_the_persistent_two_pass_kernel():
    """f32 N = 2^21: the inner plan of length 2^20 is the persistent two-pass kernel"""
    n = 1 << 21
    p = plan("f32", n)
    assert p.info()["path_name"] == "real_half" and p.info()["inner_path_name"] == "twopass"
    check_both(p, reals("f32", (2, n), 21), "f32")


@pytest.mark.parametrize("prec", ("f32", "f64"))
@pytest.mark.parametrize("n", (1, 3, 97, 1009))
def test_real_full(prec, n):
    p = plan(prec, n)
    assert p.info()["path_name"] == "real_full"
    if n == 1009:
        assert p.info()["inner_path_name"] in ("bluestein", "bluestein_fused")
    x = reals(prec, (5, n), n + 2)
    check_both(p, x, prec)
    assert launches(p) == 3 + inner_launches(prec, n, 5, False)


@pytest.mark.parametrize("prec,n", (("f32", 2048), ("f64", 512), ("f32", 400), ("f64", 97)))
def test_in_place_rows_alone_and_host_memory_give_the_same_bits(prec, n):
    torch = torch_mod()
    p = plan(prec, n)
    base = reals(prec, (5, n), 3 * n)
    x = np.concatenate([base] * 9 + [base[:2]])   # a periodic batch of 47 rows
    z = dev_run(p, x)
    env = dev_run(p, x, envelope=True)
    for r in range(5):
        assert np.array_equal(z[r::5], np.broadcast_to(dev_run(p, base[r:r + 1]), z[r::5].shape)), r
        assert np.array_equal(env[r::5], np.broadcast_to(dev_run(p, base[r:r + 1], True), env[r::5].shape)), r
    xd = torch.from_numpy(x).cuda()
    p.envelope(xd, xd)
    torch.cuda.synchronize()
    assert np.array_equal(xd.cpu().numpy(), env)
    host = np.full(x.shape, np.nan, CPLX[prec])
    p.hilbert(x, host)
    assert np.array_equal(host, z)
    host_env = np.full_like(x, np.nan)
    p.envelope(x, host_env)
    assert np.array_equal(host_env, env)
    xh = x.copy()
    p.envelope(xh, xh)
    assert np.array_equal(xh, env)


def test_async_on_a_side_stream():
    torch = torch_mod()
    p = plan("f32", 1024)
    x = reals("f32", (100, 1024), 41)
    ref = dev_run(p, x)
    s = torch.cuda.Stream()
    xd = torch.from_numpy(x).cuda()
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        out = torch.full((100, 1024), complex(float("nan"), float("nan")), dtype=torch.complex64, device="cuda")
        p.hilbert(xd, out)
    s.synchronize()
    assert np.array_equal(out.cpu().numpy(), ref)


@pytest.mark.parametrize("prec,n,row_bytes,extra", (("f32", 4096, 4096 * 4, 2), ("f64", 1009, 1009 * 16, 3)))
def test_two_scratch_chunks(prec, n, row_bytes, extra):
    """a batch over two 512 MB scratch chunks (N reals per row at half length, N complex values at full length): the
    launch count of two chunks, and the rows on both sides of the cut"""
    chunk = (512 << 20) // row_bytes
    rows = chunk + 1000
    p = plan(prec, n)
    x = reals(prec, (rows, n), 77)
    m = n // 2 if n % 2 == 0 else n
    half = n % 2 == 0
    want = (extra + inner_launches(prec, m, chunk, half)) + (extra + inner_launches(prec, m, rows - chunk, half))
    pick = [0, chunk - 1, chunk, rows - 1]
    ref = ref_hilbert(x[pick])
    z = dev_run(p, x)
    assert launches(p) == want
    assert row_err(z[pick], ref) < TOL[prec]
    assert np.array_equal(z.real, x)
    env = dev_run(p, x, envelope=True)
    assert launches(p) == want
    assert row_err(env[pick], np.abs(ref)) < TOL[prec]


def test_leading_shapes_and_batch_zero():
    torch = torch_mod()
    p = plan("f32", 256)
    x = reals("f32", (2, 3, 256), 61)
    z = dev_run(p, x)
    assert z.shape == (2, 3, 256)
    assert np.array_equal(z.reshape(6, 256), dev_run(p, x.reshape(6, 256)))
    env = dev_run(p, x, envelope=True)
    assert env.shape == (2, 3, 256)
    p.hilbert(torch.empty((0, 256), device="cuda"), torch.empty((0, 256), dtype=torch.complex64, device="cuda"))
    p.envelope(torch.empty((4, 0, 256), device="cuda"), torch.empty((4, 0, 256), device="cuda"))
    # the C entry point at batch 0 succeeds and launches nothing
    L = _lib.load()
    xd = torch.zeros(256, device="cuda")
    zd = torch.zeros(256, dtype=torch.complex64, device="cuda")
    assert L.fourier_b200_hilbert_float(p._plan, xd.data_ptr(), zd.data_ptr(), 0, 0) == 0
    assert launches(p) == 0


def test_refusals():
    torch = torch_mod()
    p = plan("f32", 512)
    x = torch.zeros(4, 512, device="cuda")
    z = torch.empty(4, 512, dtype=torch.complex64, device="cuda")
    with pytest.raises(ValueError, match="last dimension"):
        p.hilbert(x, torch.empty(4, 257, dtype=torch.complex64, device="cuda"))
    with pytest.raises(ValueError, match="shapes differ"):
        p.hilbert(x, torch.empty(3, 512, dtype=torch.complex64, device="cuda"))
    with pytest.raises(TypeError, match="expected"):
        p.hilbert(x, torch.empty(4, 512, device="cuda"))   # real output for the analytic signal
    with pytest.raises(TypeError, match="expected"):
        p.envelope(x, z)                                      # complex output for the envelope
    with pytest.raises(TypeError, match="expected"):
        p.hilbert(x.double(), z)
    with pytest.raises(ValueError, match="host or both be device"):
        p.hilbert(x, np.zeros((4, 512), np.complex64))
    with pytest.raises(ValueError, match="conj"):
        p.envelope(x._neg_view(), x)
    # the analytic signal may not overlap its input: a complex view of the input's own storage
    flat = torch.zeros(8 * 512, device="cuda")
    with pytest.raises(RuntimeError, match="overlap"):
        p.hilbert(flat[:4 * 512].view(4, 512), torch.view_as_complex(flat.view(4, 512, 2)))
    # the C entry points check a partial overlap, a mix of host and device memory and the alignment themselves
    L = _lib.load()
    rc = L.fourier_b200_hilbert_float(p._plan, flat.data_ptr(), flat.data_ptr() + 512 * 4, 4, 1)
    assert rc == 1 and "overlap" in _lib.last_error()
    rc = L.fourier_b200_hilbert_float(p._plan, flat.data_ptr(), flat.data_ptr(), 4, 0)
    assert rc == 1 and "out of place" in _lib.last_error()
    host = np.zeros((4, 512), np.complex64)
    rc = L.fourier_b200_hilbert_float(p._plan, x.data_ptr(), host.ctypes.data, 4, 0)
    assert rc == 1 and "host or both be device" in _lib.last_error()
    rc = L.fourier_b200_hilbert_async_float(p._plan, flat.data_ptr() + 4, flat.data_ptr() + 4, 4, 1, None)
    assert rc == 716, rc
    assert "16-byte aligned" in _lib.last_error()

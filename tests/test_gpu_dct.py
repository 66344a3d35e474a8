"""Discrete cosine transforms of real rows (RealFft.dct / idct, fourier_b200_dct_*) on the GPU: every fused size class,
type and norm, the half-length path (N = 2, 4, 64, 400, 4096 and f32 2^21 on the persistent two-pass kernel) and the
full-length path (N = 1, 3, 97 and a Bluestein 1009), against scipy.fft.dct in float64 on the same (rounded) inputs;
idct round trips and the orthonormal norm; in place against out of place, rows of a periodic batch against the row
alone, and host against device memory, all bit for bit; a side stream, two scratch chunks on both other paths with
their launch counts, one launch on the fused path, leading shapes, batch 0 and refusals.  Every output is NaN-filled
before the call, and a guard region behind it must stay untouched."""

import numpy as np
import pytest

import fourier_b200 as fb
from fourier_b200 import _lib

pytestmark = pytest.mark.gpu

TOL = {"f32": 2e-5, "f64": 1e-12}
REAL = {"f32": np.float32, "f64": np.float64}
NORMS = ("backward", "ortho", "forward")
# (N, FFTs per CTA of its fused class)
FUSED = [("f32", 128, 32), ("f32", 256, 32), ("f32", 512, 16), ("f32", 1024, 16), ("f32", 2048, 8), ("f64", 128, 32),
         ("f64", 256, 32), ("f64", 512, 16)]
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


def ref_dct(x, t, norm):
    from scipy.fft import dct
    return dct(np.asarray(x, np.float64), type=t, norm=norm, axis=-1)


def dev_dct(p, x, t, norm, inverse=False):
    """device dct (or idct) of numpy x into a NaN-filled output followed by a guard region -> numpy output"""
    torch = torch_mod()
    count = int(np.prod(x.shape, dtype=np.int64))
    buf = torch.full((count + GUARD,), float("nan"), dtype=tdt(p.real), device="cuda")
    buf[count:] = 12345.0
    out = buf[:count].view(x.shape)
    (p.idct if inverse else p.dct)(torch.from_numpy(x).cuda(), out, type=t, norm=norm)
    torch.cuda.synchronize()
    assert torch.all(buf[count:] == 12345.0), "a write past the output"
    return out.cpu().numpy()


def row_err(got, ref):
    """worst over rows of max |got - ref| / max |ref|; NaN counts as infinite"""
    g = np.asarray(got, np.float64).reshape(-1, np.shape(ref)[-1])
    r = np.asarray(ref, np.float64).reshape(g.shape)
    e = np.abs(g - r).max(axis=1) / np.maximum(np.abs(r).max(axis=1), 1e-300)
    return float(np.where(np.isnan(e), np.inf, e).max())


def launches(p):
    return p.info()["last_launches"]


def inner_launches(prec, m, rows):
    """launches of the complex plan of length m on `rows` rows in place, as the dct runs it in its scratch"""
    torch = torch_mod()
    c = fb.create_fft_f32(m) if prec == "f32" else fb.create_fft_f64(m)
    ct = torch.complex64 if prec == "f32" else torch.complex128
    c.fft_in_place(torch.zeros(rows, m, dtype=ct, device="cuda"))
    torch.cuda.synchronize()
    return c.info()["last_launches"]


@pytest.mark.parametrize("prec,n,c", FUSED)
@pytest.mark.parametrize("t", (2, 3))
@pytest.mark.parametrize("norm", NORMS)
def test_fused_size_classes(prec, n, c, t, norm):
    """3 C + 5 rows (a partial group) in one launch, against scipy"""
    p = plan(prec, n)
    assert p.info()["path_name"] == "real_fused"
    x = reals(prec, (3 * c + 5, n), n + 10 * t)
    got = dev_dct(p, x, t, norm)
    assert launches(p) == 1
    assert row_err(got, ref_dct(x, t, norm)) < TOL[prec]


@pytest.mark.parametrize("prec", ("f32", "f64"))
@pytest.mark.parametrize("n", (2, 4, 64, 400, 4096))
def test_real_half(prec, n):
    p = plan(prec, n)
    assert p.info()["path_name"] == "real_half"
    x = reals(prec, (7, n), n)
    for t in (2, 3):
        for norm in NORMS:
            assert row_err(dev_dct(p, x, t, norm), ref_dct(x, t, norm)) < TOL[prec], (t, norm)
            assert launches(p) == 2 + inner_launches(prec, n // 2, 7)


def test_real_half_on_the_persistent_two_pass_kernel():
    """f32 N = 2^21: the inner plan of length 2^20 is the persistent two-pass kernel"""
    n = 1 << 21
    p = plan("f32", n)
    assert p.info()["path_name"] == "real_half" and p.info()["inner_path_name"] == "twopass"
    assert "fused_twopass_kernel" in p.kernel_name()
    x = reals("f32", (2, n), 21)
    for t in (2, 3):
        assert row_err(dev_dct(p, x, t, "ortho"), ref_dct(x, t, "ortho")) < TOL["f32"], t


@pytest.mark.parametrize("prec", ("f32", "f64"))
@pytest.mark.parametrize("n", (1, 3, 97, 1009))
def test_real_full(prec, n):
    p = plan(prec, n)
    assert p.info()["path_name"] == "real_full"
    if n == 1009:
        assert p.info()["inner_path_name"] in ("bluestein", "bluestein_fused")
    x = reals(prec, (5, n), n)
    for t in (2, 3):
        for norm in NORMS:
            assert row_err(dev_dct(p, x, t, norm), ref_dct(x, t, norm)) < TOL[prec], (t, norm)
            assert launches(p) == 2 + inner_launches(prec, n, 5)


@pytest.mark.parametrize("prec,n", (("f32", 512), ("f64", 256), ("f32", 400), ("f64", 97), ("f32", 1)))
@pytest.mark.parametrize("t", (2, 3))
@pytest.mark.parametrize("norm", NORMS)
def test_idct_round_trip_and_ortho_norm(prec, n, t, norm):
    p = plan(prec, n)
    x = reals(prec, (6, n), 5 * n + t)
    y = dev_dct(p, x, t, norm)
    from scipy.fft import idct
    assert row_err(dev_dct(p, x, t, norm, inverse=True), idct(x.astype(np.float64), type=t, norm=norm)) < TOL[prec]
    back = dev_dct(p, y, t, norm, inverse=True)
    assert row_err(back, x) < 4 * TOL[prec]
    if norm == "ortho":
        ratio = np.linalg.norm(y.astype(np.float64), axis=-1) / np.linalg.norm(x.astype(np.float64), axis=-1)
        assert np.abs(ratio - 1).max() < 4 * TOL[prec]


@pytest.mark.parametrize("prec,n", (("f32", 2048), ("f64", 512), ("f32", 400), ("f64", 97)))
@pytest.mark.parametrize("t", (2, 3))
def test_in_place_rows_alone_and_host_memory_give_the_same_bits(prec, n, t):
    torch = torch_mod()
    p = plan(prec, n)
    base = reals(prec, (5, n), 3 * n + t)
    x = np.concatenate([base] * 9 + [base[:2]])   # a periodic batch of 47 rows
    got = dev_dct(p, x, t, "ortho")
    for r in range(5):
        assert np.array_equal(got[r::5], np.broadcast_to(dev_dct(p, base[r:r + 1], t, "ortho"), got[r::5].shape)), r
    xd = torch.from_numpy(x).cuda()
    p.dct(xd, xd, type=t, norm="ortho")
    torch.cuda.synchronize()
    assert np.array_equal(xd.cpu().numpy(), got)
    host = np.full_like(x, np.nan)
    p.dct(x, host, type=t, norm="ortho")
    assert np.array_equal(host, got)
    xh = x.copy()
    p.dct(xh, xh, type=t, norm="ortho")
    assert np.array_equal(xh, got)


def test_async_on_a_side_stream():
    torch = torch_mod()
    p = plan("f32", 1024)
    x = reals("f32", (100, 1024), 41)
    ref = dev_dct(p, x, 2, "backward")
    s = torch.cuda.Stream()
    xd = torch.from_numpy(x).cuda()
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        out = torch.full((100, 1024), float("nan"), dtype=torch.float32, device="cuda")
        p.dct(xd, out)
    s.synchronize()
    assert np.array_equal(out.cpu().numpy(), ref)


@pytest.mark.parametrize("prec,n,row_bytes", (("f32", 4096, 4096 * 4), ("f64", 1009, 1009 * 16)))
@pytest.mark.parametrize("t", (2, 3))
def test_two_scratch_chunks(prec, n, row_bytes, t):
    """a batch over two 512 MB scratch chunks (N reals per row at half length, N complex values at full length): the
    launch count of two chunks, and the rows on both sides of the cut"""
    chunk = (512 << 20) // row_bytes
    rows = chunk + 1000
    p = plan(prec, n)
    x = reals(prec, (rows, n), 77 + t)
    got = dev_dct(p, x, t, "forward")
    m = n // 2 if n % 2 == 0 else n
    assert launches(p) == (2 + inner_launches(prec, m, chunk)) + (2 + inner_launches(prec, m, rows - chunk))
    pick = [0, chunk - 1, chunk, rows - 1]
    assert row_err(got[pick], ref_dct(x[pick], t, "forward")) < TOL[prec]


def test_leading_shapes_and_batch_zero():
    torch = torch_mod()
    p = plan("f32", 256)
    x = reals("f32", (2, 3, 256), 61)
    got = dev_dct(p, x, 3, "ortho")
    assert got.shape == (2, 3, 256)
    assert np.array_equal(got.reshape(6, 256), dev_dct(p, x.reshape(6, 256), 3, "ortho"))
    out = torch.full((0, 256), float("nan"), device="cuda")
    p.dct(torch.empty((0, 256), device="cuda"), out)
    # the C entry point at batch 0 succeeds and launches nothing
    L = _lib.load()
    xd = torch.zeros(256, device="cuda")
    assert L.fourier_b200_dct_float(p._plan, xd.data_ptr(), xd.data_ptr(), 0, 2, 0) == 0
    assert launches(p) == 0


def test_refusals():
    torch = torch_mod()
    p = plan("f32", 512)
    x = torch.zeros(4, 512, device="cuda")
    out = torch.empty(4, 512, device="cuda")
    with pytest.raises(ValueError, match="last dimension"):
        p.dct(x, torch.empty(4, 256, device="cuda"))
    with pytest.raises(ValueError, match="shapes differ"):
        p.dct(x, torch.empty(3, 512, device="cuda"))
    with pytest.raises(TypeError, match="expected"):
        p.dct(x, out.double())
    with pytest.raises(ValueError, match="type"):
        p.dct(x, out, type=1)
    with pytest.raises(ValueError, match="norm"):
        p.idct(x, out, norm="none")
    with pytest.raises(ValueError, match="host or both be device"):
        p.dct(x, np.zeros((4, 512), np.float32))
    with pytest.raises(ValueError, match="conj"):
        p.dct(x._neg_view(), out)
    # the C entry points check a partial overlap, a mix of host and device memory and the alignment themselves
    L = _lib.load()
    flat = torch.zeros(5 * 512, device="cuda")
    rc = L.fourier_b200_dct_float(p._plan, flat.data_ptr(), flat.data_ptr() + 512 * 4, 4, 2, 0)
    assert rc == 1 and "overlap" in _lib.last_error()
    host = np.zeros((4, 512), np.float32)
    rc = L.fourier_b200_dct_float(p._plan, x.data_ptr(), host.ctypes.data, 4, 2, 0)
    assert rc == 1 and "host or both be device" in _lib.last_error()
    rc = L.fourier_b200_dct_async_float(p._plan, flat.data_ptr() + 4, flat.data_ptr() + 4, 4, 2, 0, None)
    assert rc == 716, rc
    assert "16-byte aligned" in _lib.last_error()

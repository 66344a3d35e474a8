"""Shared test helpers: the reference test-suite's comparison rule and input procedure, and the CPU emulators."""
import json
import os
import shutil
import subprocess

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


def golden_10pt():
    with open(os.path.join(HERE, "golden", "integrity_10pt.json")) as f:
        g = json.load(f)
    x = np.array([complex(a, b) for a, b in g["x"]], dtype=np.complex128)
    y = np.array([complex(a, b) for a, b in g["y"]], dtype=np.complex128)
    return x, y


def _ulp_diff(a, b):
    """|a-b| in units in the last place, float_cmp style (ordered-integer distance)."""
    if a.dtype == np.float32:
        ia, ib = a.view(np.int32).astype(np.int64), b.view(np.int32).astype(np.int64)
        ia = np.where(ia < 0, np.int64(-(2**31)) - ia, ia)
        ib = np.where(ib < 0, np.int64(-(2**31)) - ib, ib)
        return np.abs(ia - ib)
    ia, ib = a.view(np.int64), b.view(np.int64)
    fa = np.where(ia < 0, -(ia.astype(np.float64) + 2.0**63), ia.astype(np.float64))
    fb = np.where(ib < 0, -(ib.astype(np.float64) + 2.0**63), ib.astype(np.float64))
    return np.abs(fa - fb)


def assert_near_reference_rule(actual, expected):
    """fourier/tests/integrity.rs:89-143: per component approx_eq with epsilon 1e-4 | 8 ulps (f32),
    1e-11 | 8 ulps (f64)."""
    actual = np.ascontiguousarray(actual)
    expected = np.ascontiguousarray(expected).astype(actual.dtype)
    real = np.float32 if actual.dtype == np.complex64 else np.float64
    eps = 1e-4 if real == np.float32 else 1e-11
    a = actual.view(real)
    e = expected.view(real)
    ok = (np.abs(a.astype(np.float64) - e.astype(np.float64)) <= eps) | (_ulp_diff(a, e) <= 8)
    assert ok.all(), f"{(~ok).sum()} components differ beyond {eps}|8ulp; worst {np.abs(a - e).max()}"


def rel_err(got, ref):
    """North-star parity metric: max|got-ref| / max|ref| (SURVEY.md 8c)."""
    got = np.asarray(got).astype(np.complex128)
    ref = np.asarray(ref).astype(np.complex128)
    return float(np.abs(got - ref).max() / max(np.abs(ref).max(), 1e-300))


def sweep_input(max_size, dtype, forward, seed=0xDEADBEEF):
    """Procedure of integrity.rs:152-165: N(0, sigma) components, sigma = 1 forward, MAX_SIZE inverse.
    (The reference's RNG streams are ChaCha + thread_rng and half non-deterministic; the procedure is
    reproduced, not the bits.)"""
    rng = np.random.default_rng(seed)
    sigma = 1.0 if forward else float(max_size)
    z = rng.normal(0.0, sigma, max_size) + 1j * rng.normal(0.0, sigma, max_size)
    return z.astype(dtype)


def poisoned_like(x):
    """An output buffer like `x` (numpy array or torch tensor) filled with NaN, so that a sample the transform never
    stores cannot pass for a result left behind by an earlier call in a reused allocation."""
    if isinstance(x, np.ndarray):
        return np.full_like(x, np.nan)
    import torch
    return torch.full_like(x, complex(float("nan"), float("nan")))


def truth_ld(x, code):
    """Reference in long double: numpy's FFT on clongdouble (computed natively, not through f64), with the Transform
    scaling definitions applied in long double.  An input exact in f32 or f64 converts exactly, so for f64 data this
    is more precise than the kernels, which truth_f64 is not."""
    x = np.asarray(x).astype(np.clongdouble)
    if code in (0, 3):
        y = np.fft.fft(x, axis=-1)
    else:
        y = np.fft.ifft(x, axis=-1) * np.longdouble(x.shape[-1])
    assert y.dtype == np.clongdouble
    return scale_ld(y, code)


def scale_ld(y, code):
    """Applies the scale of Transform `code` in long double to the unscaled forward (codes 0, 3) or unscaled inverse
    (codes 1, 2, 4) transform `y`."""
    n = np.longdouble(y.shape[-1])
    if code == 1:
        return y / n
    if code in (3, 4):
        return y / np.sqrt(n)
    return y


def per_transform_err(got, ref):
    """max_k |got[b,k] - ref[b,k]| / max_k |ref[b,k]| for every transform b of a batch (last axis = transform), in the
    precision of `ref`: one bad transform cannot hide behind the others.  NaN (an unstored sample) counts as infinite."""
    got = np.asarray(got).reshape(-1, np.shape(ref)[-1])
    ref = np.asarray(ref).reshape(got.shape)
    err = np.empty(got.shape[0])
    rows = max(1, (1 << 20) // got.shape[1])   # bounds the long-double temporaries
    for b0 in range(0, got.shape[0], rows):
        g, r = got[b0:b0 + rows], ref[b0:b0 + rows]
        e = np.abs(g.astype(r.dtype) - r).max(axis=1) / np.maximum(np.abs(r).max(axis=1), 1e-300)
        err[b0:b0 + rows] = e
    return np.where(np.isnan(err), np.inf, err)


def truth_f64(x, code):
    """Independent reference: numpy pocketfft in f64, with the Transform scaling definitions
    (fourier-algorithms/src/fft.rs:5-16, autosort/mod.rs:381-385)."""
    x = np.asarray(x).astype(np.complex128)
    n = x.shape[-1]
    if code in (0, 3):
        y = np.fft.fft(x, axis=-1)
    else:
        y = np.fft.ifft(x, axis=-1) * n
    scale = {0: 1.0, 1: 1.0 / n, 2: 1.0, 3: 1.0 / np.sqrt(n), 4: 1.0 / np.sqrt(n)}[code]
    return y * scale


def run_emulator(name, tmp_dir):
    """Compiles tools/<name>.cu (host code only, nvcc; the test skips without it) into tmp_dir, runs it and returns the
    CompletedProcess, after printing its stdout."""
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    exe = os.path.join(str(tmp_dir), name)
    csrc = os.path.join(ROOT, "fourier_b200", "csrc")
    subprocess.run([nvcc, "-std=c++17", "-O1", "--expt-relaxed-constexpr", "-gencode", "arch=compute_90a,code=sm_90a",
                    "-I", csrc, os.path.join(ROOT, "tools", name + ".cu"), os.path.join(csrc, "host_math.cu"),
                    "-o", exe], check=True, capture_output=True)
    r = subprocess.run([exe], capture_output=True, text=True)
    print(r.stdout)
    return r

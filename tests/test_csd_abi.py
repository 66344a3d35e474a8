"""CPU-side checks of the cross-spectral density and coherence entry points: the eight fourier_b200_csd_* and
fourier_b200_coherence_* symbols are declared in fourier_b200.h, listed in _lib.EXTENSION_SYMBOLS and exported; the
refusals that need no plan return cudaErrorInvalidValue without a device, with a message naming the argument; and a C
program calling all eight with the header's macros compiles against the header with strict warnings."""
import ctypes
import math
import os
import re
import subprocess

import pytest

from fourier_b200 import _lib, build as fbuild

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INCLUDE = os.path.join(ROOT, "include")
LIBDIR = os.path.join(ROOT, "fourier_b200", "lib")

SYMBOLS = [f"fourier_b200_{fn}_{op}{t}" for fn in ("csd", "coherence") for t in ("float", "double")
           for op in ("", "async_")]


@pytest.fixture(scope="module")
def libfourier():
    fbuild.build()
    return _lib.load()


def test_symbols_declared_listed_and_exported(libfourier):
    header = open(os.path.join(INCLUDE, "fourier_b200.h")).read()
    declared = set(re.findall(r"\b(fourier_b200_(?:csd|coherence)_[a-z_0-9]+)\s*\(", header))
    assert set(SYMBOLS) == declared
    assert set(SYMBOLS) <= set(_lib.EXTENSION_SYMBOLS)
    out = subprocess.run(["nm", "-D", "--defined-only", _lib.LIB_PATH], capture_output=True, text=True, check=True)
    exported = {l.split()[-1] for l in out.stdout.splitlines() if " T " in l}
    assert set(SYMBOLS) <= exported


def _check(fn, good, cases, batch_args):
    for pos, value, word in cases:
        args = list(good)
        args[pos] = value
        for batch in (1, 0):
            assert fn(*args, *batch_args(batch)) == 1, (args, batch)
            assert word in _lib.last_error(), (args, batch, _lib.last_error())


def test_refusals_without_a_plan(libfourier):
    """NULL arguments, y_rows == 0, hop == 0, in_len == 0, detrend other than 0 and 1 and, for the csd, scaling other
    than 0 and 1 and fs zero, negative, infinite or NaN return cudaErrorInvalidValue (1) before the plan is touched, at
    batch 1 and batch 0; the fake plan pointer is never dereferenced on these paths."""
    buf = ctypes.create_string_buffer(256)
    fake = ctypes.cast(buf, ctypes.c_void_p)
    # (plan, x, y, y_rows, in_len, window, hop, detrend, ...)
    common = [(0, None, "null"), (1, None, "null"), (2, None, "null"), (5, None, "null"), (3, 0, "y_rows"),
              (6, 0, "hop"), (4, 0, "in_len"), (7, 2, "detrend"), (7, -1, "detrend")]
    for t in ("float", "double"):
        # csd: (..., detrend, scaling, fs, out)
        good = (fake, buf, buf, 1, 8, buf, 2, 1, 0, 1.0, buf)
        cases = common + [(10, None, "null"), (8, 2, "scaling"), (8, -1, "scaling"), (9, 0.0, "fs"), (9, -1.0, "fs"),
                          (9, math.inf, "fs"), (9, math.nan, "fs")]
        _check(getattr(libfourier, f"fourier_b200_csd_{t}"), good, cases, lambda b: (b,))
        _check(getattr(libfourier, f"fourier_b200_csd_async_{t}"), good, cases, lambda b: (b, None))
        # coherence: (..., detrend, out)
        good = (fake, buf, buf, 1, 8, buf, 2, 1, buf)
        cases = common + [(8, None, "null")]
        _check(getattr(libfourier, f"fourier_b200_coherence_{t}"), good, cases, lambda b: (b,))
        _check(getattr(libfourier, f"fourier_b200_coherence_async_{t}"), good, cases, lambda b: (b, None))


C_PROGRAM = r"""
#include <stdio.h>
#include "fourier_b200.h"

int main(void) {
  struct fourier_b200_rfft_float *pf = fourier_b200_rfft_create_float(512);
  struct fourier_b200_rfft_double *pd = fourier_b200_rfft_create_double(400);
  static float x[2 * 4096], y[4096], wf[512], of[2 * (512 / 2 + 1)], pf_out[2 * 2 * (512 / 2 + 1)];
  static double xd[4000], yd[4000], wd[400], od[400 / 2 + 1], pd_out[2 * (400 / 2 + 1)];
  int rc = 0;
  if (!pf || !pd) {
    printf("no device: %s\n", fourier_b200_last_error());
    fourier_b200_rfft_destroy_float(pf);
    fourier_b200_rfft_destroy_double(pd);
    return 0;
  }
  rc |= fourier_b200_csd_float(pf, x, y, 1, 4096, wf, 256, FOURIER_B200_DETREND_CONSTANT, FOURIER_B200_WELCH_DENSITY,
                               1.0, pf_out, 2);
  rc |= fourier_b200_csd_double(pd, xd, yd, 1, 4000, wd, 160, FOURIER_B200_DETREND_NONE, FOURIER_B200_WELCH_SPECTRUM,
                                16000.0, pd_out, 1);
  rc |= fourier_b200_csd_async_float(pf, x, y, 1, 4096, wf, 256, FOURIER_B200_DETREND_NONE,
                                     FOURIER_B200_WELCH_DENSITY, 2.5, pf_out, 0, NULL);
  rc |= fourier_b200_csd_async_double(pd, xd, yd, 1, 4000, wd, 160, FOURIER_B200_DETREND_CONSTANT,
                                      FOURIER_B200_WELCH_SPECTRUM, 1.0, pd_out, 0, NULL);
  rc |= fourier_b200_coherence_float(pf, x, x, 2, 4096, wf, 256, FOURIER_B200_DETREND_CONSTANT, of, 2);
  rc |= fourier_b200_coherence_double(pd, xd, yd, 1, 4000, wd, 160, FOURIER_B200_DETREND_NONE, od, 1);
  rc |= fourier_b200_coherence_async_float(pf, x, y, 1, 4096, wf, 256, FOURIER_B200_DETREND_NONE, of, 0, NULL);
  rc |= fourier_b200_coherence_async_double(pd, xd, yd, 1, 4000, wd, 160, FOURIER_B200_DETREND_CONSTANT, od, 0, NULL);
  printf("%d\n", rc);
  fourier_b200_rfft_destroy_float(pf);
  fourier_b200_rfft_destroy_double(pd);
  return 0;
}
"""


def test_c_program_compiles_against_the_header(tmp_path, libfourier):
    src = tmp_path / "csd_test.c"
    src.write_text(C_PROGRAM)
    exe = tmp_path / "csd_test"
    subprocess.run(["gcc", "-std=c11", "-Wall", "-Wextra", "-pedantic", "-Werror", "-I", INCLUDE, str(src), "-o", str(exe),
                    "-L", LIBDIR, "-lfourier", f"-Wl,-rpath,{LIBDIR}"], check=True, capture_output=True)
    assert exe.exists()

"""CPU-side checks of the Welch entry points: the four fourier_b200_welch_* symbols are declared in fourier_b200.h, listed
in _lib.EXTENSION_SYMBOLS and exported; the refusals that need no plan return cudaErrorInvalidValue without a device,
with a message naming the argument; and a C program calling all four with the header's macros compiles against the
header with strict warnings."""
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

WELCH_SYMBOLS = [f"fourier_b200_welch_{op}{t}" for t in ("float", "double") for op in ("", "async_")]


@pytest.fixture(scope="module")
def libfourier():
    fbuild.build()
    return _lib.load()


def test_welch_symbols_declared_listed_and_exported(libfourier):
    header = open(os.path.join(INCLUDE, "fourier_b200.h")).read()
    declared = set(re.findall(r"\b(fourier_b200_welch_[a-z_0-9]+)\s*\(", header))
    assert set(WELCH_SYMBOLS) == declared
    assert set(WELCH_SYMBOLS) <= set(_lib.EXTENSION_SYMBOLS)
    for macro in ("FOURIER_B200_DETREND_NONE 0", "FOURIER_B200_DETREND_CONSTANT 1", "FOURIER_B200_WELCH_DENSITY 0",
                  "FOURIER_B200_WELCH_SPECTRUM 1"):
        assert f"#define {macro}" in header
    out = subprocess.run(["nm", "-D", "--defined-only", _lib.LIB_PATH], capture_output=True, text=True, check=True)
    exported = {l.split()[-1] for l in out.stdout.splitlines() if " T " in l}
    assert set(WELCH_SYMBOLS) <= exported


def test_refusals_without_a_plan(libfourier):
    """NULL arguments, hop == 0, in_len == 0, detrend and scaling other than 0 and 1, and fs zero, negative, infinite or
    NaN return cudaErrorInvalidValue (1) before the plan is touched, at batch 1 and batch 0; the fake plan pointer is
    never dereferenced on these paths."""
    buf = ctypes.create_string_buffer(256)
    fake = ctypes.cast(buf, ctypes.c_void_p)
    # (plan, in, in_len, window, hop, detrend, scaling, fs, out)
    good = (fake, buf, 8, buf, 2, 1, 0, 1.0, buf)
    cases = [(0, None, "null"), (1, None, "null"), (3, None, "null"), (8, None, "null"), (4, 0, "hop"),
             (2, 0, "in_len"), (5, 2, "detrend"), (5, -1, "detrend"), (6, 2, "scaling"), (6, -1, "scaling"),
             (7, 0.0, "fs"), (7, -1.0, "fs"), (7, math.inf, "fs"), (7, math.nan, "fs")]
    for t in ("float", "double"):
        sync = getattr(libfourier, f"fourier_b200_welch_{t}")
        asyn = getattr(libfourier, f"fourier_b200_welch_async_{t}")
        for pos, value, word in cases:
            args = list(good)
            args[pos] = value
            for batch in (1, 0):
                assert sync(*args, batch) == 1, (t, args, batch)
                assert word in _lib.last_error(), (t, args, batch, _lib.last_error())
                assert asyn(*args, batch, None) == 1, (t, args, batch)
                assert word in _lib.last_error(), (t, args, batch, _lib.last_error())


C_PROGRAM = r"""
#include <stdio.h>
#include "fourier_b200.h"

int main(void) {
  struct fourier_b200_rfft_float *pf = fourier_b200_rfft_create_float(512);
  struct fourier_b200_rfft_double *pd = fourier_b200_rfft_create_double(400);
  static float x[2 * 4096], wf[512], yf[2 * (512 / 2 + 1)];
  static double xd[4000], wd[400], yd[400 / 2 + 1];
  struct fourier_b200_plan_info info;
  int rc = 0;
  if (!pf || !pd) {
    printf("no device: %s\n", fourier_b200_last_error());
    fourier_b200_rfft_destroy_float(pf);
    fourier_b200_rfft_destroy_double(pd);
    return 0;
  }
  rc |= fourier_b200_welch_float(pf, x, 4096, wf, 256, FOURIER_B200_DETREND_CONSTANT, FOURIER_B200_WELCH_DENSITY, 1.0,
                                 yf, 2);
  rc |= fourier_b200_welch_double(pd, xd, 4000, wd, 160, FOURIER_B200_DETREND_NONE, FOURIER_B200_WELCH_SPECTRUM, 16000.0,
                                  yd, 1);
  rc |= fourier_b200_welch_async_float(pf, x, 4096, wf, 256, FOURIER_B200_DETREND_NONE, FOURIER_B200_WELCH_DENSITY, 2.5,
                                       yf, 0, NULL);
  rc |= fourier_b200_welch_async_double(pd, xd, 4000, wd, 160, FOURIER_B200_DETREND_CONSTANT,
                                        FOURIER_B200_WELCH_SPECTRUM, 1.0, yd, 0, NULL);
  rc |= fourier_b200_rfft_info_float(pf, &info);
  printf("%d %s %llu\n", rc, fourier_b200_path_name(info.path), (unsigned long long)info.last_launches);
  fourier_b200_rfft_destroy_float(pf);
  fourier_b200_rfft_destroy_double(pd);
  return 0;
}
"""


def test_c_program_compiles_against_the_header(tmp_path, libfourier):
    src = tmp_path / "welch_test.c"
    src.write_text(C_PROGRAM)
    exe = tmp_path / "welch_test"
    subprocess.run(["gcc", "-std=c11", "-Wall", "-Wextra", "-pedantic", "-Werror", "-I", INCLUDE, str(src), "-o", str(exe),
                    "-L", LIBDIR, "-lfourier", f"-Wl,-rpath,{LIBDIR}"], check=True, capture_output=True)
    assert exe.exists()

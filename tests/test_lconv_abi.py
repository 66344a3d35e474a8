"""CPU-side checks of the linear convolution entry points: the four fourier_b200_linear_convolve_real_* symbols are
declared in fourier_b200.h, listed in _lib.EXTENSION_SYMBOLS and exported; the refusals that need no plan return
cudaErrorInvalidValue without a device; and a C program calling all four compiles against the header with strict
warnings."""
import ctypes
import os
import re
import subprocess

import pytest

from fourier_b200 import _lib, build as fbuild

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INCLUDE = os.path.join(ROOT, "include")
LIBDIR = os.path.join(ROOT, "fourier_b200", "lib")

LCONV_SYMBOLS = [f"fourier_b200_linear_convolve_real_{op}{t}" for t in ("float", "double") for op in ("", "async_")]


@pytest.fixture(scope="module")
def libfourier():
    fbuild.build()
    return _lib.load()


def test_lconv_symbols_declared_listed_and_exported(libfourier):
    header = open(os.path.join(INCLUDE, "fourier_b200.h")).read()
    declared = set(re.findall(r"\b(fourier_b200_linear_convolve_[a-z_0-9]+)\s*\(", header))
    assert set(LCONV_SYMBOLS) == declared
    assert set(LCONV_SYMBOLS) <= set(_lib.EXTENSION_SYMBOLS)
    out = subprocess.run(["nm", "-D", "--defined-only", _lib.LIB_PATH], capture_output=True, text=True, check=True)
    exported = {l.split()[-1] for l in out.stdout.splitlines() if " T " in l}
    assert set(LCONV_SYMBOLS) <= exported
    for name, value in (("FULL", 0), ("SAME", 1), ("VALID", 2)):
        assert re.search(rf"#define FOURIER_B200_LINEAR_{name} {value}\b", header), name


def test_refusals_without_a_plan(libfourier):
    """NULL arguments, spectrum_rows == 0, taps == 0, in_len == 0, an unknown mode and mode valid with in_len < taps
    return cudaErrorInvalidValue (1) before the plan is touched, batch 0 included; the fake plan pointer is never
    dereferenced on these paths."""
    buf = ctypes.create_string_buffer(256)
    fake = ctypes.cast(buf, ctypes.c_void_p)
    # (plan, in, in_len, spectrum, spectrum_rows, taps, mode, out, batch)
    cases = [((None, buf, 8, buf, 1, 3, 0, buf, 1), "null"), ((fake, None, 8, buf, 1, 3, 0, buf, 1), "null"),
             ((fake, buf, 8, None, 1, 3, 0, buf, 1), "null"), ((fake, buf, 8, buf, 1, 3, 0, None, 1), "null"),
             ((fake, buf, 8, buf, 0, 3, 0, buf, 1), "spectrum_rows"), ((fake, buf, 8, buf, 1, 0, 0, buf, 1), "taps"),
             ((fake, buf, 0, buf, 1, 3, 0, buf, 1), "in_len"), ((fake, buf, 8, buf, 1, 3, 3, buf, 1), "mode"),
             ((fake, buf, 8, buf, 1, 3, -1, buf, 1), "mode"), ((fake, buf, 2, buf, 1, 3, 2, buf, 1), "valid"),
             ((fake, buf, 8, buf, 1, 0, 0, buf, 0), "taps"), ((fake, buf, 2, buf, 1, 3, 2, buf, 0), "valid")]
    for t in ("float", "double"):
        sync = getattr(libfourier, f"fourier_b200_linear_convolve_real_{t}")
        asyn = getattr(libfourier, f"fourier_b200_linear_convolve_real_async_{t}")
        for args, word in cases:
            assert sync(*args) == 1, args
            assert word in _lib.last_error(), (args, _lib.last_error())
            assert asyn(*args, None) == 1, args
            assert word in _lib.last_error(), (args, _lib.last_error())


C_PROGRAM = r"""
#include <stdio.h>
#include "fourier_b200.h"

int main(void) {
  struct fourier_b200_rfft_float *pf = fourier_b200_rfft_create_float(2048);
  struct fourier_b200_rfft_double *pd = fourier_b200_rfft_create_double(1009);
  static float x[2 * 5000], y[2 * (5000 + 128)];
  static float spec[2 * (2048 / 2 + 1)];   /* one row of 1025 interleaved complex values */
  static double xd[3000], yd[3000], hd[2 * (1009 / 2 + 1)];
  struct fourier_b200_plan_info info;
  int rc = 0;
  if (!pf || !pd) {
    printf("no device: %s\n", fourier_b200_last_error());
    fourier_b200_rfft_destroy_float(pf);
    fourier_b200_rfft_destroy_double(pd);
    return 0;
  }
  rc |= fourier_b200_linear_convolve_real_float(pf, x, 5000, spec, 1, 129, FOURIER_B200_LINEAR_FULL, y, 2);
  rc |= fourier_b200_linear_convolve_real_double(pd, xd, 3000, hd, 1, 65, FOURIER_B200_LINEAR_SAME, yd, 1);
  rc |= fourier_b200_linear_convolve_real_async_float(pf, x, 5000, spec, 1, 129, FOURIER_B200_LINEAR_VALID, y, 0,
                                                      NULL);
  rc |= fourier_b200_linear_convolve_real_async_double(pd, xd, 3000, hd, 1, 65, FOURIER_B200_LINEAR_FULL, yd, 0, NULL);
  rc |= fourier_b200_rfft_info_float(pf, &info);
  printf("%d %s %llu\n", rc, fourier_b200_path_name(info.path), (unsigned long long)info.last_launches);
  fourier_b200_rfft_destroy_float(pf);
  fourier_b200_rfft_destroy_double(pd);
  return 0;
}
"""


def test_c_program_compiles_against_the_header(tmp_path, libfourier):
    src = tmp_path / "lconv_test.c"
    src.write_text(C_PROGRAM)
    exe = tmp_path / "lconv_test"
    subprocess.run(["gcc", "-std=c11", "-Wall", "-Wextra", "-pedantic", "-Werror", "-I", INCLUDE, str(src), "-o", str(exe),
                    "-L", LIBDIR, "-lfourier", f"-Wl,-rpath,{LIBDIR}"], check=True, capture_output=True)
    assert exe.exists()

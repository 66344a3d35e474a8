"""CPU-side checks of the convolution entry points: the four fourier_b200_convolve_real_* symbols are declared in
fourier_b200.h, listed in _lib.EXTENSION_SYMBOLS and exported, NULL arguments are refused without a device, and a C
program calling them compiles against the header with strict warnings."""
import ctypes
import os
import re
import subprocess

import pytest

from fourier_b200 import _lib, build as fbuild

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INCLUDE = os.path.join(ROOT, "include")
LIBDIR = os.path.join(ROOT, "fourier_b200", "lib")

CONV_SYMBOLS = [f"fourier_b200_convolve_real_{op}{t}" for t in ("float", "double") for op in ("", "async_")]


@pytest.fixture(scope="module")
def libfourier():
    fbuild.build()
    return _lib.load()


def test_conv_symbols_declared_listed_and_exported(libfourier):
    header = open(os.path.join(INCLUDE, "fourier_b200.h")).read()
    declared = set(re.findall(r"\b(fourier_b200_convolve_[a-z_0-9]+)\s*\(", header))
    assert set(CONV_SYMBOLS) == declared
    assert set(CONV_SYMBOLS) <= set(_lib.EXTENSION_SYMBOLS)
    out = subprocess.run(["nm", "-D", "--defined-only", _lib.LIB_PATH], capture_output=True, text=True, check=True)
    exported = {l.split()[-1] for l in out.stdout.splitlines() if " T " in l}
    assert set(CONV_SYMBOLS) <= exported


def test_null_arguments_are_refused(libfourier):
    """A NULL plan, input, spectrum or output, and spectrum_rows == 0, return cudaErrorInvalidValue (1) before any
    device work; a fake plan pointer is never dereferenced on these paths."""
    buf = ctypes.create_string_buffer(256)
    fake = ctypes.cast(buf, ctypes.c_void_p)
    for t in ("float", "double"):
        sync = getattr(libfourier, f"fourier_b200_convolve_real_{t}")
        asyn = getattr(libfourier, f"fourier_b200_convolve_real_async_{t}")
        cases = [((None, buf, buf, 1, buf, 1), "null"), ((fake, None, buf, 1, buf, 1), "null"),
                 ((fake, buf, None, 1, buf, 1), "null"), ((fake, buf, buf, 1, None, 1), "null"),
                 ((fake, buf, buf, 0, buf, 1), "spectrum_rows")]
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
  static float x[2 * 2048], y[2 * 2048];
  static float spec[2 * (2048 / 2 + 1)];   /* one row of 1025 interleaved complex values */
  static double xd[1009], hd[2 * (1009 / 2 + 1)];
  struct fourier_b200_plan_info info;
  int rc = 0;
  if (!pf || !pd) {
    printf("no device: %s\n", fourier_b200_last_error());
    fourier_b200_rfft_destroy_float(pf);
    fourier_b200_rfft_destroy_double(pd);
    return 0;
  }
  rc |= fourier_b200_convolve_real_float(pf, x, spec, 1, y, 2);
  rc |= fourier_b200_convolve_real_float(pf, x, spec, 1, x, 2);
  rc |= fourier_b200_convolve_real_double(pd, xd, hd, 1, xd, 1);
  rc |= fourier_b200_convolve_real_async_float(pf, x, spec, 1, y, 0, NULL);
  rc |= fourier_b200_convolve_real_async_double(pd, xd, hd, 1, xd, 0, NULL);
  rc |= fourier_b200_rfft_info_float(pf, &info);
  printf("%d %s %llu\n", rc, fourier_b200_path_name(info.path), (unsigned long long)info.last_launches);
  fourier_b200_rfft_destroy_float(pf);
  fourier_b200_rfft_destroy_double(pd);
  return 0;
}
"""


def test_c_program_compiles_against_the_header(tmp_path, libfourier):
    src = tmp_path / "conv_test.c"
    src.write_text(C_PROGRAM)
    exe = tmp_path / "conv_test"
    subprocess.run(["gcc", "-std=c11", "-Wall", "-Wextra", "-pedantic", "-Werror", "-I", INCLUDE, str(src), "-o", str(exe),
                    "-L", LIBDIR, "-lfourier", f"-Wl,-rpath,{LIBDIR}"], check=True, capture_output=True)
    assert exe.exists()

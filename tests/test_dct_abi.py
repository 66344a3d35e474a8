"""CPU-side checks of the DCT entry points: the four fourier_b200_dct_* symbols are declared in fourier_b200.h, listed in
_lib.EXTENSION_SYMBOLS and exported, with the three FOURIER_B200_DCT_NORM_* macros; the refusals that need no plan
return cudaErrorInvalidValue without a device, with a message naming the argument; and a C program calling all four
with the header's macros compiles against the header with strict warnings."""
import ctypes
import os
import re
import subprocess

import pytest

from fourier_b200 import _lib, build as fbuild

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INCLUDE = os.path.join(ROOT, "include")
LIBDIR = os.path.join(ROOT, "fourier_b200", "lib")

DCT_SYMBOLS = [f"fourier_b200_dct_{op}{t}" for t in ("float", "double") for op in ("", "async_")]


@pytest.fixture(scope="module")
def libfourier():
    fbuild.build()
    return _lib.load()


def test_dct_symbols_declared_listed_and_exported(libfourier):
    header = open(os.path.join(INCLUDE, "fourier_b200.h")).read()
    declared = set(re.findall(r"\b(fourier_b200_dct_[a-z_0-9]+)\s*\(", header))
    assert set(DCT_SYMBOLS) == declared
    assert set(DCT_SYMBOLS) <= set(_lib.EXTENSION_SYMBOLS)
    for macro in ("FOURIER_B200_DCT_NORM_BACKWARD 0", "FOURIER_B200_DCT_NORM_ORTHO 1", "FOURIER_B200_DCT_NORM_FORWARD 2"):
        assert f"#define {macro}" in header
    out = subprocess.run(["nm", "-D", "--defined-only", _lib.LIB_PATH], capture_output=True, text=True, check=True)
    exported = {l.split()[-1] for l in out.stdout.splitlines() if " T " in l}
    assert set(DCT_SYMBOLS) <= exported


def test_refusals_without_a_plan(libfourier):
    """NULL arguments, a type other than 2 and 3 and an unknown norm return cudaErrorInvalidValue (1) before the plan is
    touched, at batch 1 and batch 0; the fake plan pointer is never dereferenced on these paths."""
    buf = ctypes.create_string_buffer(256)
    fake = ctypes.cast(buf, ctypes.c_void_p)
    # (plan, in, out, batch, type, norm)
    good = (fake, buf, buf, 1, 2, 0)
    cases = [(0, None, "null"), (1, None, "null"), (2, None, "null"), (4, 1, "type"), (4, 4, "type"), (4, 0, "type"),
             (4, -2, "type"), (5, 3, "norm"), (5, -1, "norm")]
    for t in ("float", "double"):
        sync = getattr(libfourier, f"fourier_b200_dct_{t}")
        asyn = getattr(libfourier, f"fourier_b200_dct_async_{t}")
        for pos, value, word in cases:
            args = list(good)
            args[pos] = value
            for batch in (1, 0):
                args[3] = batch
                assert sync(*args) == 1, (t, args)
                assert word in _lib.last_error(), (t, args, _lib.last_error())
                assert asyn(*args, None) == 1, (t, args)
                assert word in _lib.last_error(), (t, args, _lib.last_error())


C_PROGRAM = r"""
#include <stdio.h>
#include "fourier_b200.h"

int main(void) {
  struct fourier_b200_rfft_float *pf = fourier_b200_rfft_create_float(512);
  struct fourier_b200_rfft_double *pd = fourier_b200_rfft_create_double(97);
  static float xf[2 * 512], yf[2 * 512];
  static double xd[3 * 97];
  struct fourier_b200_plan_info info;
  int rc = 0;
  if (!pf || !pd) {
    printf("no device: %s\n", fourier_b200_last_error());
    fourier_b200_rfft_destroy_float(pf);
    fourier_b200_rfft_destroy_double(pd);
    return 0;
  }
  rc |= fourier_b200_dct_float(pf, xf, yf, 2, 2, FOURIER_B200_DCT_NORM_ORTHO);
  rc |= fourier_b200_dct_double(pd, xd, xd, 3, 3, FOURIER_B200_DCT_NORM_BACKWARD);
  rc |= fourier_b200_dct_async_float(pf, xf, yf, 0, 3, FOURIER_B200_DCT_NORM_FORWARD, NULL);
  rc |= fourier_b200_dct_async_double(pd, xd, xd, 0, 2, FOURIER_B200_DCT_NORM_BACKWARD, NULL);
  rc |= fourier_b200_rfft_info_float(pf, &info);
  printf("%d %s %llu\n", rc, fourier_b200_path_name(info.path), (unsigned long long)info.last_launches);
  fourier_b200_rfft_destroy_float(pf);
  fourier_b200_rfft_destroy_double(pd);
  return 0;
}
"""


def test_c_program_compiles_against_the_header(tmp_path, libfourier):
    src = tmp_path / "dct_test.c"
    src.write_text(C_PROGRAM)
    exe = tmp_path / "dct_test"
    subprocess.run(["gcc", "-std=c11", "-Wall", "-Wextra", "-pedantic", "-Werror", "-I", INCLUDE, str(src), "-o", str(exe),
                    "-L", LIBDIR, "-lfourier", f"-Wl,-rpath,{LIBDIR}"], check=True, capture_output=True)
    assert exe.exists()

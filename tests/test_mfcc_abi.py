"""CPU-side checks of the MFCC entry points: the four fourier_b200_mfcc_* symbols are declared in fourier_b200.h, listed
in _lib.EXTENSION_SYMBOLS and exported; the refusals that need no plan return cudaErrorInvalidValue without a device,
with a message naming the argument, at batch 1 and batch 0; and a C program calling all four compiles against the header
with strict warnings."""
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

MFCC_SYMBOLS = [f"fourier_b200_mfcc_{op}{t}" for t in ("float", "double") for op in ("", "async_")]


@pytest.fixture(scope="module")
def libfourier():
    fbuild.build()
    return _lib.load()


def test_mfcc_symbols_declared_listed_and_exported(libfourier):
    header = open(os.path.join(INCLUDE, "fourier_b200.h")).read()
    declared = set(re.findall(r"\b(fourier_b200_mfcc_[a-z_0-9]+)\s*\(", header))
    assert set(MFCC_SYMBOLS) == declared
    assert set(MFCC_SYMBOLS) <= set(_lib.EXTENSION_SYMBOLS)
    out = subprocess.run(["nm", "-D", "--defined-only", _lib.LIB_PATH], capture_output=True, text=True, check=True)
    exported = {l.split()[-1] for l in out.stdout.splitlines() if " T " in l}
    assert set(MFCC_SYMBOLS) <= exported


# argument positions of (plan, in, in_len, window, hop, boundary, power, filters, n_mels, log_offset, log_floor,
# log_scale, top_db, top_db_rows, dct, n_out, bias, out)
IN, IN_LEN, WINDOW, HOP, BOUNDARY, POWER, FILTERS, N_MELS = 1, 2, 3, 4, 5, 6, 7, 8
OFFSET, FLOOR, SCALE, TOP_DB, ROWS, DCT, N_OUT, BIAS, OUT = 9, 10, 11, 12, 13, 14, 15, 16, 17


def test_refusals_without_a_plan(libfourier):
    """Every refusal that needs no plan returns cudaErrorInvalidValue (1) before the plan is touched, at batch 1 and
    batch 0 (a batch that is not a multiple of top_db_rows: at batch 1 only), with the argument named; the fake plan
    pointer is never dereferenced on these paths."""
    buf = ctypes.create_string_buffer(256)
    fake = ctypes.cast(buf, ctypes.c_void_p)
    good = [fake, buf, 8, buf, 2, 1, 2, buf, 4, 0.0, 1e-10, 10 / math.log(10), 80.0, 1, buf, 3, 0.0, buf]
    nan, inf = math.nan, math.inf
    cases = [(IN, None, "null"), (WINDOW, None, "null"), (FILTERS, None, "null"), (OUT, None, "null"),
             (0, None, "null"), (HOP, 0, "hop"), (BOUNDARY, 3, "boundary"), (BOUNDARY, -1, "boundary"),
             (IN_LEN, 0, "in_len"), (POWER, 0, "power"), (POWER, 3, "power"), (N_MELS, 0, "n_mels"),
             (N_OUT, 0, "n_out"), (OFFSET, nan, "log_offset"), (OFFSET, inf, "log_offset"), (BIAS, nan, "bias"),
             (BIAS, -inf, "bias"), (FLOOR, 0.0, "log_floor"), (FLOOR, -1.0, "log_floor"), (FLOOR, inf, "log_floor"),
             (FLOOR, nan, "log_floor"), (SCALE, 0.0, "log_scale"), (SCALE, -2.0, "log_scale"),
             (SCALE, inf, "log_scale"), (TOP_DB, nan, "top_db"), (TOP_DB, -1.0, "top_db"),
             (TOP_DB, -inf, "top_db"), (ROWS, 0, "top_db_rows")]
    identity = [(DCT, None), (N_OUT, 3)]   # dct NULL (the identity) with n_out != n_mels
    for t in ("float", "double"):
        sync = getattr(libfourier, f"fourier_b200_mfcc_{t}")
        asyn = getattr(libfourier, f"fourier_b200_mfcc_async_{t}")

        def refused(args, batch, word):
            assert sync(*args, batch) == 1, (t, args, batch)
            assert word in _lib.last_error(), (t, args, batch, _lib.last_error())
            assert asyn(*args, batch, None) == 1, (t, args, batch)
            assert word in _lib.last_error(), (t, args, batch, _lib.last_error())

        for pos, value, word in cases:
            args = list(good)
            args[pos] = value
            for batch in (1, 0):
                refused(args, batch, word)
        args = list(good)
        for pos, value in identity:
            args[pos] = value
        for batch in (1, 0):
            refused(args, batch, "n_out == n_mels")
        # with the clamp on, the batch must be whole groups; top_db = +inf turns the clamp off, and the same call
        # then gets past the checks to the plan (not exercised here: the plan is fake)
        args = list(good)
        args[ROWS] = 2
        for batch in (1, 3):
            refused(args, batch, "multiple of top_db_rows")


C_PROGRAM = r"""
#include <math.h>
#include <stdio.h>
#include "fourier_b200.h"

int main(void) {
  struct fourier_b200_rfft_float *pf = fourier_b200_rfft_create_float(512);
  struct fourier_b200_rfft_double *pd = fourier_b200_rfft_create_double(400);
  static float x[2 * 4096], wf[512], ff[80 * (512 / 2 + 1)], df[80 * 40], yf[2 * 33 * 40];
  static double xd[4000], wd[400], fd[80 * (400 / 2 + 1)], dd[80 * 13], yd[26 * 80];
  const double ten_ln10 = 10.0 / log(10.0);
  struct fourier_b200_plan_info info;
  int rc = 0;
  if (!pf || !pd) {
    printf("no device: %s\n", fourier_b200_last_error());
    fourier_b200_rfft_destroy_float(pf);
    fourier_b200_rfft_destroy_double(pd);
    return 0;
  }
  rc |= fourier_b200_mfcc_float(pf, x, 4096, wf, 128, FOURIER_B200_STFT_REFLECT, 2, ff, 80, 0.0, 1e-10, ten_ln10, 80.0,
                                1, df, 40, 0.0, yf, 2);
  rc |= fourier_b200_mfcc_double(pd, xd, 4000, wd, 160, FOURIER_B200_STFT_ZEROS, 2, fd, 80, 0.0, 1e-10,
                                 1.0 / (4.0 * log(10.0)), 2.0, 1, NULL, 80, 1.0, yd, 1);
  rc |= fourier_b200_mfcc_async_float(pf, x, 4096, wf, 128, FOURIER_B200_STFT_NONE, 1, ff, 80, 1e-6, 1.17549435e-38,
                                      1.0, HUGE_VAL, 1, df, 40, 0.0, yf, 0, NULL);
  rc |= fourier_b200_mfcc_async_double(pd, xd, 4000, wd, 160, FOURIER_B200_STFT_REFLECT, 2, fd, 80, 0.0, 1e-10,
                                       ten_ln10, 80.0, 1, dd, 13, 0.0, yd, 0, NULL);
  rc |= fourier_b200_rfft_info_float(pf, &info);
  printf("%d %s %llu\n", rc, fourier_b200_path_name(info.path), (unsigned long long)info.last_launches);
  fourier_b200_rfft_destroy_float(pf);
  fourier_b200_rfft_destroy_double(pd);
  return 0;
}
"""


def test_c_program_compiles_against_the_header(tmp_path, libfourier):
    src = tmp_path / "mfcc_test.c"
    src.write_text(C_PROGRAM)
    exe = tmp_path / "mfcc_test"
    subprocess.run(["gcc", "-std=c11", "-Wall", "-Wextra", "-pedantic", "-Werror", "-I", INCLUDE, str(src), "-o", str(exe),
                    "-L", LIBDIR, "-lfourier", f"-Wl,-rpath,{LIBDIR}", "-lm"], check=True, capture_output=True)
    assert exe.exists()

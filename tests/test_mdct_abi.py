"""CPU-side checks of the type-IV DCT, MDCT and IMDCT entry points: the twelve fourier_b200_dct4_* / mdct_* / imdct_*
symbols are declared in fourier_b200.h, listed in _lib.EXTENSION_SYMBOLS and exported; the refusals that need no plan
(a NULL argument, an unknown norm, in_len 0, frames 0, out_len 0) return cudaErrorInvalidValue without a device, at
batch 1 and batch 0, with a message naming the argument; and a C program calling all twelve with the header's norm
macros compiles against the header with strict warnings."""
import ctypes
import os
import re
import subprocess

import pytest

from fourier_b200 import _lib, build as fbuild

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INCLUDE = os.path.join(ROOT, "include")
LIBDIR = os.path.join(ROOT, "fourier_b200", "lib")

MDCT_SYMBOLS = [f"fourier_b200_{fn}_{op}{t}" for fn in ("dct4", "mdct", "imdct") for t in ("float", "double")
                for op in ("", "async_")]


@pytest.fixture(scope="module")
def libfourier():
    fbuild.build()
    return _lib.load()


def test_mdct_symbols_declared_listed_and_exported(libfourier):
    header = open(os.path.join(INCLUDE, "fourier_b200.h")).read()
    declared = set(re.findall(r"\b(fourier_b200_(?:dct4|mdct|imdct)_[a-z_0-9]+)\s*\(", header))
    assert len(MDCT_SYMBOLS) == 12
    assert set(MDCT_SYMBOLS) == declared
    assert set(MDCT_SYMBOLS) <= set(_lib.EXTENSION_SYMBOLS)
    out = subprocess.run(["nm", "-D", "--defined-only", _lib.LIB_PATH], capture_output=True, text=True, check=True)
    exported = {l.split()[-1] for l in out.stdout.splitlines() if " T " in l}
    assert set(MDCT_SYMBOLS) <= exported


def _refused(libfourier, fn, good, batch_pos, cases):
    for t in ("float", "double"):
        sync = getattr(libfourier, f"fourier_b200_{fn}_{t}")
        asyn = getattr(libfourier, f"fourier_b200_{fn}_async_{t}")
        for pos, value, word in cases:
            args = list(good)
            args[pos] = value
            for batch in (1, 0):
                args[batch_pos] = batch
                assert sync(*args) == 1, (fn, t, args)
                assert word in _lib.last_error(), (fn, t, args, _lib.last_error())
                assert asyn(*args, None) == 1, (fn, t, args)
                assert word in _lib.last_error(), (fn, t, args, _lib.last_error())


def test_refusals_without_a_plan(libfourier):
    """cudaErrorInvalidValue (1) before the plan is touched; the fake plan pointer is never dereferenced on these
    paths"""
    buf = ctypes.create_string_buffer(256)
    fake = ctypes.cast(buf, ctypes.c_void_p)
    norms = [(-1, "unknown norm"), (3, "unknown norm")]
    # dct4(plan, in, out, batch, norm)
    _refused(libfourier, "dct4", (fake, buf, buf, 1, 0), 3,
             [(0, None, "argument: plan"), (1, None, "argument: in"), (2, None, "argument: out")]
             + [(4, v, w) for v, w in norms])
    # mdct(plan, in, in_len, window, center, norm, out, batch)
    _refused(libfourier, "mdct", (fake, buf, 64, buf, 1, 0, buf, 1), 7,
             [(0, None, "argument: plan"), (1, None, "argument: in"), (3, None, "argument: window"),
              (6, None, "argument: out"), (2, 0, "in_len")] + [(5, v, w) for v, w in norms])
    # imdct(plan, in, frames, window, center, norm, out, out_len, batch)
    _refused(libfourier, "imdct", (fake, buf, 2, buf, 1, 0, buf, 64, 1), 8,
             [(0, None, "argument: plan"), (1, None, "argument: in"), (3, None, "argument: window"),
              (6, None, "argument: out"), (2, 0, "frames"), (7, 0, "out_len")] + [(5, v, w) for v, w in norms])


C_PROGRAM = r"""
#include <stdio.h>
#include "fourier_b200.h"

int main(void) {
  struct fourier_b200_rfft_float *pf = fourier_b200_rfft_create_float(1024);
  struct fourier_b200_rfft_double *pd = fourier_b200_rfft_create_double(96);
  static float xf[4 * 1024], wf[2 * 1024], Xf[5 * 1024], yf[4 * 1024];
  static double xd[5 * 96], wd[2 * 96], Xd[7 * 96], yd[5 * 96];
  struct fourier_b200_plan_info info;
  int rc = 0;
  if (!pf || !pd) {
    printf("no device: %s\n", fourier_b200_last_error());
    fourier_b200_rfft_destroy_float(pf);
    fourier_b200_rfft_destroy_double(pd);
    return 0;
  }
  rc |= fourier_b200_dct4_float(pf, xf, xf, 4, FOURIER_B200_DCT_NORM_ORTHO);
  rc |= fourier_b200_dct4_double(pd, xd, yd, 5, FOURIER_B200_DCT_NORM_BACKWARD);
  rc |= fourier_b200_dct4_async_float(pf, xf, yf, 0, FOURIER_B200_DCT_NORM_FORWARD, NULL);
  rc |= fourier_b200_dct4_async_double(pd, xd, yd, 0, FOURIER_B200_DCT_NORM_ORTHO, NULL);
  rc |= fourier_b200_mdct_float(pf, xf, 4 * 1024, wf, 1, FOURIER_B200_DCT_NORM_ORTHO, Xf, 1);
  rc |= fourier_b200_mdct_double(pd, xd, 5 * 96, wd, 1, FOURIER_B200_DCT_NORM_BACKWARD, Xd, 1);
  rc |= fourier_b200_mdct_async_float(pf, xf, 4 * 1024, wf, 1, FOURIER_B200_DCT_NORM_ORTHO, Xf, 0, NULL);
  rc |= fourier_b200_mdct_async_double(pd, xd, 5 * 96, wd, 0, FOURIER_B200_DCT_NORM_FORWARD, Xd, 0, NULL);
  rc |= fourier_b200_imdct_float(pf, Xf, 5, wf, 1, FOURIER_B200_DCT_NORM_ORTHO, yf, 4 * 1024, 1);
  rc |= fourier_b200_imdct_double(pd, Xd, 7, wd, 1, FOURIER_B200_DCT_NORM_BACKWARD, yd, 5 * 96, 1);
  rc |= fourier_b200_imdct_async_float(pf, Xf, 5, wf, 1, FOURIER_B200_DCT_NORM_ORTHO, yf, 4 * 1024, 0, NULL);
  rc |= fourier_b200_imdct_async_double(pd, Xd, 7, wd, 0, FOURIER_B200_DCT_NORM_FORWARD, yd, 5 * 96, 0, NULL);
  rc |= fourier_b200_rfft_info_float(pf, &info);
  printf("%d %s %llu\n", rc, fourier_b200_path_name(info.path), (unsigned long long)info.last_launches);
  fourier_b200_rfft_destroy_float(pf);
  fourier_b200_rfft_destroy_double(pd);
  return 0;
}
"""


def test_c_program_compiles_against_the_header(tmp_path, libfourier):
    src = tmp_path / "mdct_test.c"
    src.write_text(C_PROGRAM)
    exe = tmp_path / "mdct_test"
    subprocess.run(["gcc", "-std=c11", "-Wall", "-Wextra", "-pedantic", "-Werror", "-I", INCLUDE, str(src), "-o", str(exe),
                    "-L", LIBDIR, "-lfourier", f"-Wl,-rpath,{LIBDIR}"], check=True, capture_output=True)
    assert exe.exists()

"""CPU-side checks of the short-time Fourier transform entry points: the eight fourier_b200_stft_* / fourier_b200_istft_*
symbols are declared in fourier_b200.h, listed in _lib.EXTENSION_SYMBOLS and exported, with the three boundary macros;
the refusals that need no plan return cudaErrorInvalidValue without a device; and a C program calling all eight
compiles against the header with strict warnings."""
import ctypes
import os
import re
import subprocess

import pytest

from fourier_b200 import _lib, build as fbuild

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INCLUDE = os.path.join(ROOT, "include")
LIBDIR = os.path.join(ROOT, "fourier_b200", "lib")

STFT_SYMBOLS = [f"fourier_b200_{fn}_{op}{t}" for fn in ("stft", "istft") for t in ("float", "double")
                for op in ("", "async_")]


@pytest.fixture(scope="module")
def libfourier():
    fbuild.build()
    return _lib.load()


def test_stft_symbols_declared_listed_and_exported(libfourier):
    header = open(os.path.join(INCLUDE, "fourier_b200.h")).read()
    declared = set(re.findall(r"\b(fourier_b200_i?stft_[a-z_0-9]+)\s*\(", header))
    assert set(STFT_SYMBOLS) == declared
    assert set(STFT_SYMBOLS) <= set(_lib.EXTENSION_SYMBOLS)
    out = subprocess.run(["nm", "-D", "--defined-only", _lib.LIB_PATH], capture_output=True, text=True, check=True)
    exported = {l.split()[-1] for l in out.stdout.splitlines() if " T " in l}
    assert set(STFT_SYMBOLS) <= exported
    for name, value in (("NONE", 0), ("ZEROS", 1), ("REFLECT", 2)):
        assert re.search(rf"#define FOURIER_B200_STFT_{name} {value}\b", header), name


def test_refusals_without_a_plan(libfourier):
    """NULL arguments, hop == 0, an unknown boundary, in_len == 0, frames == 0 and out_len == 0 return
    cudaErrorInvalidValue (1) before the plan is touched, batch 0 included; the fake plan pointer is never dereferenced
    on these paths."""
    buf = ctypes.create_string_buffer(256)
    fake = ctypes.cast(buf, ctypes.c_void_p)
    # (plan, in, in_len, window, hop, boundary, out, batch)
    fwd = [((None, buf, 8, buf, 2, 1, buf, 1), "null"), ((fake, None, 8, buf, 2, 1, buf, 1), "null"),
           ((fake, buf, 8, None, 2, 1, buf, 1), "null"), ((fake, buf, 8, buf, 2, 1, None, 1), "null"),
           ((fake, buf, 8, buf, 0, 1, buf, 1), "hop"), ((fake, buf, 8, buf, 2, 3, buf, 1), "boundary"),
           ((fake, buf, 8, buf, 2, -1, buf, 1), "boundary"), ((fake, buf, 0, buf, 2, 1, buf, 1), "in_len"),
           ((fake, buf, 8, buf, 0, 1, buf, 0), "hop"), ((fake, buf, 0, buf, 2, 2, buf, 0), "in_len")]
    # (plan, in, frames, window, hop, center, out, out_len, batch)
    inv = [((None, buf, 4, buf, 2, 1, buf, 8, 1), "null"), ((fake, None, 4, buf, 2, 1, buf, 8, 1), "null"),
           ((fake, buf, 4, None, 2, 1, buf, 8, 1), "null"), ((fake, buf, 4, buf, 2, 1, None, 8, 1), "null"),
           ((fake, buf, 4, buf, 0, 1, buf, 8, 1), "hop"), ((fake, buf, 0, buf, 2, 1, buf, 8, 1), "frames"),
           ((fake, buf, 4, buf, 2, 1, buf, 0, 1), "out_len"), ((fake, buf, 0, buf, 2, 0, buf, 8, 0), "frames"),
           ((fake, buf, 4, buf, 2, 0, buf, 0, 0), "out_len")]
    for t in ("float", "double"):
        for fn, cases in (("stft", fwd), ("istft", inv)):
            sync = getattr(libfourier, f"fourier_b200_{fn}_{t}")
            asyn = getattr(libfourier, f"fourier_b200_{fn}_async_{t}")
            for args, word in cases:
                assert sync(*args) == 1, (fn, args)
                assert word in _lib.last_error(), (fn, args, _lib.last_error())
                assert asyn(*args, None) == 1, (fn, args)
                assert word in _lib.last_error(), (fn, args, _lib.last_error())


C_PROGRAM = r"""
#include <stdio.h>
#include "fourier_b200.h"

int main(void) {
  struct fourier_b200_rfft_float *pf = fourier_b200_rfft_create_float(512);
  struct fourier_b200_rfft_double *pd = fourier_b200_rfft_create_double(400);
  static float x[2 * 4096], wf[512], yf[2 * 4096];
  static float sf[2 * 2 * 33 * (512 / 2 + 1)];   /* 2 rows of 33 frames of 257 interleaved complex values */
  static double xd[4000], wd[400], yd[4000], sd[2 * 26 * (400 / 2 + 1)];
  struct fourier_b200_plan_info info;
  int rc = 0;
  if (!pf || !pd) {
    printf("no device: %s\n", fourier_b200_last_error());
    fourier_b200_rfft_destroy_float(pf);
    fourier_b200_rfft_destroy_double(pd);
    return 0;
  }
  rc |= fourier_b200_stft_float(pf, x, 4096, wf, 128, FOURIER_B200_STFT_REFLECT, sf, 2);
  rc |= fourier_b200_istft_float(pf, sf, 33, wf, 128, 1, yf, 4096, 2);
  rc |= fourier_b200_stft_double(pd, xd, 4000, wd, 160, FOURIER_B200_STFT_ZEROS, sd, 1);
  rc |= fourier_b200_istft_double(pd, sd, 26, wd, 160, 1, yd, 4000, 1);
  rc |= fourier_b200_stft_async_float(pf, x, 4096, wf, 128, FOURIER_B200_STFT_NONE, sf, 0, NULL);
  rc |= fourier_b200_istft_async_float(pf, sf, 29, wf, 128, 0, yf, 4096, 0, NULL);
  rc |= fourier_b200_stft_async_double(pd, xd, 4000, wd, 160, FOURIER_B200_STFT_REFLECT, sd, 0, NULL);
  rc |= fourier_b200_istft_async_double(pd, sd, 26, wd, 160, 1, yd, 4000, 0, NULL);
  rc |= fourier_b200_rfft_info_float(pf, &info);
  printf("%d %s %llu\n", rc, fourier_b200_path_name(info.path), (unsigned long long)info.last_launches);
  fourier_b200_rfft_destroy_float(pf);
  fourier_b200_rfft_destroy_double(pd);
  return 0;
}
"""


def test_c_program_compiles_against_the_header(tmp_path, libfourier):
    src = tmp_path / "stft_test.c"
    src.write_text(C_PROGRAM)
    exe = tmp_path / "stft_test"
    subprocess.run(["gcc", "-std=c11", "-Wall", "-Wextra", "-pedantic", "-Werror", "-I", INCLUDE, str(src), "-o", str(exe),
                    "-L", LIBDIR, "-lfourier", f"-Wl,-rpath,{LIBDIR}"], check=True, capture_output=True)
    assert exe.exists()

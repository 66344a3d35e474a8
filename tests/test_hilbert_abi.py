"""CPU-side checks of the analytic-signal entry points: the four fourier_b200_hilbert_* symbols are declared in
fourier_b200.h, listed in _lib.EXTENSION_SYMBOLS and exported, with the FOURIER_B200_HILBERT_ANALYTIC and _ENVELOPE
macros; the refusals that need no plan return cudaErrorInvalidValue without a device, with a message naming the
argument; and a C program calling all four with the header's macros compiles against the header with strict
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

HILBERT_SYMBOLS = [f"fourier_b200_hilbert_{op}{t}" for t in ("float", "double") for op in ("", "async_")]


@pytest.fixture(scope="module")
def libfourier():
    fbuild.build()
    return _lib.load()


def test_hilbert_symbols_declared_listed_and_exported(libfourier):
    header = open(os.path.join(INCLUDE, "fourier_b200.h")).read()
    declared = set(re.findall(r"\b(fourier_b200_hilbert_[a-z_0-9]+)\s*\(", header))
    assert set(HILBERT_SYMBOLS) == declared
    assert set(HILBERT_SYMBOLS) <= set(_lib.EXTENSION_SYMBOLS)
    for macro in ("FOURIER_B200_HILBERT_ANALYTIC 0", "FOURIER_B200_HILBERT_ENVELOPE 1"):
        assert f"#define {macro}" in header
    out = subprocess.run(["nm", "-D", "--defined-only", _lib.LIB_PATH], capture_output=True, text=True, check=True)
    exported = {l.split()[-1] for l in out.stdout.splitlines() if " T " in l}
    assert set(HILBERT_SYMBOLS) <= exported


def test_refusals_without_a_plan(libfourier):
    """NULL arguments and an unknown output return cudaErrorInvalidValue (1) before the plan is touched, at batch 1 and
    batch 0, with a message naming the argument; the fake plan pointer is never dereferenced on these paths."""
    buf = ctypes.create_string_buffer(256)
    fake = ctypes.cast(buf, ctypes.c_void_p)
    # (plan, in, out, batch, output)
    good = (fake, buf, buf, 1, 0)
    cases = [(0, None, "argument: plan"), (1, None, "argument: in"), (2, None, "argument: out"),
             (4, 2, "unknown output"), (4, -1, "unknown output"), (4, 7, "unknown output")]
    for t in ("float", "double"):
        sync = getattr(libfourier, f"fourier_b200_hilbert_{t}")
        asyn = getattr(libfourier, f"fourier_b200_hilbert_async_{t}")
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
  struct fourier_b200_rfft_float *pf = fourier_b200_rfft_create_float(2048);
  struct fourier_b200_rfft_double *pd = fourier_b200_rfft_create_double(97);
  static float xf[2 * 2048], zf[2 * 2 * 2048];
  static double xd[3 * 97];
  struct fourier_b200_plan_info info;
  int rc = 0;
  if (!pf || !pd) {
    printf("no device: %s\n", fourier_b200_last_error());
    fourier_b200_rfft_destroy_float(pf);
    fourier_b200_rfft_destroy_double(pd);
    return 0;
  }
  rc |= fourier_b200_hilbert_float(pf, xf, zf, 2, FOURIER_B200_HILBERT_ANALYTIC);
  rc |= fourier_b200_hilbert_double(pd, xd, xd, 3, FOURIER_B200_HILBERT_ENVELOPE);
  rc |= fourier_b200_hilbert_async_float(pf, xf, zf, 0, FOURIER_B200_HILBERT_ENVELOPE, NULL);
  rc |= fourier_b200_hilbert_async_double(pd, xd, xd, 0, FOURIER_B200_HILBERT_ANALYTIC, NULL);
  rc |= fourier_b200_rfft_info_float(pf, &info);
  printf("%d %s %llu\n", rc, fourier_b200_path_name(info.path), (unsigned long long)info.last_launches);
  fourier_b200_rfft_destroy_float(pf);
  fourier_b200_rfft_destroy_double(pd);
  return 0;
}
"""


def test_c_program_compiles_against_the_header(tmp_path, libfourier):
    src = tmp_path / "hilbert_test.c"
    src.write_text(C_PROGRAM)
    exe = tmp_path / "hilbert_test"
    subprocess.run(["gcc", "-std=c11", "-Wall", "-Wextra", "-pedantic", "-Werror", "-I", INCLUDE, str(src), "-o", str(exe),
                    "-L", LIBDIR, "-lfourier", f"-Wl,-rpath,{LIBDIR}"], check=True, capture_output=True)
    assert exe.exists()

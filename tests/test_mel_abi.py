"""CPU-side checks of the mel spectrogram entry points: the four fourier_b200_mel_spectrogram_* symbols are declared in
fourier_b200.h, listed in _lib.EXTENSION_SYMBOLS and exported; the refusals that need no plan return
cudaErrorInvalidValue without a device, with a message naming the argument; and a C program calling all four compiles
against the header with strict warnings."""
import ctypes
import os
import re
import subprocess

import pytest

from fourier_b200 import _lib, build as fbuild

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INCLUDE = os.path.join(ROOT, "include")
LIBDIR = os.path.join(ROOT, "fourier_b200", "lib")

MEL_SYMBOLS = [f"fourier_b200_mel_spectrogram_{op}{t}" for t in ("float", "double") for op in ("", "async_")]


@pytest.fixture(scope="module")
def libfourier():
    fbuild.build()
    return _lib.load()


def test_mel_symbols_declared_listed_and_exported(libfourier):
    header = open(os.path.join(INCLUDE, "fourier_b200.h")).read()
    declared = set(re.findall(r"\b(fourier_b200_mel_[a-z_0-9]+)\s*\(", header))
    assert set(MEL_SYMBOLS) == declared
    assert set(MEL_SYMBOLS) <= set(_lib.EXTENSION_SYMBOLS)
    out = subprocess.run(["nm", "-D", "--defined-only", _lib.LIB_PATH], capture_output=True, text=True, check=True)
    exported = {l.split()[-1] for l in out.stdout.splitlines() if " T " in l}
    assert set(MEL_SYMBOLS) <= exported


def test_refusals_without_a_plan(libfourier):
    """NULL arguments, hop == 0, an unknown boundary, in_len == 0, power 0 or 3 and n_mels == 0 return
    cudaErrorInvalidValue (1) before the plan is touched, at batch 1 and batch 0; the fake plan pointer is never
    dereferenced on these paths."""
    buf = ctypes.create_string_buffer(256)
    fake = ctypes.cast(buf, ctypes.c_void_p)
    # (plan, in, in_len, window, hop, boundary, power, filters, n_mels, out)
    good = (fake, buf, 8, buf, 2, 1, 2, buf, 4, buf)
    cases = [(0, None, "null"), (1, None, "null"), (3, None, "null"), (7, None, "null"), (9, None, "null"),
             (4, 0, "hop"), (5, 3, "boundary"), (5, -1, "boundary"), (2, 0, "in_len"), (6, 0, "power"),
             (6, 3, "power"), (8, 0, "n_mels")]
    for t in ("float", "double"):
        sync = getattr(libfourier, f"fourier_b200_mel_spectrogram_{t}")
        asyn = getattr(libfourier, f"fourier_b200_mel_spectrogram_async_{t}")
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
  static float x[2 * 4096], wf[512], ff[80 * (512 / 2 + 1)], yf[2 * 33 * 80];
  static double xd[4000], wd[400], fd[80 * (400 / 2 + 1)], yd[26 * 80];
  struct fourier_b200_plan_info info;
  int rc = 0;
  if (!pf || !pd) {
    printf("no device: %s\n", fourier_b200_last_error());
    fourier_b200_rfft_destroy_float(pf);
    fourier_b200_rfft_destroy_double(pd);
    return 0;
  }
  rc |= fourier_b200_mel_spectrogram_float(pf, x, 4096, wf, 128, FOURIER_B200_STFT_REFLECT, 2, ff, 80, yf, 2);
  rc |= fourier_b200_mel_spectrogram_double(pd, xd, 4000, wd, 160, FOURIER_B200_STFT_ZEROS, 1, fd, 80, yd, 1);
  rc |= fourier_b200_mel_spectrogram_async_float(pf, x, 4096, wf, 128, FOURIER_B200_STFT_NONE, 2, ff, 80, yf, 0, NULL);
  rc |= fourier_b200_mel_spectrogram_async_double(pd, xd, 4000, wd, 160, FOURIER_B200_STFT_REFLECT, 2, fd, 80, yd, 0,
                                                  NULL);
  rc |= fourier_b200_rfft_info_float(pf, &info);
  printf("%d %s %llu\n", rc, fourier_b200_path_name(info.path), (unsigned long long)info.last_launches);
  fourier_b200_rfft_destroy_float(pf);
  fourier_b200_rfft_destroy_double(pd);
  return 0;
}
"""


def test_c_program_compiles_against_the_header(tmp_path, libfourier):
    src = tmp_path / "mel_test.c"
    src.write_text(C_PROGRAM)
    exe = tmp_path / "mel_test"
    subprocess.run(["gcc", "-std=c11", "-Wall", "-Wextra", "-pedantic", "-Werror", "-I", INCLUDE, str(src), "-o", str(exe),
                    "-L", LIBDIR, "-lfourier", f"-Wl,-rpath,{LIBDIR}"], check=True, capture_output=True)
    assert exe.exists()

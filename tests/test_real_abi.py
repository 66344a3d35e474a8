"""CPU-side checks of the real-input transform API: every new symbol is declared in fourier_b200.h and exported,
create refuses without a device (no CPU fallback), and a C program using the API compiles against the header with
strict warnings."""
import os
import re
import subprocess

import pytest

from fourier_b200 import _lib, build as fbuild

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INCLUDE = os.path.join(ROOT, "include")
LIBDIR = os.path.join(ROOT, "fourier_b200", "lib")

RFFT_SYMBOLS = [f"fourier_b200_rfft_{op}_{t}" for t in ("float", "double")
                for op in ("create", "destroy", "forward", "forward_async", "inverse", "inverse_async", "info", "kernel")]


@pytest.fixture(scope="module")
def libfourier():
    fbuild.build()
    return _lib.load()


def test_rfft_symbols_declared_listed_and_exported(libfourier):
    header = open(os.path.join(INCLUDE, "fourier_b200.h")).read()
    declared = set(re.findall(r"\b(fourier_b200_rfft_[a-z_0-9]+)\s*\(", header))
    assert set(RFFT_SYMBOLS) == declared
    assert set(RFFT_SYMBOLS) <= set(_lib.EXTENSION_SYMBOLS)
    out = subprocess.run(["nm", "-D", "--defined-only", _lib.LIB_PATH], capture_output=True, text=True, check=True)
    exported = {l.split()[-1] for l in out.stdout.splitlines() if " T " in l}
    assert set(RFFT_SYMBOLS) <= exported


def test_path_names_of_real_plans(libfourier):
    names = [libfourier.fourier_b200_path_name(p).decode() for p in range(11)]
    assert names[8:] == ["real_fused", "real_half", "real_full"]
    assert names[:8] == ["trivial", "onchip", "twopass", "global_stages", "bluestein", "bluestein_fused", "onchip_cta",
                         "threepass"]


def test_rfft_create_without_a_gpu_returns_null(libfourier):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    import fourier_b200 as fb
    for t in ("float", "double"):
        assert not getattr(libfourier, f"fourier_b200_rfft_create_{t}")(2048)
        assert "no usable CUDA device" in _lib.last_error()
    with pytest.raises(RuntimeError, match="no usable CUDA device"):
        fb.create_rfft_f32(2048)


def test_rfft_null_plan_is_refused(libfourier):
    """Argument checks that need no device: a NULL plan, and destroy(NULL) as a no-op."""
    import ctypes
    buf = ctypes.create_string_buffer(64)
    for t in ("float", "double"):
        assert getattr(libfourier, f"fourier_b200_rfft_forward_{t}")(None, buf, buf, 1, 0) != 0
        assert "null" in _lib.last_error()
        assert getattr(libfourier, f"fourier_b200_rfft_inverse_async_{t}")(None, buf, buf, 1, 1, None) != 0
        getattr(libfourier, f"fourier_b200_rfft_destroy_{t}")(None)
        assert getattr(libfourier, f"fourier_b200_rfft_kernel_{t}")(None) == b""


C_PROGRAM = r"""
#include <stdio.h>
#include "fourier_b200.h"

int main(void) {
  struct fourier_b200_rfft_float *pf = fourier_b200_rfft_create_float(2048);
  struct fourier_b200_rfft_double *pd = fourier_b200_rfft_create_double(2018);
  float x[2 * 2048];
  float spec[2 * (2048 / 2 + 1) * 2];   /* two rows of 1025 interleaved complex values */
  struct fourier_b200_plan_info info;
  int rc = 0;
  if (!pf || !pd) {
    printf("no device: %s\n", fourier_b200_last_error());
    fourier_b200_rfft_destroy_float(pf);
    fourier_b200_rfft_destroy_double(pd);
    return 0;
  }
  rc |= fourier_b200_rfft_forward_float(pf, x, spec, 2, 0);
  rc |= fourier_b200_rfft_inverse_float(pf, spec, x, 2, 1);
  rc |= fourier_b200_rfft_forward_async_float(pf, x, spec, 0, 3, NULL);
  rc |= fourier_b200_rfft_inverse_async_double(pd, spec, NULL, 0, 4, NULL);
  rc |= fourier_b200_rfft_forward_double(pd, NULL, NULL, 0, 0);
  rc |= fourier_b200_rfft_inverse_double(pd, NULL, NULL, 0, 2);
  rc |= fourier_b200_rfft_forward_async_double(pd, NULL, NULL, 0, 0, NULL);
  rc |= fourier_b200_rfft_inverse_async_float(pf, NULL, NULL, 0, 1, NULL);
  rc |= fourier_b200_rfft_info_float(pf, &info);
  rc |= fourier_b200_rfft_info_double(pd, &info);
  printf("%s %s %d %s\n", fourier_b200_rfft_kernel_float(pf), fourier_b200_rfft_kernel_double(pd), rc,
         fourier_b200_path_name(info.path));
  fourier_b200_rfft_destroy_float(pf);
  fourier_b200_rfft_destroy_double(pd);
  return 0;
}
"""


def test_c_program_compiles_against_the_header(tmp_path, libfourier):
    src = tmp_path / "rfft_test.c"
    src.write_text(C_PROGRAM)
    exe = tmp_path / "rfft_test"
    subprocess.run(["gcc", "-std=c11", "-Wall", "-Wextra", "-pedantic", "-Werror", "-I", INCLUDE, str(src), "-o", str(exe),
                    "-L", LIBDIR, "-lfourier", f"-Wl,-rpath,{LIBDIR}"], check=True, capture_output=True)
    assert exe.exists()

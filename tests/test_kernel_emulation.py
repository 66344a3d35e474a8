"""Runs the fused kernels' device code (tilefft.cuh / twopass_kernels.cuh, all __host__ __device__) on
the CPU through tools/emulate.cu: every thread of every CTA, phase by phase, for each supported
two-pass configuration, against a double-precision FFT; also asserts the shared-memory exchange is
bank-conflict free.  This is the no-GPU check of index maps, twiddle tables and layouts."""
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.skipif(shutil.which("nvcc") is None and not os.path.exists("/usr/local/cuda/bin/nvcc"),
                    reason="nvcc not available")
def test_emulated_kernels_match_f64_fft(tmp_path):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    exe = tmp_path / "emulate"
    csrc = os.path.join(ROOT, "fourier_b200", "csrc")
    subprocess.run([nvcc, "-std=c++17", "-O1", "--expt-relaxed-constexpr", "-gencode",
                    "arch=compute_90a,code=sm_90a", "-I", csrc, os.path.join(ROOT, "tools", "emulate.cu"),
                    os.path.join(csrc, "host_math.cu"), "-o", str(exe)], check=True, capture_output=True)
    r = subprocess.run([str(exe)], capture_output=True, text=True)
    print(r.stdout)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "EMULATION OK" in r.stdout
    for line in r.stdout.splitlines():
        if "exchange conflicts" in line:
            assert "write x1, read x1" in line, line

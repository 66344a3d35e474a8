"""Runs the fused kernels' device code (tilefft.cuh / twopass_kernels.cuh, all __host__ __device__) on
the CPU through tools/emulate.cu: every thread of every CTA, phase by phase, for each supported
two-pass configuration, against a double-precision FFT; also asserts the shared-memory exchange is
bank-conflict free.  This is the no-GPU check of index maps, twiddle tables and layouts."""
from helpers import run_emulator


def test_emulated_kernels_match_f64_fft(tmp_path):
    r = run_emulator("emulate", tmp_path)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "EMULATION OK" in r.stdout
    for line in r.stdout.splitlines():
        if "exchange conflicts" in line:
            assert "write x1, read x1" in line, line

"""Runs the device code of the real-input transforms (real_kernels.cuh, RealBody in onchip_kernels.cuh) on the CPU
through tools/emulate_real.cu: the fused on-chip real kernel of every on-chip size class in both precisions, forward
and inverse, and the untangle / tangle steps for even and odd M = N/2, thread by thread against a double-precision
DFT.  The emulator records every spectrum access: none may be wider than one complex value or misaligned (f32
spectrum rows of odd index start 8 bytes off a 16-byte boundary)."""
import re

import pytest

from helpers import run_emulator


@pytest.fixture(scope="module")
def emulation(tmp_path_factory):
    return run_emulator("emulate_real", tmp_path_factory.mktemp("emulate_real"))


def test_emulated_real_kernels_match_f64_dft(emulation):
    assert emulation.returncode == 0, emulation.stdout + emulation.stderr
    assert "EMULATION OK" in emulation.stdout


def test_every_size_class_and_step_ran(emulation):
    out = emulation.stdout
    for n in (128, 256, 512, 1024, 2048):
        for d in ("forward", "inverse"):
            assert re.search(rf"fused f32 N={n} {d}: .* OK", out), (n, d)
    for n in (128, 256, 512):
        for d in ("forward", "inverse"):
            assert re.search(rf"fused f64 N={n} {d}: .* OK", out), (n, d)
    for p in ("f32", "f64"):
        for m in (512, 1000, 1009):   # even and odd M
            for step in ("untangle", "tangle"):
                assert re.search(rf"steps {p} {step} N={2 * m} \(M={m}\): .* OK", out), (p, step, m)


def test_park_and_reversed_read_are_conflict_free(emulation):
    lines = [l for l in emulation.stdout.splitlines() if "exchange conflicts" in l]
    assert len(lines) == 8
    for line in lines:
        assert "write x1, read x1" in line, line


def test_spectrum_accessed_one_complex_value_at_a_time(emulation):
    """f32: no access wider than 8 bytes, none misaligned, and odd rows (8 bytes off 16) were really touched."""
    current = None
    checked = 0
    for line in emulation.stdout.splitlines():
        m = re.match(r"(fused|steps) (f32|f64)", line)
        if m:
            current = m.group(2)
        if "spectrum accesses" in line:
            m = re.search(r"accesses: (\d+) \((\d+) at odd rows\), widest (\d+) B, misaligned (\d+), outside (\d+)", line)
            assert m, line
            total, odd, widest, misaligned, outside = map(int, m.groups())
            assert total > 0 and odd > 0 and misaligned == 0 and outside == 0, line
            assert widest == (8 if current == "f32" else 16), line
            checked += 1
    assert checked == 2 * 8 + 2 * 2 * 6

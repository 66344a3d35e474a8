"""Runs the device code of the convolution of real rows (real::conv_pair in real_kernels.cuh, ConvBody in
onchip_kernels.cuh) on the CPU through tools/emulate_conv.cu: the fused on-chip conv kernel of every on-chip size class
in both precisions with three spectrum rows, and the pair step alone for even and odd M = N/2, thread by thread against
a direct circular convolution in double.  The emulator records every read of H: none may be wider than one complex
value or misaligned, and f32 rows of odd index (8 bytes off a 16-byte boundary) must really be read."""
import re

import pytest

from helpers import run_emulator


@pytest.fixture(scope="module")
def emulation(tmp_path_factory):
    return run_emulator("emulate_conv", tmp_path_factory.mktemp("emulate_conv"))


def test_emulated_conv_matches_direct_convolution(emulation):
    assert emulation.returncode == 0, emulation.stdout + emulation.stderr
    assert "EMULATION OK" in emulation.stdout


def test_every_size_class_batch_and_pair_ran(emulation):
    out = emulation.stdout
    sizes = {"f32": (128, 256, 512, 1024, 2048), "f64": (128, 256, 512)}
    for p, ns in sizes.items():
        for n in ns:
            runs = re.findall(rf"fused {p} N={n} F=3 batch=(\d+) row0=(\d+): .* OK", out)
            batches = {int(b) for b, _ in runs}
            assert 5 in batches and len(batches) == 2, (p, n, runs)
            assert {int(r) for _, r in runs} == {0, 2}, (p, n, runs)
    for p in ("f32", "f64"):
        for m in (512, 1000, 1009):   # even and odd M
            assert re.search(rf"pair {p} conv_pair N={2 * m} \(M={m}\): .* OK", out), (p, m)


def test_write_back_and_stage_a_reads_are_conflict_free(emulation):
    lines = [l for l in emulation.stdout.splitlines() if "exchange conflicts" in l]
    assert len(lines) == 8
    for line in lines:
        assert "write-back x1, stage-A read x1" in line, line


def test_spectrum_read_one_complex_value_at_a_time(emulation):
    """f32: no access wider than 8 bytes, none misaligned, and odd rows (8 bytes off 16) were really read."""
    current = None
    checked = 0
    for line in emulation.stdout.splitlines():
        m = re.match(r"(fused|pair) (f32|f64)", line)
        if m:
            current = m.group(2)
        if "H accesses" in line:
            m = re.search(r"accesses: (\d+) \((\d+) at odd rows\), widest (\d+) B, misaligned (\d+), outside (\d+)", line)
            assert m, line
            total, odd, widest, misaligned, outside = map(int, m.groups())
            assert total > 0 and odd > 0 and misaligned == 0 and outside == 0, line
            assert widest == (8 if current == "f32" else 16), line
            checked += 1
    assert checked == 8 * 4 + 2 * 6

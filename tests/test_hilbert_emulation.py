"""Runs the device code of the analytic signal and envelope (HilbertBody in onchip_kernels.cuh and the real::hilbert*
steps of real_kernels.cuh) on the CPU through tools/emulate_hilbert.cu: the fused body of every on-chip size class in
both precisions with both outputs, on a batch that leaves a partial group, against a direct DFT -> G -> inverse DFT in
double; the analytic signal's real part equal to the input bit for bit, the envelope in place equal to the envelope out
of place bit for bit; every input read in its row and every output written once.  Also the element steps of the other
paths for N = 1, 2, 96 and 97 over two chunks of rows, and the bank conflicts of the new pair phase."""
import re

import pytest

from helpers import run_emulator

FUSED = re.compile(r"^fused (f32|f64) output=(analytic|envelope) N=(\d+) batch=(\d+): max rel err (\S+), "
                   r"outside row (\d+), not once (\d+), (real part|in place) (\w+) (OK|FAIL)$")
ELEMENTS = re.compile(r"^elements (f32|f64) (half|full) N=(\d+) output=(analytic|envelope) chunks=2: max rel err (\S+), "
                      r"real part (exact|inexact) (OK|FAIL)$")
CONFLICTS = re.compile(r"(f32|f64) L=(\d+) threads \d+ conflicts: pairs Z\[k\] x(\d+), Z\[L-k\] x(\d+)$")

# the on-chip size classes (onchip_configs.cuh) as N = 2L, and their FFTs per CTA (C)
SIZES = {"f32": {128: 32, 256: 32, 512: 16, 1024: 16, 2048: 8}, "f64": {128: 32, 256: 32, 512: 16}}


@pytest.fixture(scope="module")
def emulation(tmp_path_factory):
    return run_emulator("emulate_hilbert", tmp_path_factory.mktemp("emulate_hilbert"))


def _match(emulation, pattern):
    return [m.groups() for m in map(pattern.match, emulation.stdout.splitlines()) if m]


def test_emulated_hilbert_matches_direct_sums(emulation):
    assert emulation.returncode == 0, emulation.stdout + emulation.stderr
    assert "EMULATION OK" in emulation.stdout


def test_every_size_class_and_output_ran(emulation):
    runs = _match(emulation, FUSED)
    want = {(p, o, n) for p, classes in SIZES.items() for n in classes for o in ("analytic", "envelope")}
    assert {(r[0], r[1], int(r[2])) for r in runs} == want
    for r in runs:
        c = SIZES[r[0]][int(r[2])]
        assert int(r[3]) % c != 0 and int(r[3]) > c, r   # a full group and a partial one
        assert float(r[4]) < (1e-5 if r[0] == "f32" else 1e-12), r
        exact = ("real part", "exact") if r[1] == "analytic" else ("in place", "same")
        assert r[5:] == ("0", "0") + exact + ("OK",), r


def test_other_paths_elements(emulation):
    elements = _match(emulation, ELEMENTS)
    assert {(r[0], int(r[2]), r[3]) for r in elements} == {
        (p, n, o) for p in ("f32", "f64") for n in (1, 2, 96, 97) for o in ("analytic", "envelope")}
    for r in elements:
        assert r[1] == ("full" if int(r[2]) % 2 else "half"), r
        assert float(r[4]) < (1e-5 if r[0] == "f32" else 1e-12) and r[5:] == ("exact", "OK"), r


def test_shared_memory_conflicts_reported(emulation):
    """The pair phase reads and writes the park without bank conflicts (DESIGN.md §4.19)."""
    lines = [m.groups() for m in map(CONFLICTS.search, emulation.stdout.splitlines()) if m]
    assert {(p, 2 * int(l)) for p, l, *_ in lines} == {(p, n) for p, c in SIZES.items() for n in c}
    for line in lines:
        assert all(int(d) == 1 for d in line[2:]), line

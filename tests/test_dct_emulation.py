"""Runs the device code of the discrete cosine transforms (Dct2Body / Dct3Body in onchip_kernels.cuh and the real::dct*
steps of real_kernels.cuh) on the CPU through tools/emulate_dct.cu: both fused bodies of every on-chip size class in
both precisions, all three norms, a batch that leaves a partial group, and in place against out of place, against a
direct O(N^2) DCT in double; every input read must lie in its row and every output be written once.  Also the element
steps of the other paths for N = 1, 2, 96 and 97 over two chunks of rows, and the bank conflicts of the new phases."""
import re

import pytest

from helpers import run_emulator

FUSED = re.compile(r"^fused (f32|f64) type=([23]) N=(\d+) batch=(\d+) norm=(backward|ortho|forward): max rel err (\S+), "
                   r"outside row (\d+), not once (\d+), in place (same|differs) (OK|FAIL)$")
ELEMENTS = re.compile(r"^elements (f32|f64) (half|full) N=(\d+) type=([23]) norm=(\w+) chunks=2: max rel err (\S+) "
                      r"(OK|FAIL)$")
CONFLICTS = re.compile(r"(f32|f64) L=(\d+) threads \d+ conflicts: type 2 load x(\d+), pairs read x(\d+), park x(\d+), "
                       r"store x(\d+); type 3 load x(\d+), pairs read x(\d+), park x(\d+), store x(\d+)$")

# the on-chip size classes (onchip_configs.cuh) as N = 2L, and their FFTs per CTA (C)
SIZES = {"f32": {128: 32, 256: 32, 512: 16, 1024: 16, 2048: 8}, "f64": {128: 32, 256: 32, 512: 16}}


@pytest.fixture(scope="module")
def emulation(tmp_path_factory):
    return run_emulator("emulate_dct", tmp_path_factory.mktemp("emulate_dct"))


def _match(emulation, pattern):
    return [m.groups() for m in map(pattern.match, emulation.stdout.splitlines()) if m]


def test_emulated_dct_matches_direct_sums(emulation):
    assert emulation.returncode == 0, emulation.stdout + emulation.stderr
    assert "EMULATION OK" in emulation.stdout


def test_every_size_class_type_and_norm_ran(emulation):
    runs = _match(emulation, FUSED)
    want = {(p, t, n, nm) for p, classes in SIZES.items() for n in classes for t in ("2", "3")
            for nm in ("backward", "ortho", "forward")}
    assert {(r[0], r[1], int(r[2]), r[4]) for r in runs} == want
    for r in runs:
        c = SIZES[r[0]][int(r[2])]
        assert int(r[3]) % c != 0 and int(r[3]) > c, r   # a full group and a partial one
        assert float(r[5]) < (1e-5 if r[0] == "f32" else 1e-12), r
        assert r[6:] == ("0", "0", "same", "OK"), r


def test_other_paths_elements(emulation):
    elements = _match(emulation, ELEMENTS)
    assert {(r[0], int(r[2]), r[3], r[4]) for r in elements} == {
        (p, n, t, nm) for p in ("f32", "f64") for n in (1, 2, 96, 97) for t in ("2", "3")
        for nm in ("backward", "ortho", "forward")}
    for r in elements:
        assert r[1] == ("full" if int(r[2]) % 2 else "half"), r
        assert float(r[5]) < (1e-5 if r[0] == "f32" else 1e-12) and r[6] == "OK", r


def test_shared_memory_conflicts_reported(emulation):
    """The new load, pair, park and store phases are at most two-way conflicted (DESIGN.md §4.16)."""
    lines = [m.groups() for m in map(CONFLICTS.search, emulation.stdout.splitlines()) if m]
    assert {(p, 2 * int(l)) for p, l, *_ in lines} == {(p, n) for p, c in SIZES.items() for n in c}
    for line in lines:
        assert all(1 <= int(d) <= 2 for d in line[2:]), line

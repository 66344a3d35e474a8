"""Runs the device code of the cross-spectral density and coherence (CsdBody in onchip_kernels.cuh through the CPU driver
that keeps the kernel's barriers between warps; real::WelchItems, spec_pair, cross_terms, csd_out, coherence_out,
cross_accumulate_one, csd_finish_one and coherence_finish_one in real_kernels.cuh) on the CPU through
tools/emulate_csd.cu: the fused kernel and the finish of both outputs for every on-chip size class in both precisions,
both detrends, the csd's two scalings, hops 1, N/4, N and N+3, rows of F = 1, F < C/2, B-1, B, B+1 and 2B+3 frames,
y_rows 1 and y_rows = batch, against a direct windowed DFT in double; and the other paths' accumulate and finish
elements over two chunks of frames for N = 96 and 97.  Every x and y read and every partial and output write is
checked."""
import re

import pytest

from helpers import run_emulator

FUSED = re.compile(r"^fused (csd|coherence) (f32|f64) N=(\d+) H=(\d+) L=(\d+) batch=(\d+) y_rows=(\d+) F=(\d+) B=(\d+) "
                   r"items=(\d+) per_group=(\d+) detrend=(none|constant) scaling=(density|spectrum|none)( partial)?: "
                   r"max (rel|abs) err (\S+), outside row (\d+), not once (\d+), im edges (\S+) (OK|FAIL)$")
ELEMENTS = re.compile(r"^elements (csd|coherence) N=(\d+) F=7 B=(\d+) items=2 chunks=2: max err (\S+) (OK|FAIL)$")
CONFLICTS = re.compile(r"(csd|coherence) threads +\d+  conflicts: park read x(\d+); accumulate x(\d+); flush read x(\d+)$")

# the on-chip size classes (onchip_configs.cuh) as N = 2L, and their FFTs per CTA (C); a round runs C/2 frame pairs
SIZES = {"f32": {128: 32, 256: 32, 512: 16, 1024: 16, 2048: 8}, "f64": {128: 32, 256: 32, 512: 16}}
TOL = {("csd", "f32"): 1e-5, ("csd", "f64"): 1e-12, ("coherence", "f32"): 5e-5, ("coherence", "f64"): 1e-12}


@pytest.fixture(scope="module")
def emulation(tmp_path_factory):
    return run_emulator("emulate_csd", tmp_path_factory.mktemp("emulate_csd"))


def _match(emulation, pattern):
    return [m.groups() for m in map(pattern.match, emulation.stdout.splitlines()) if m]


def test_emulated_csd_and_coherence_match_direct_sums(emulation):
    assert emulation.returncode == 0, emulation.stdout + emulation.stderr
    assert "EMULATION OK" in emulation.stdout


def test_every_size_class_hop_row_length_and_argument_ran(emulation):
    runs = _match(emulation, FUSED)
    for kind in ("csd", "coherence"):
        for p, classes in SIZES.items():
            for n, c in classes.items():
                mine = [r for r in runs if r[0] == kind and r[1] == p and int(r[2]) == n]
                assert {int(r[3]) for r in mine} == {1, n // 4, n, n + 3}, (kind, p, n)
                b = 4 * (c // 2)   # real::welch_block over C/2 pair columns
                assert {int(r[7]) for r in mine if int(r[3]) == n // 4} == {1, c // 4 + 1, b - 1, b, b + 1, 2 * b + 3}
                assert {r[11] for r in mine} == {"none", "constant"}, (kind, p, n)
                if kind == "csd":
                    assert {r[12] for r in mine} == {"density", "spectrum"}, (kind, p, n)
                assert any(r[6] == "1" for r in mine) and any(int(r[6]) == int(r[5]) > 1 for r in mine)
                assert any(int(r[9]) > 1 for r in mine) and any(r[13] for r in mine), (kind, p, n)
    for r in runs:
        assert r[16:] == ("0", "0", "+0", "OK"), r
        assert float(r[15]) < TOL[(r[0], r[1])], r


def test_other_paths_elements(emulation):
    elements = _match(emulation, ELEMENTS)
    assert {(r[0], int(r[1])) for r in elements} == {(k, n) for k in ("csd", "coherence") for n in (96, 97)}
    for r in elements:
        assert float(r[3]) < 1e-12 and r[4] == "OK", r


def test_shared_memory_conflicts_reported(emulation):
    lines = [m.groups() for m in map(CONFLICTS.search, emulation.stdout.splitlines()) if m]
    assert len(lines) == 2 * sum(len(v) for v in SIZES.values())
    for _, park, acc, flush in lines:
        assert int(park) >= 1 and int(acc) >= 1 and int(flush) >= 1

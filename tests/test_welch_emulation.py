"""Runs the device code of the Welch power spectral density (WelchBody in onchip_kernels.cuh through its CPU driver;
real::WelchItems, welch_out, welch_accumulate_one and welch_finish_one in real_kernels.cuh) on the CPU through
tools/emulate_welch.cu: the fused kernel and the finish of every on-chip size class in both precisions, detrend none and
constant, both scalings with fs = 1 and 2.5, hops 1, N/4, N/2, N and N+3 and rows of F = 1, F < C, B-1, B, B+1 and 2B+3
frames, against a direct windowed DFT in double; and the other paths' accumulate and finish elements over two chunks of
frames for N = 96 and 97.  Every input read and every partial and output write is checked."""
import re

import pytest

from helpers import run_emulator

FUSED = re.compile(r"^fused (f32|f64) N=(\d+) H=(\d+) L=(\d+) batch=(\d+) F=(\d+) B=(\d+) items=(\d+) per_group=(\d+) "
                   r"detrend=(none|constant) scaling=(density|spectrum) fs=(\S+?)( partial)?: max rel err (\S+), "
                   r"outside row (\d+), not once (\d+) (OK|FAIL)$")
ELEMENTS = re.compile(r"^elements N=(\d+) F=7 B=(\d+) items=2 chunks=2: max rel err (\S+) (OK|FAIL)$")
CONFLICTS = re.compile(r"park write x(\d+), stage-A read x(\d+); accumulate x(\d+); flush read x(\d+)$")

# the on-chip size classes (onchip_configs.cuh) as N = 2L, and their FFTs per CTA (C)
SIZES = {"f32": {128: 32, 256: 32, 512: 16, 1024: 16, 2048: 8}, "f64": {128: 32, 256: 32, 512: 16}}


@pytest.fixture(scope="module")
def emulation(tmp_path_factory):
    return run_emulator("emulate_welch", tmp_path_factory.mktemp("emulate_welch"))


def _match(emulation, pattern):
    return [m.groups() for m in map(pattern.match, emulation.stdout.splitlines()) if m]


def test_emulated_welch_matches_direct_sums(emulation):
    assert emulation.returncode == 0, emulation.stdout + emulation.stderr
    assert "EMULATION OK" in emulation.stdout


def test_every_size_class_hop_row_length_and_argument_ran(emulation):
    runs = _match(emulation, FUSED)
    for p, classes in SIZES.items():
        for n, c in classes.items():
            mine = [r for r in runs if r[0] == p and int(r[1]) == n]
            assert {int(r[2]) for r in mine} == {1, n // 4, n // 2, n, n + 3}, (p, n)
            b = 4 * c   # real::welch_block for rows of more than C and at most 1024 C frames
            assert {int(r[5]) for r in mine if int(r[2]) == n // 4} == {1, c // 2 + 1, b - 1, b, b + 1, 2 * b + 3}, (p, n)
            assert {(r[9], r[10], float(r[11])) for r in mine} == {
                (d, s, fs) for d in ("none", "constant") for s, fs in (("density", 1.0), ("density", 2.5),
                                                                       ("spectrum", 1.0))}, (p, n)
            assert any(int(r[5]) < c for r in mine) and any(int(r[7]) > 1 for r in mine), (p, n)
            assert any(r[12] for r in mine), (p, n)   # a batch of short rows leaves a partial group
    for r in runs:
        assert r[14:] == ("0", "0", "OK"), r


def test_other_paths_elements(emulation):
    elements = _match(emulation, ELEMENTS)
    assert {int(r[0]) for r in elements} == {96, 97}
    for r in elements:
        assert float(r[2]) < 1e-12 and r[3] == "OK", r


def test_shared_memory_conflicts_reported(emulation):
    """The load's park write at most two-way and its stage-A read conflict-free, as in the stft emulator; the accumulator
    update and the flush's reads are printed (DESIGN.md §4.15)."""
    lines = [m.groups() for m in map(CONFLICTS.search, emulation.stdout.splitlines()) if m]
    assert len(lines) == sum(len(v) for v in SIZES.values())
    for park, stage_a, acc, flush in lines:
        assert int(park) <= 2 and stage_a == "1" and int(acc) >= 1 and int(flush) >= 1, (park, stage_a, acc, flush)

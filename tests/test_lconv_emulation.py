"""Runs the device code of the linear convolution of real rows by overlap-save (LinConvBody in onchip_kernels.cuh,
real::SegMap and the gather / scatter elements in real_kernels.cuh) on the CPU through tools/emulate_lconv.cu: the fused
kernel of every on-chip size class in both precisions for K in {1, 2, 33, N/2, N-1, N}, every mode and row lengths
around the segment length S = N - K + 1, and the gather / scatter maps of the other paths for an even and an odd N,
against a direct linear convolution in double.  Every input read and output write is checked against its row."""
import re

import pytest

from helpers import run_emulator

LINE = re.compile(r"^(fused|maps) (?:(f32|f64) )?N=(\d+) K=(\d+) (full|same|valid) L=(\d+) F=3 batch=(\d+) "
                  r"segments=(\d+).*: max rel err (\S+), reads outside row (\d+), writes outside row (\d+), "
                  r"unwritten (\d+), written twice (\d+) (OK|FAIL)$")


@pytest.fixture(scope="module")
def emulation(tmp_path_factory):
    return run_emulator("emulate_lconv", tmp_path_factory.mktemp("emulate_lconv"))


@pytest.fixture(scope="module")
def runs(emulation):
    return [m.groups() for m in map(LINE.match, emulation.stdout.splitlines()) if m]


def test_emulated_lconv_matches_direct_convolution(emulation):
    assert emulation.returncode == 0, emulation.stdout + emulation.stderr
    assert "EMULATION OK" in emulation.stdout


def test_no_stray_missing_or_double_access(runs):
    assert runs
    for r in runs:
        assert r[9:13] == ("0", "0", "0", "0") and r[13] == "OK", r


def test_every_size_class_tap_count_mode_and_length_ran(runs):
    sizes = {"f32": (128, 256, 512, 1024, 2048), "f64": (128, 256, 512)}
    for p, ns in sizes.items():
        for n in ns:
            mine = [r for r in runs if r[0] == "fused" and r[1] == p and int(r[2]) == n]
            for k in (1, 2, 33, n // 2, n - 1, n):
                s = n - k + 1
                for mode in ("full", "same", "valid"):
                    lens = {int(r[5]) for r in mine if int(r[3]) == k and r[4] == mode and r[6] == "5"}
                    want = {l for l in (1, s - 1, s, s + 1, 3 * s + 7) if l >= 1 and (mode != "valid" or l >= k)}
                    assert lens == want, (p, n, k, mode, lens, want)
            assert any(int(r[6]) != 5 for r in mine), (p, n)   # the batch whose segments leave a partial group
            assert any(int(r[7]) > 1 for r in mine), (p, n)
    for n in (96, 97):   # an even and an odd N
        assert any(r[0] == "maps" and int(r[2]) == n for r in runs), n


def test_host_runs_of_segments_give_the_same_outputs(emulation):
    lines = [l for l in emulation.stdout.splitlines() if l.startswith("maps ")]
    assert lines and all("host runs same" in l for l in lines)


def test_shared_phases_are_conflict_free(emulation):
    """ConvBody's phases have no bank conflicts; the store's reads of the park as reals at most two-way (the size
    classes whose FFTs share a warp)"""
    lines = [l for l in emulation.stdout.splitlines() if "exchange conflicts" in l]
    assert len(lines) == 8
    for line in lines:
        assert "write-back x1, stage-A read x1" in line, line
        assert re.search(r"store read x[12]$", line), line

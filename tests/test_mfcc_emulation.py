"""Runs the device code of the MFCC and log-mel spectrogram (MfccBody in onchip_kernels.cuh, both its max-sweep and
output instantiations; real::log_mel, max_key, max_fold, clamp_threshold, clamp_db and mfcc_dot in real_kernels.cuh) on
the CPU through tools/emulate_mfcc.cu: the fused kernel of every on-chip size class in both precisions for every
boundary, hops 1, N/4 and N+3, powers 1 and 2, three banks (40 HTK mels, L-1 HTK mels, an all-zero row), projections
dct NULL, 13 and 2 TP + 3, bias 0 and 1.5, the clamp off and binding with groups of 1 and 2 rows, against a direct
windowed DFT, power, bank, log, clamp and projection in double; the group slots against the maxima of the log-mels; and
the chunked route's element steps over two chunks of frames for N = 96 and 97.  Every input, weight and matrix read and
every output write is checked."""
import re

import pytest

from helpers import run_emulator

FUSED = re.compile(r"^fused (f32|f64) N=(\d+) (none|zeros|reflect) H=(\d+) L=(\d+) batch=(\d+) frames=(\d+) "
                   r"bank=(htk|full|zero-row) mels=(\d+) p=([12]) out=(\d+)( \(identity\))? bias=(\S+) clamp=(on|off) "
                   r"rows=([12])( partial)?: max rel err (\S+), outside row (\d+), not once (\d+), outside band (\d+), "
                   r"dct outside (\d+), slots off (\d+), zero rows off (\d+) (OK|FAIL)$")
CHUNKS = re.compile(r"^chunks N=(\d+) frames=8 rows=2 chunks=2: max rel err (\S+), slot rel err (\S+), clamped (\d+) "
                    r"(OK|FAIL)$")
CONFLICTS = re.compile(r"mfcc +threads +\d+  conflicts: log-mel write x(\d+); projection read x(\d+)$")

# the on-chip size classes (onchip_configs.cuh) as N = 2L, and the lanes per FFT (TP)
SIZES = {"f32": {128: 8, 256: 8, 512: 16, 1024: 16, 2048: 32}, "f64": {128: 8, 256: 8, 512: 16}}
TOL = {"f32": 1e-5, "f64": 1e-12}


@pytest.fixture(scope="module")
def emulation(tmp_path_factory):
    return run_emulator("emulate_mfcc", tmp_path_factory.mktemp("emulate_mfcc"))


def _match(emulation, pattern):
    return [m.groups() for m in map(pattern.match, emulation.stdout.splitlines()) if m]


def test_emulated_mfcc_matches_direct_sums(emulation):
    assert emulation.returncode == 0, emulation.stdout + emulation.stderr
    assert "EMULATION OK" in emulation.stdout


def test_every_size_class_and_case_ran(emulation):
    runs = _match(emulation, FUSED)
    for p, classes in SIZES.items():
        for n, tp in classes.items():
            mine = [r for r in runs if r[0] == p and int(r[1]) == n]
            for boundary in ("none", "zeros", "reflect"):
                assert {int(r[3]) for r in mine if r[2] == boundary} == {1, n // 4, n + 3}, (p, n, boundary)
            assert {(r[7], int(r[8])) for r in mine} == {("htk", 40), ("full", n // 2 - 1), ("zero-row", 40)}, (p, n)
            assert {r[9] for r in mine} == {"1", "2"}
            outs = {(int(r[10]), bool(r[11]), r[13]) for r in mine if int(r[3]) == n // 4}
            for clamp in ("on", "off"):
                assert any(ident for _, ident, c in outs if c == clamp), (p, n, clamp)
                assert any(o == 13 for o, _, c in outs if c == clamp), (p, n, clamp)
                assert any(o == 2 * tp + 3 for o, _, c in outs if c == clamp), (p, n, clamp)
            assert {float(r[12]) for r in mine} == {0.0, 1.5}
            assert {r[14] for r in mine} == {"1", "2"}
            assert any(r[15] for r in mine), (p, n)   # a batch whose frames leave a partial group
    for r in runs:
        assert float(r[16]) < TOL[r[0]], r
        assert r[17:] == ("0", "0", "0", "0", "0", "0", "OK"), r


def test_chunked_route_elements(emulation):
    chunks = _match(emulation, CHUNKS)
    assert {int(r[0]) for r in chunks} == {96, 97}
    for r in chunks:
        assert float(r[1]) < 1e-12 and float(r[2]) < 1e-12 and int(r[3]) > 0 and r[4] == "OK", r


def test_shared_memory_conflicts_reported(emulation):
    """the new phases' shared accesses (DESIGN.md §4.18): at most two-way, one line per size class"""
    lines = [m.groups() for m in map(CONFLICTS.search, emulation.stdout.splitlines()) if m]
    assert len(lines) == sum(len(v) for v in SIZES.values())
    for write, read in lines:
        assert 1 <= int(write) <= 2 and 1 <= int(read) <= 2, (write, read)

"""Runs the device code of the mel spectrogram (MelBody in onchip_kernels.cuh; real::band_scan, mel_dot, power_pair and
mel_spectrum_one in real_kernels.cuh) on the CPU through tools/emulate_mel.cu: the fused kernel of every on-chip size
class in both precisions for every boundary, hops 1, N/4 and N+3, powers 1 and 2 and three filter banks (HTK triangular,
one dense random row, and N/2+6 rows with zero rows, single weights at bins 0 and N/2 and negative weights) against a
direct windowed DFT, power and bank in double; and the spectrum path's per-output function over two chunks of frames
and the band rule for N = 96 and 97.  Every input read, output write and weight read is checked."""
import re

import pytest

from helpers import run_emulator

FUSED = re.compile(r"^fused (f32|f64) N=(\d+) (none|zeros|reflect) H=(\d+) L=(\d+) batch=(\d+) frames=(\d+) "
                   r"bank=(htk|dense|special) mels=(\d+) p=([12])( partial)?: max rel err (\S+), outside row (\d+), "
                   r"not once (\d+), outside band (\d+), zero rows not 0 (\d+) (OK|FAIL)$")
SPECTRA = re.compile(r"^spectra N=(\d+) bank=(htk|dense|special) mels=(\d+) p=([12]) chunks=2: max rel err (\S+), "
                     r"outside row (\d+), not once (\d+), outside band (\d+), zero rows not 0 (\d+) (OK|FAIL)$")
BANDS = re.compile(r"^bands N=(\d+) bank=(htk|dense|special) mels=(\d+): (OK|FAIL)$")
CONFLICTS = re.compile(r"park write x(\d+), stage-A read x(\d+); power write x(\d+); mel read x(\d+) \(HTK, 80 mels\)$")

# the on-chip size classes (onchip_configs.cuh) as N = 2L: every one must have been emulated
SIZES = {"f32": (128, 256, 512, 1024, 2048), "f64": (128, 256, 512)}


@pytest.fixture(scope="module")
def emulation(tmp_path_factory):
    return run_emulator("emulate_mel", tmp_path_factory.mktemp("emulate_mel"))


def _match(emulation, pattern):
    return [m.groups() for m in map(pattern.match, emulation.stdout.splitlines()) if m]


def test_emulated_mel_matches_direct_sums(emulation):
    assert emulation.returncode == 0, emulation.stdout + emulation.stderr
    assert "EMULATION OK" in emulation.stdout


def test_every_size_class_boundary_hop_power_and_bank_ran(emulation):
    runs = _match(emulation, FUSED)
    for p, ns in SIZES.items():
        for n in ns:
            mine = [r for r in runs if r[0] == p and int(r[1]) == n]
            bins = n // 2 + 1
            for boundary in ("none", "zeros", "reflect"):
                at = {(int(r[3]), r[7], int(r[9])) for r in mine if r[2] == boundary}
                # hop N/4: every bank at both powers
                assert {(n // 4, b, pw) for b in ("htk", "dense", "special") for pw in (1, 2)} <= at, (p, n, boundary)
                for hop in (1, n + 3):
                    assert {int(r[3]) for r in mine if r[2] == boundary} >= {hop}, (p, n, boundary, hop)
            mels = {r[7]: int(r[8]) for r in mine}
            assert mels == {"htk": 80, "dense": 1, "special": bins + 5}, (p, n, mels)
            assert any(r[10] for r in mine), (p, n)   # a batch whose frames leave a partial group
    for r in runs:
        assert r[12:] == ("0", "0", "0", "0", "OK"), r


def test_spectrum_path_and_band_rule(emulation):
    spectra = _match(emulation, SPECTRA)
    bands = _match(emulation, BANDS)
    for n in (96, 97):
        assert {(r[1], r[3]) for r in spectra if int(r[0]) == n} == {(b, pw) for b in ("htk", "dense", "special")
                                                                      for pw in ("1", "2")}, n
        assert {r[1] for r in bands if int(r[0]) == n} == {"htk", "dense", "special"}, n
    for r in spectra:
        assert float(r[4]) < 1e-12 and r[5:] == ("0", "0", "0", "0", "OK"), r
    for r in bands:
        assert r[3] == "OK", r


def test_shared_memory_conflicts_reported(emulation):
    """StftBody's load phases as in the stft emulator (park write at most two-way, stage-A read conflict-free), the power
    write into the park at most two-way; the mel phase's worst case is printed (DESIGN.md §4.14)."""
    lines = [m.groups() for m in map(CONFLICTS.search, emulation.stdout.splitlines()) if m]
    assert len(lines) == sum(len(v) for v in SIZES.values())
    for park, stage_a, power, mel in lines:
        assert int(park) <= 2 and stage_a == "1" and int(power) <= 2, (park, stage_a, power)
        assert int(mel) >= 1

"""Runs the device code of the short-time Fourier transform (StftBody in onchip_kernels.cuh, real::FrameMap and the
gather / overlap-add elements and run cut in real_kernels.cuh) on the CPU through tools/emulate_stft.cu: the fused
forward kernel of every on-chip size class in both precisions for every boundary, hops 1, 37, N/4, N and N+3 and row
lengths from the smallest legal one up, against a direct windowed DFT in double; and the gather and overlap-add of the
other paths for an even and an odd N, the inverse over runs cut at several places.  Every input read, spectrum write
and output write is checked."""
import re

import pytest

from helpers import run_emulator

FUSED = re.compile(r"^fused (f32|f64) N=(\d+) (none|zeros|reflect) H=(\d+) L=(\d+) batch=(\d+) frames=(\d+)( partial)?: "
                   r"max rel err (\S+), outside row (\d+), not once (\d+) (OK|FAIL)$")
GATHER = re.compile(r"^gather N=(\d+) (none|zeros|reflect) H=(\d+) L=(\d+) .*: max rel err (\S+), outside row (\d+), "
                    r"not once (\d+) (OK|FAIL)$")
OLA = re.compile(r"^overlap-add N=(\d+) center=(\d) H=(\d+) frames=(\d+) out_len=(\d+) scratch=(\d+) runs=(\d+) "
                 r"(same bits|DIFFERENT BITS): max rel err (\S+), outside row (\d+), not once (\d+) (OK|FAIL)$")


@pytest.fixture(scope="module")
def emulation(tmp_path_factory):
    return run_emulator("emulate_stft", tmp_path_factory.mktemp("emulate_stft"))


def _match(emulation, pattern):
    return [m.groups() for m in map(pattern.match, emulation.stdout.splitlines()) if m]


def test_emulated_stft_matches_direct_sums(emulation):
    assert emulation.returncode == 0, emulation.stdout + emulation.stderr
    assert "EMULATION OK" in emulation.stdout


def test_every_size_class_boundary_hop_and_length_ran(emulation):
    runs = _match(emulation, FUSED)
    sizes = {"f32": (128, 256, 512, 1024, 2048), "f64": (128, 256, 512)}
    for p, ns in sizes.items():
        for n in ns:
            mine = [r for r in runs if r[0] == p and int(r[1]) == n]
            for boundary, least, pad in (("none", n, 0), ("zeros", 1, n // 2), ("reflect", n // 2 + 1, n // 2)):
                for hop in (1, 37, n // 4, n, n + 3):
                    lens = {int(r[4]) for r in mine if r[2] == boundary and int(r[3]) == hop}
                    assert {least, n, n + 1} <= lens, (p, n, boundary, hop, lens)
                    assert any(1 + (l + 2 * pad - n) // hop >= 4 for l in lens), (p, n, boundary, hop, lens)
            assert any(r[7] for r in mine), (p, n)   # a batch whose frames leave a partial group
    for r in runs:
        assert r[9:] == ("0", "0", "OK"), r


def test_spectrum_accesses_are_one_aligned_complex_value(emulation):
    lines = [l for l in emulation.stdout.splitlines() if "stft spectrum accesses" in l]
    assert lines and all(l.endswith("OK") and "misaligned 0, outside 0" in l for l in lines)
    for l in lines:
        widest = int(re.search(r"widest (\d+) B", l).group(1))
        assert widest in (8, 16), l


def test_gather_and_overlap_add_maps(emulation):
    gathers = _match(emulation, GATHER)
    olas = _match(emulation, OLA)
    for n in (96, 97):
        assert {r[1] for r in gathers if int(r[0]) == n} == {"none", "zeros", "reflect"}, n
        mine = [r for r in olas if int(r[0]) == n]
        assert {r[1] for r in mine} == {"0", "1"}, n
        assert any(int(r[6]) > 2 for r in mine), n   # some inverse was cut into several runs of one row
    for r in gathers:
        assert r[5:] == ("0", "0", "OK"), r
    for r in olas:
        assert r[7] == "same bits" and r[9:] == ("0", "0", "OK"), r


def test_load_phase_conflicts_reported(emulation):
    """The park writes are at most two-way (size classes whose FFTs share a warp); the stage-A reads conflict-free."""
    lines = [l for l in emulation.stdout.splitlines() if "load conflicts" in l]
    assert len(lines) == 8
    for line in lines:
        assert re.search(r"park write x[12], stage-A read x1$", line), line

"""Runs the device code of the type-IV DCT and the MDCT (Dct4Body / MdctBody in onchip_kernels.cuh and the real::dct4*,
mdct* and imdct* steps of real_kernels.cuh) on the CPU through tools/emulate_mdct.cu: Dct4Body for every on-chip size
class in both precisions, all three norms, a batch of C + 3 rows, and in place against out of place; MdctBody with
center on and off at four row lengths on batches that leave a partial group; against the direct formulas in double.
Every input read must lie in its row and every output be written once.  Also the element steps of the other paths for
N = 2, 4 and 96 over two chunks, imdct_add_one over the istft_runs cuts of several scratch sizes (the same bits, and
the round trip back to the input), and the bank conflicts of the new phases."""
import re

import pytest

from helpers import run_emulator

DCT4 = re.compile(r"^fused dct4 (f32|f64) N=(\d+) batch=(\d+) norm=(backward|ortho|forward): max rel err (\S+), "
                  r"outside row (\d+), not once (\d+), in place (same|differs) (OK|FAIL)$")
MDCT = re.compile(r"^fused mdct (f32|f64) N=(\d+) center=([01]) L=(\d+) frames=(\d+) batch=(\d+) norm=(\w+): max rel err "
                  r"(\S+), outside row (\d+), not once (\d+) (OK|FAIL)$")
ELEMENTS = re.compile(r"^elements (f32|f64) (dct4|mdct|imdct) N=(\d+) (.*) (OK|FAIL)$")
CONFLICTS = re.compile(r"(f32|f64) L=(\d+) threads \d+ conflicts: load x(\d+), pre x(\d+), post x(\d+), "
                       r"store x(\d+)$")

# the on-chip size classes (onchip_configs.cuh) as N = 2L, and their FFTs per CTA (C)
SIZES = {"f32": {128: 32, 256: 32, 512: 16, 1024: 16, 2048: 8}, "f64": {128: 32, 256: 32, 512: 16}}
TOL = {"f32": 1e-5, "f64": 1e-12}


@pytest.fixture(scope="module")
def emulation(tmp_path_factory):
    return run_emulator("emulate_mdct", tmp_path_factory.mktemp("emulate_mdct"))


def _match(emulation, pattern):
    return [m.groups() for m in map(pattern.match, emulation.stdout.splitlines()) if m]


def test_emulated_mdct_matches_direct_sums(emulation):
    assert emulation.returncode == 0, emulation.stdout + emulation.stderr
    assert "EMULATION OK" in emulation.stdout


def test_every_dct4_size_class_and_norm_ran(emulation):
    runs = _match(emulation, DCT4)
    assert {(r[0], int(r[1]), r[3]) for r in runs} == {
        (p, n, nm) for p, classes in SIZES.items() for n in classes for nm in ("backward", "ortho", "forward")}
    for r in runs:
        assert int(r[2]) == SIZES[r[0]][int(r[1])] + 3, r
        assert float(r[4]) < TOL[r[0]], r
        assert r[5:] == ("0", "0", "same", "OK"), r


def test_every_mdct_size_class_center_and_length_ran(emulation):
    runs = _match(emulation, MDCT)
    seen = {}
    for r in runs:
        p, n, center, length, frames, batch = r[0], int(r[1]), int(r[2]), int(r[3]), int(r[4]), int(r[5])
        c = SIZES[p][n]
        assert frames * batch > c and (frames * batch) % c != 0, r   # a full group of frames and a partial one
        assert float(r[7]) < TOL[p], r
        assert r[8:] == ("0", "0", "OK"), r
        seen.setdefault((p, n, center), set()).add(length)
    assert set(seen) == {(p, n, c) for p, classes in SIZES.items() for n in classes for c in (0, 1)}
    for (p, n, center), lengths in seen.items():
        assert (1 if center else 2 * n) in lengths and 2 * n + 1 in lengths and 4 * n in lengths, (p, n, center)
        assert len(lengths) == 4


def test_other_paths_elements(emulation):
    elements = _match(emulation, ELEMENTS)
    kinds = {(r[0], r[1], int(r[2])) for r in elements}
    assert kinds == {(p, k, n) for p in ("f32", "f64") for k in ("dct4", "mdct", "imdct") for n in (2, 4, 96)}
    for r in elements:
        assert r[4] == "OK", r
        if r[1] == "imdct":
            assert "outputs same, not once 0" in r[3], r
        err = float(re.search(r"max rel err ([^,\s]+)", r[3]).group(1))
        assert err < TOL[r[0]], r


def test_shared_memory_conflicts_reported(emulation):
    """The new load, pre-twiddle, post and store phases are at most two-way conflicted (DESIGN.md §4.20)."""
    lines = [m.groups() for m in map(CONFLICTS.search, emulation.stdout.splitlines()) if m]
    assert {(p, 2 * int(l)) for p, l, *_ in lines} == {(p, n) for p, c in SIZES.items() for n in c}
    for line in lines:
        assert all(1 <= int(d) <= 2 for d in line[2:]), line

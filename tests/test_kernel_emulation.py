"""Runs the fused kernels' device code (tilefft.cuh / twopass_kernels.cuh, all __host__ __device__) on
the CPU through tools/emulate.cu: every thread of every CTA, phase by phase, for each configuration of the
library's tables, against a double-precision FFT; also asserts the shared-memory exchange is
bank-conflict free.  This is the no-GPU check of index maps, twiddle tables and layouts.

The emulator enumerates the tables the library selects from (onchip_configs.cuh, twopass::visit_config,
fused_configs.cuh).  The lists below are the independent statement of what must be covered, so a configuration
that falls out of a table fails here instead of silently dropping out of the emulation."""
import re

import pytest

from helpers import run_emulator

ONCHIP = {"f32": (64, 128, 256, 512, 1024), "f64": (64, 128, 256)}
BLUESTEIN = {"f32": (64, 256, 1024), "f64": (64, 256)}
TWOPASS = {"f32": range(11, 21), "f64": range(9, 17)}
# persistent kernel: the configuration of every size
FUSED = {"f32": range(13, 21), "f64": (12, 13, 14, 16)}


@pytest.fixture(scope="module")
def emulation(tmp_path_factory):
    return run_emulator("emulate", tmp_path_factory.mktemp("emulate"))


def blocks(out):
    """Label (the text before the first ':') of each unindented line -> the indented lines that follow it."""
    res, cur = {}, None
    for line in out.splitlines():
        if line and not line.startswith(" "):
            cur = res.setdefault(line.split(":")[0], [])
        elif cur is not None:
            cur.append(line.strip())
    return res


def both_directions_ok(lines):
    return all(any(l.startswith(d + ":") and l.endswith("OK") for l in lines) for d in ("forward", "inverse"))


def test_emulated_kernels_match_f64_fft(emulation):
    assert emulation.returncode == 0, emulation.stdout + emulation.stderr
    assert "EMULATION OK" in emulation.stdout
    for line in emulation.stdout.splitlines():
        if "exchange conflicts" in line:
            assert "write x1, read x1" in line, line


def test_every_onchip_and_bluestein_class_ran(emulation):
    out = emulation.stdout
    for p, sizes in ONCHIP.items():
        for l in sizes:
            for d in ("forward", "inverse"):
                assert re.search(rf"^onchip {p} L={l} {d}: .* OK$", out, re.M), (p, l, d)
    for p, sizes in BLUESTEIN.items():
        for l in sizes:
            for d in ("forward", "inverse"):
                assert re.search(rf"^bluestein {p} N=\d+ \(L={l}\) {d}: .* OK$", out, re.M), (p, l, d)


def test_every_two_pass_size_ran(emulation):
    b = blocks(emulation.stdout)
    for p, ks in TWOPASS.items():
        for k in ks:
            label = f"{p} 2^{k}"
            assert label in b and both_directions_ok(b[label]), (label, b.get(label))


def test_every_persistent_configuration_ran(emulation):
    b = blocks(emulation.stdout)
    labels = [f"fused {p} 2^{k}" for p, ks in FUSED.items() for k in ks]
    for label in labels:
        assert label in b and both_directions_ok(b[label]), (label, b.get(label))


def test_every_persistent_queue_checked(emulation):
    out = emulation.stdout
    for p, ks in FUSED.items():
        for k in ks:
            assert re.search(rf"^fused work queue {p} 2\^{k}(, pair items)? \(T1 .*properties OK$", out, re.M), (p, k)

"""Records what the reference's own FFI test programs need from libfourier.so.

    python -m oracle.ffi_symbols REFERENCE_CHECKOUT

Compiles fourier-ffi/test.c and test.cpp of a reference checkout with the reference's warning flags
(fourier-ffi/CMakeLists.txt:9-13), once against the reference's header and once against include/fourier.h, into
oracle/_ref/ (git-ignored), and writes the symbols each object leaves undefined to
tests/golden/reference_ffi_symbols.json.  tests/test_abi.py checks libfourier.so against that file, so the
drop-in check needs no reference checkout.
"""
import json
import os
import subprocess
import sys

_HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(_HERE)
OUT_DIR = os.path.join(_HERE, "_ref")
GOLDEN = os.path.join(ROOT, "tests", "golden", "reference_ffi_symbols.json")
PROGRAMS = (("test.c", "gcc"), ("test.cpp", "g++"))


def undefined_symbols(obj):
    out = subprocess.run(["nm", "-u", obj], capture_output=True, text=True, check=True).stdout
    return sorted({line.split()[-1] for line in out.splitlines() if line.strip()})


def record(reference):
    ffi = os.path.join(reference, "fourier-ffi")
    os.makedirs(OUT_DIR, exist_ok=True)
    entries = {}
    for src, cc in PROGRAMS:
        for hdr, inc in (("ours", os.path.join(ROOT, "include")), ("reference", os.path.join(ffi, "include"))):
            obj = os.path.join(OUT_DIR, f"{src}.{hdr}.o")
            subprocess.run([cc, "-Wall", "-Wextra", "-pedantic", "-Werror", "-I", inc, "-c", os.path.join(ffi, src),
                            "-o", obj], check=True, capture_output=True)
            entries[f"{src}-{hdr}"] = undefined_symbols(obj)
    data = {"source": "undefined symbols of the reference's fourier-ffi/test.c and test.cpp, compiled with "
                      "-Wall -Wextra -pedantic -Werror against the named header (oracle/ffi_symbols.py)",
            "undefined": entries}
    with open(GOLDEN, "w") as f:
        json.dump(data, f, sort_keys=True)
        f.write("\n")
    return GOLDEN


if __name__ == "__main__":
    if len(sys.argv) != 2:
        raise SystemExit(__doc__)
    print(record(sys.argv[1]))

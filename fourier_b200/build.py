"""Builds libfourier.so (hand-written sm_90a CUDA + the C ABI) in-tree with nvcc.

    python -m fourier_b200.build [--force]

Output: fourier_b200/lib/libfourier.so.0.1.0 with SONAME libfourier.so.0 and the usual symlinks
(the reference's cdylib is named `fourier` with SONAME libfourier.so.0:
fourier-ffi/CMakeLists.txt:15-19,55-65).  Objects go to build/ (git-ignored).  nvcc cross-compiles
without a GPU.
"""
import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(HERE, "csrc")
LIBDIR = os.path.join(HERE, "lib")
OBJDIR = os.path.join(ROOT, "build", "obj")
VERSION = "0.1.0"
SONAME = "libfourier.so.0"
REAL = f"libfourier.so.{VERSION}"

SOURCES = ["plan.cu", "host_math.cu", "stockham_generic.cu", "onchip.cu", "cta_fft.cu", "twopass.cu", "synth.cu", "exchange.cu", "dist_fft.cu", "bigpow2.cu", "real.cu", "capi.cu"]

# H100: the kernels use TMA and mbarrier, so the arch-specific target is required
GENCODE = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = [
    "-std=c++17", "-O3", "-lineinfo",
    *GENCODE,
    "-Xcompiler", "-fPIC,-fvisibility=hidden",
    "--expt-relaxed-constexpr",
    "-diag-suppress", "20012",
]


def nvcc():
    exe = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(exe):
        raise RuntimeError("nvcc not found: libfourier.so cannot be built (there is no CPU fallback)")
    return exe


def _deps():
    hdrs = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".h", ".cuh"))]
    hdrs += [os.path.join(ROOT, "include", f) for f in os.listdir(os.path.join(ROOT, "include"))]
    return hdrs


def _stale(target, sources):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(s) > t for s in sources)


def lib_path():
    return os.path.join(LIBDIR, REAL)


def build(force=False, verbose=False):
    os.makedirs(OBJDIR, exist_ok=True)
    os.makedirs(LIBDIR, exist_ok=True)
    hdrs = _deps()
    exe = nvcc()
    jobs = []
    objs = []
    for src in SOURCES:
        s = os.path.join(CSRC, src)
        o = os.path.join(OBJDIR, src.replace(".cu", ".o"))
        objs.append(o)
        if force or _stale(o, [s] + hdrs):
            jobs.append([exe] + NVCC_FLAGS + ["-c", s, "-o", o])

    def run(cmd):
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("nvcc failed:\n" + " ".join(cmd) + "\n" + r.stdout + r.stderr)
        if verbose and (r.stdout or r.stderr):
            print(r.stdout + r.stderr)

    with ThreadPoolExecutor(max_workers=min(8, max(1, len(jobs)))) as ex:
        list(ex.map(run, jobs))
    out = lib_path()
    if force or jobs or _stale(out, objs):
        run([exe, "-shared", *GENCODE, "-Xlinker", f"-soname={SONAME}",
             "-o", out] + objs)
        for link in (SONAME, "libfourier.so"):
            lp = os.path.join(LIBDIR, link)
            if os.path.lexists(lp):
                os.remove(lp)
            os.symlink(REAL, lp)
    return out


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))

"""Every complex path outside the persistent two-pass kernel, checked transform by transform: the trivial copy (N = 1),
the CTA kernel, the on-chip kernels, the fused and CTA-chirp Bluestein kernels, unfused Bluestein around an inner plan,
the per-stage path over HBM, the three-pass path, their chunk loops and the host-pointer pipeline.

Every case runs one check on a periodic, scaled batch: row b is 2^s(b) * base[b mod P], P = 97 random rows, s(b) cycling
over the 49 exponents -24 .. 24 (49 and 97 are coprime: no two neighbouring rows are equal, and the pattern repeats only
every 4753 rows).  Scaling by a power of two commutes with every IEEE operation, FMA included, as long as nothing
overflows or underflows, and every kernel's arithmetic is data-independent.  So

  1. only the base rows need a reference: numpy's FFT in long double, per transform, within the bound of the path;
  2. every other row is checked on the device, bit for bit: out[b] * 2^-s(b) == out[b mod P] * 2^-s(b mod P).  A row
     that picks up a neighbour's data fails, even when the neighbour is 2^48 times smaller;
  3. outputs start as NaN and a decoy call on other input runs first;
  4. the batch is bit-identical in place and out of place, and its base rows to the same rows run one at a time;
  5. the plan runs the path the case is meant for (path_name, inner_path_name and kernel_name(), from expected_path).

Batches are sized from the launch rules so that grid-stride loops wrap and scratch / staging chunk loops run more than
once; transforms too large for a long-double reference are checked on closed-form inputs (an impulse and a few tones).
Cases that do not fit the free device memory are skipped with the reason."""
import math

import numpy as np
import pytest
import torch

import fourier_b200 as fb
from helpers import per_transform_err, poisoned_like, scale_ld, truth_ld
from test_gpu_persistent_schedule import check_bits, device_input, run

pytestmark = pytest.mark.gpu

T = fb.Transform
TDT = {"f32": torch.complex64, "f64": torch.complex128}
BITS = {"f32": torch.int32, "f64": torch.int64}
ESIZE = {"f32": 8, "f64": 16}   # bytes per complex sample
P = 97                          # base rows of a periodic batch (prime)
SPAN = 49                       # exponents -24 .. 24
FIRST, DECOY = 11, 700001       # first_transform of the base rows and of the decoy rows
MIB, GIB = 1 << 20, 1 << 30

# ---- the plan's selection rules (Plan::init, init_bluestein, cta_fits, init_bigpow2, init_threepass_radix3) ----------
ONCHIP = {"f32": {64: 4, 128: 4, 256: 3, 512: 2, 1024: 2}, "f64": {64: 3, 128: 2, 256: 1}}   # L: min CTAs per SM
ONCHIP_TP = {64: 8, 128: 8, 256: 16, 512: 16, 1024: 32}     # threads per transform (L / E)
BLUE_FUSED = {"f32": {64: 8, 256: 8, 1024: 16}, "f64": {64: 8, 256: 8}}   # L = M / 2: warps per CTA
TWOPASS = {"f32": range(11, 21), "f64": range(9, 17)}       # log2 N of the two-pass kernels
PERSISTENT = {"f32": range(13, 21), "f64": (12, 13, 14, 16)}
THREEPASS = {"f32": range(21, 31), "f64": range(17, 25)}
SMEM_LIMIT = 227 * 1024
SCRATCH = 512 * MIB            # kScratchTargetBytes
HOST_CHUNK = 64 * MIB          # kHostChunkBytes
ZERO_COPY, SINGLE = 64 << 10, 1 * MIB   # kHostZeroCopyBytes, kHostSmallBytes
BIG_CHUNK = 2 * GIB            # exec_bigpow2: intermediate of at most 2 GiB

# per-transform bounds per path (tools/emulate.cu on the same arithmetic; general stages have no emulator bound)
BOUND = {"trivial": (0.0, 0.0), "onchip": (2e-6, 5e-15), "twopass": (2e-6, 5e-15), "threepass": (2e-6, 5e-15),
         "threepass_radix3": (2e-6, 1e-14), "onchip_cta": (3e-6, 5e-15), "global_stages": (3e-6, 1e-14),
         "bluestein_fused": (4e-6, 1e-13), "bluestein": (4e-6, 1e-13)}


def smooth(n):
    while n % 2 == 0:
        n //= 2
    while n % 3 == 0:
        n //= 3
    return n == 1


def log2(n):
    return n.bit_length() - 1


def is_pow2(n):
    return n & (n - 1) == 0


def padded(e):
    return e + (e >> 5)


def cta_smem(real, group, n):
    return 2 * (padded(group * n) + 1) * ESIZE[real]


def cta_fits(real, n):
    return 2 <= n < (1 << 20) and cta_smem(real, 1, n) <= SMEM_LIMIT


def bluestein_m(n):
    m = 1
    while m < 2 * n - 1:
        m <<= 1
    return m


def expected_path(real, n):
    """-> (path_name, inner_path_name, a fragment of kernel_name())"""
    if n == 1:
        return "trivial", "trivial", "scale_copy_kernel"
    if smooth(n):
        if is_pow2(n):
            if n in ONCHIP[real]:
                return "onchip", "trivial", "onchip::onchip_fft_kernel"
            if log2(n) in TWOPASS[real]:
                kernel = "fused::fused_twopass_kernel" if log2(n) in PERSISTENT[real] else "twopass::tile_kernel"
                return "twopass", "trivial", kernel
            if log2(n) in THREEPASS[real]:
                return "threepass", "twopass", "outer::column_kernel"
        if cta_fits(real, n):
            return "onchip_cta", "trivial", "cta::cta_fft_kernel"
        r, b = n, 1
        while r % 3 == 0 and b < 27:
            r, b = r // 3, b * 3
        if b > 1 and is_pow2(r) and r % 3 and log2(r) in TWOPASS[real]:
            return "threepass", "twopass", "outer::radix3_column_kernel"
        return "global_stages", "trivial", "stockham_stage_kernel"
    m = bluestein_m(n)
    if m // 2 in BLUE_FUSED[real]:
        return "bluestein_fused", "trivial", "onchip::bluestein_fused_kernel"
    if cta_fits(real, m):
        return "bluestein_fused", "trivial", "cta::cta_fft_kernel (chirp mode)"
    return "bluestein", expected_path(real, m)[0], "chirp / pointwise kernels"


def bound(real, n):
    path, _, kernel = expected_path(real, n)
    if path == "threepass" and "radix3" in kernel:
        path = "threepass_radix3"
    return BOUND[path][0 if real == "f32" else 1]


def cta_group(real, n):
    """group_for (cta_fft.cu): transforms per CTA iteration"""
    gmax = max(1, (32768 // ESIZE[real]) // n)
    radices, r = [], n
    while r % 16 == 0:
        radices, r = radices + [16], r // 16
    for q in (8, 4, 2):
        if r % q == 0 and r // q % 2:
            radices, r = radices + [q], r // q
    while r % 9 == 0:
        radices, r = radices + [9], r // 9
    if r % 3 == 0:
        radices, r = radices + [3], r // 3
    best, best_eff = gmax, 0.0
    for g in range(gmax, max(1, gmax // 2) - 1, -1):
        work = slots = 0.0
        for q in radices:
            bf = g * (n // q)
            work += bf * q
            slots += math.ceil(bf / 256) * 256 * q
        if work / slots > best_eff + 1e-9:
            best, best_eff = g, work / slots
    return best


def grid_wrapping_batch(real, n):
    """A batch of about 1.3 sweeps of the grid of the kernel that serves n (cta_fft.cu launch, onchip.cu launch and
    bluestein), ending in a partial group; None when the path has no such grid-stride loop."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    path, _, kernel = expected_path(real, n)
    if path == "onchip":
        group = 256 // ONCHIP_TP[n]
        grid = sms * ONCHIP[real][n] * 4
    elif kernel.startswith("cta::cta_fft_kernel"):
        len_ = n if path == "onchip_cta" else bluestein_m(n)
        group = cta_group(real, len_)
        grid = sms * max(1, min(8, SMEM_LIMIT // (cta_smem(real, group, len_) + 1024)))
    elif kernel == "onchip::bluestein_fused_kernel":
        group = BLUE_FUSED[real][bluestein_m(n) // 2] * 32 // ONCHIP_TP[bluestein_m(n) // 2]
        grid = sms * 2
    else:
        return None
    return int(1.3 * grid) * group + max(1, group // 2)


def global_stages(n):
    """number of radix stages of init_global_stages"""
    twos = threes = 0
    while n % 2 == 0:
        n, twos = n // 2, twos + 1
    while n % 3 == 0:
        n, threes = n // 3, threes + 1
    stages = 0
    while twos >= 5 or twos == 3:
        stages, twos = stages + 1, twos - 3
    while twos >= 2:
        stages, twos = stages + 1, twos - 2
    return stages + (twos == 1) + threes


# ---- resources -------------------------------------------------------------------------------------------------------

def require(nbytes, what):
    """Skips (never fails) when `nbytes` of device memory, plus a margin, are not free."""
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    free = torch.cuda.mem_get_info()[0]
    if free < nbytes * 1.05 + 512 * MIB:
        pytest.skip(f"{what} needs {nbytes / GIB:.1f} GiB of device memory, {free / GIB:.1f} GiB free")


def make_plan(real, n):
    p = fb.create_fft_f32(n) if real == "f32" else fb.create_fft_f64(n)
    path, inner, kernel = expected_path(real, n)
    info, name = p.info(), p.kernel_name()
    assert (info["path_name"], info["inner_path_name"]) == (path, inner) and kernel in name, \
        f"{real} N={n}: plan runs {info['path_name']} / {info['inner_path_name']} / {name!r}, expected {path} / " \
        f"{inner} / {kernel!r}"
    return p


# ---- periodic, scaled batches ---------------------------------------------------------------------------------------

def exponents(rows):
    return rows % SPAN - (SPAN // 2)


def pow2(s, real):
    """exactly 2^s for an integer tensor s, as a real tensor of the precision"""
    if real == "f32":
        return ((s + 127) << 23).to(torch.int32).view(torch.float32)
    return ((s + 1023) << 52).view(torch.float64)


def _row_step(n):
    return max(1, (64 * MIB) // n)


def periodic_input(real, n, batch, first):
    """-> the periodic batch (device) and its base rows (host, unscaled)"""
    base = device_input(real, min(P, batch), n, first)
    x = torch.empty((batch, n), dtype=TDT[real], device="cuda")
    xr, br = torch.view_as_real(x), torch.view_as_real(base)
    for r0 in range(0, batch, _row_step(n)):
        rows = torch.arange(r0, min(batch, r0 + _row_step(n)), device="cuda")
        torch.mul(br[rows % P], pow2(exponents(rows), real)[:, None, None], out=xr[r0:r0 + rows.numel()])
    return x, base.cpu().numpy()


def unscaled(y, real, r0, r1):
    """rows r0 .. r1-1 of y times 2^-s(b), as a real view"""
    rows = torch.arange(r0, r1, device="cuda")
    return torch.view_as_real(y[r0:r1]) * pow2(-exponents(rows), real)[:, None, None]


def periodic_mismatch(y, real):
    """-> the rows b >= P whose unscaled bits differ from those of row b mod P"""
    batch, n = y.shape
    if batch <= P:
        return []
    base = unscaled(y, real, 0, P).view(BITS[real])
    bad = []
    for r0 in range(P, batch, _row_step(n)):
        r1 = min(batch, r0 + _row_step(n))
        u = unscaled(y, real, r0, r1).view(BITS[real])
        rows = torch.arange(r0, r1, device="cuda") % P
        diff = (u != base[rows]).flatten(1).any(dim=1)
        bad += (torch.nonzero(diff).flatten() + r0).tolist()
    return bad


def reference_error(y, ref, real, tol, what):
    """per-transform error of the base rows of y (unscaled) against `ref`; -> (worst, failure text or None)"""
    rows = ref.shape[0]
    u = torch.view_as_complex(unscaled(y, real, 0, rows).contiguous()).cpu().numpy()
    err = per_transform_err(u, ref)
    bad = np.nonzero(~(err <= tol))[0]
    if bad.size == 0:
        return float(err.max()), None
    return float(err.max()), (f"{what}: {bad.size} of {rows} base transforms off the long-double reference (tol "
                              f"{tol:.0e}, worst {err.max():.2e}): rows {bad[:8].tolist()}")


class Refs:
    """Unscaled long-double spectra of the base rows, forward and inverse, computed on first use."""

    def __init__(self, base):
        self.base, self.cache = base, {}

    def __call__(self, code, rows):
        fwd = T(code).is_forward()
        if fwd not in self.cache:
            self.cache[fwd] = truth_ld(self.base, int(T.Fft if fwd else T.UnscaledIfft))
        return scale_ld(self.cache[fwd][:rows], int(code))


def one_by_one(p, x, code):
    """Every transform of `x` on its own (batch 1), from a copy at an allocation's start: a row of an odd f32 length
    does not start on the 16 bytes the library requires."""
    out = poisoned_like(x)
    for b in range(x.shape[0]):
        y = poisoned_like(x[b:b + 1])
        p.transform(x[b:b + 1].clone(), y, code)
        out[b] = y[0]
    return out


def check_batch(p, real, n, x, refs, code, tol, what, decoy=None, single=True, in_place=True):
    """The standard check of one call on the periodic batch x; -> (worst error, failures, launches of the call)"""
    batch = x.shape[0]
    rows = min(P, batch)
    out = run(p, x, code, decoy)
    launched = p.info()["last_launches"]
    worst, msg = reference_error(out, refs(code, rows), real, tol, what)
    failures = [msg] if msg else []
    bad = periodic_mismatch(out, real)
    if bad:
        failures.append(f"{what}: {len(bad)} of {batch - P} rows beyond the base rows differ from their base row "
                        f"(scaled by a power of two): rows {bad[:8]}, b mod P = {[b % P for b in bad[:8]]}")
    if in_place:
        z = x.clone()
        p.transform_in_place(z, code)
        failures += [m for m in [check_bits(z, out, real, P, f"{what}: in place vs out of place")] if m]
        del z
    if single:
        s = one_by_one(p, x[:rows], code)
        failures += [m for m in [check_bits(out[:rows], s, real, P, f"{what}: base rows vs batch 1")] if m]
    return worst, failures, launched


def check_size(real, n, batches, codes_at=None, tag=""):
    """The standard check of size n at each batch (Fft and SqrtScaledIfft; every code at the batches in codes_at)."""
    p = make_plan(real, n)
    tol = bound(real, n)
    top = max(batches)
    require(5 * top * n * ESIZE[real], f"{real} N={n} batch {top}")
    x, base = periodic_input(real, n, top, FIRST)
    decoy, _ = periodic_input(real, n, top, DECOY)
    refs = Refs(base)
    failures, worst = [], 0.0
    for batch in batches:
        codes = list(T) if batch in (codes_at or ()) else [T.Fft, T.SqrtScaledIfft]
        for code in codes:
            w, f, _ = check_batch(p, real, n, x[:batch], refs, code, tol, f"{code.name} batch {batch}", decoy[:batch])
            worst, failures = max(worst, w), failures + f
    torch.cuda.synchronize()
    print(f"\n{real} N={n} {p.info()['path_name']} {p.kernel_name()}{tag}: batches {batches}, worst per-transform "
          f"error {worst:.2e} (bound {tol:.0e})", end="")
    p.close()
    assert not failures, f"{real} N={n}:\n  " + "\n  ".join(failures)


# ---- 1. every {2,3}-smooth N <= 40000, and N = 1 -----------------------------------------------------------------------

SMOOTH = sorted({2 ** a * 3 ** b for a in range(16) for b in range(10) if 2 ** a * 3 ** b <= 40000})
SMOOTH_CASES = [(r, n) for r in ("f32", "f64") for n in SMOOTH]


@pytest.mark.parametrize("real,n", SMOOTH_CASES, ids=[f"{r}-{n}" for r, n in SMOOTH_CASES])
def test_smooth_size(real, n):
    batches = [1, 3, P]
    wrap = grid_wrapping_batch(real, n)
    if wrap:
        batches.append(wrap)
    check_size(real, n, batches, codes_at=(P,), tag=f", grid-wrapping batch {wrap}" if wrap else "")


def test_trivial_in_place_launches_nothing():
    p = make_plan("f32", 1)
    x, _ = periodic_input("f32", 1, P, FIRST)
    for code in T:   # every scale is 1 at N = 1
        z = x.clone()
        p.transform_in_place(z, code)
        assert p.info()["last_launches"] == 0, code
        assert check_bits(z, x, "f32", P, f"{code.name} in place") is None
    p.close()


# ---- 2. Bluestein: every inner size ---------------------------------------------------------------------------------

def _primes_in(lo, hi):
    for n in range(hi, lo - 1, -1):
        if n > 1 and all(n % q for q in range(2, int(n ** 0.5) + 1)):
            return n
    return None


def bluestein_sizes(m):
    """non-smooth N with inner size m: the smallest, the largest and a prime"""
    lo, hi = m // 4 + 1, m // 2
    ns = [n for n in range(lo, min(hi, lo + 64) + 1) if not smooth(n)][:1]
    ns += [n for n in range(hi, max(lo, hi - 64) - 1, -1) if not smooth(n)][:1]
    prime = _primes_in(lo, hi)
    return sorted(set(ns + ([prime] if prime else [])))


BLUE_M = {"f32": [1 << k for k in range(4, 21)], "f64": [1 << k for k in range(4, 19)]}
BLUE_CASES = [(r, m) for r in ("f32", "f64") for m in BLUE_M[r]]


@pytest.mark.parametrize("real,m", BLUE_CASES, ids=[f"{r}-M{m}" for r, m in BLUE_CASES])
def test_bluestein_inner_size(real, m):
    ns = bluestein_sizes(m)
    if m <= 128:   # every non-smooth N <= 64
        ns = sorted(set(ns) | {n for n in range(m // 4 + 1, m // 2 + 1) if n <= 64 and not smooth(n)})
    if real == "f32" and m == 1 << 14:
        ns = sorted(set(ns) | {4099})      # inner persistent plan
    if real == "f64" and m == 1 << 13:
        ns = sorted(set(ns) | {2053})
    for n in ns:
        assert bluestein_m(n) == m
        batches = [1, 3, P] if n * P <= 8 * MIB else [2]
        wrap = grid_wrapping_batch(real, n) if n == ns[-1] else None
        check_size(real, n, batches + ([wrap] if wrap else []), tag=f", grid-wrapping batch {wrap}" if wrap else "")


# ---- 3. chunk loops ---------------------------------------------------------------------------------------------------

def launches(p, x, code=T.Fft):
    p.transform(x, poisoned_like(x), code)
    return p.info()["last_launches"]


def check_chunked(real, n, batch, chunk):
    """The standard check (Fft) on a batch that the library splits into chunks of `chunk`; last_launches must count
    every chunk."""
    assert batch > chunk
    p = make_plan(real, n)
    require(5 * batch * n * ESIZE[real], f"{real} N={n} batch {batch}")
    x, base = periodic_input(real, n, batch, FIRST)
    decoy, _ = periodic_input(real, n, batch, DECOY)
    failures = []
    worst, f, got = check_batch(p, real, n, x, Refs(base), T.Fft, bound(real, n), f"Fft batch {batch}", decoy)
    failures += f
    del decoy
    full, rest = divmod(batch, chunk)
    want = full * launches(p, x[:chunk]) + (launches(p, x[:rest]) if rest else 0)
    assert got == want, f"{real} N={n} batch {batch}: {got} launches, {full} chunks of {chunk} + {rest} need {want}"
    print(f"\n{real} N={n} {p.info()['path_name']}: batch {batch} in chunks of {chunk}, {got} launches, worst "
          f"per-transform error {worst:.2e}", end="")
    p.close()
    assert not failures, "\n  ".join(failures)


@pytest.mark.parametrize("real,n", [("f32", 19683), ("f64", 7776)])
def test_global_stages_scratch_chunks(real, n):
    chunk = SCRATCH // (n * ESIZE[real])
    check_chunked(real, n, 2 * chunk + 7, chunk)


@pytest.mark.parametrize("real,n,batch", [("f32", 1500001, 17), ("f64", 100003, 129)])
def test_unfused_bluestein_scratch_chunks(real, n, batch):
    check_chunked(real, n, batch, SCRATCH // (bluestein_m(n) * ESIZE[real]))


# ---- 4. three-pass powers of two -------------------------------------------------------------------------------------

THREEPASS_CASES = [(r, 1 << k) for r in ("f32", "f64") for k in THREEPASS[r]]
LD_LIMIT = {"f32": 1 << 25, "f64": 1 << 22}   # largest size checked against a long-double FFT


def closed_form_inputs(real, n):
    """-> device batch of 2: an impulse at an odd n0 in the top half, and three tones (integer frequencies f with
    amplitudes a: x[j] = sum a exp(+2 pi i f j / N), spectrum N a at bin f, 0 elsewhere)"""
    n0 = n - n // 3 | 1
    x = torch.zeros((2, n), dtype=TDT[real], device="cuda")
    x[0, n0] = 1
    tones = [(3, 0.5), (n // 2 + 12345, -0.25j), (n - 7, 0.125 + 0.125j)]
    step = 1 << 24
    for j0 in range(0, n, step):
        j = torch.arange(j0, min(n, j0 + step), device="cuda", dtype=torch.int64)
        acc = torch.zeros(j.numel(), dtype=torch.complex128, device="cuda")
        for f, a in tones:
            ang = (2 * math.pi / n) * ((j * f) % n).to(torch.float64)
            acc += a * torch.polar(torch.ones_like(ang), ang)
        x[1, j0:j0 + j.numel()] = acc.to(TDT[real])
    return x, n0, tones


def closed_form_errors(y, real, n, n0, tones):
    """per-transform errors of the two closed-form rows; the impulse's spectrum w_N^{(k n0) mod N} is evaluated with the
    index reduced exactly in int64, in float64 on the device (f32) or in long double on the host (f64)"""
    step = 1 << 24
    e_imp = e_tone = 0.0
    peak = max(abs(n * a) for _, a in tones)
    for k0 in range(0, n, step):
        k = torch.arange(k0, min(n, k0 + step), device="cuda", dtype=torch.int64)
        d = y[1, k0:k0 + k.numel()].to(torch.complex128)
        for f, a in tones:
            if k0 <= f < k0 + k.numel():
                d[f - k0] -= n * a
        e_tone = max(e_tone, d.abs().max().item() / peak)
        r = (k * n0) % n
        if real == "f32":
            ang = (-2 * math.pi / n) * r.to(torch.float64)
            ref = torch.polar(torch.ones_like(ang), ang)
            e_imp = max(e_imp, (y[0, k0:k0 + k.numel()].to(torch.complex128) - ref).abs().max().item())
        else:
            ang = np.longdouble(-2) * np.arccos(np.longdouble(-1)) * r.cpu().numpy().astype(np.longdouble) / n
            ref = np.cos(ang) + 1j * np.sin(ang)
            got = y[0, k0:k0 + k.numel()].cpu().numpy().astype(np.clongdouble)
            e_imp = max(e_imp, float(np.abs(got - ref).max()))
    return e_imp, e_tone


@pytest.mark.parametrize("real,n", THREEPASS_CASES, ids=[f"{r}-2^{log2(n)}" for r, n in THREEPASS_CASES])
def test_threepass_power_of_two(real, n):
    p = make_plan(real, n)
    row = n * ESIZE[real]
    work = max(row, min(2 * row, BIG_CHUNK // row * row))   # exec_bigpow2's intermediate at batch 2
    if torch.cuda.mem_get_info()[0] >= 9 * row + work + GIB:
        batch = 2
    else:
        batch = 1
        require(4 * row + work, f"{real} N=2^{log2(n)}")
    tol = bound(real, n)
    failures = []
    if n <= LD_LIMIT[real]:
        x, base = periodic_input(real, n, batch, FIRST)
        worst, failures, _ = check_batch(p, real, n, x, Refs(base), T.Fft, tol, f"Fft batch {batch}")
        what = f"long-double reference, worst {worst:.2e}"
        del x
    else:
        # random input: in place and batch 1, bit for bit
        x = device_input(real, batch, n, FIRST)
        out = run(p, x, T.Fft)
        p.transform_in_place(x, T.Fft)
        failures += [m for m in [check_bits(x, out, real, P, "in place vs out of place")] if m]
        fb.fill_input(x, first_transform=FIRST)   # the same rows again
        single = torch.empty((1, n), dtype=TDT[real], device="cuda")
        for b in range(batch):
            single.fill_(complex(float("nan"), float("nan")))
            p.transform(x[b:b + 1], single, T.Fft)
            failures += [m for m in [check_bits(out[b:b + 1], single, real, P, f"row {b}: batch {batch} vs 1")] if m]
        del x, out, single
        # closed-form inputs against their exact spectra, as one batch of 2 (at f32 2^30: 2^31 elements)
        require(5 * row + work, f"{real} N=2^{log2(n)} closed-form batch of 2")
        x, n0, tones = closed_form_inputs(real, n)
        y = run(p, x, T.Fft)
        del x
        e_imp, e_tone = closed_form_errors(y, real, n, n0, tones)
        del y
        what = f"impulse at {n0}: {e_imp:.2e}, tones: {e_tone:.2e}"
        failures += [f"{what} (tol {tol:.0e})"] if not (e_imp <= tol and e_tone <= tol) else []
    torch.cuda.synchronize()
    print(f"\n{real} N=2^{log2(n)} {p.kernel_name()}: batch {batch}, {what}", end="")
    p.close()
    assert not failures, f"{real} N=2^{log2(n)}:\n  " + "\n  ".join(failures)


@pytest.mark.parametrize("real,n,batch", [("f32", 1 << 28, 3), ("f64", 1 << 24, 9)])
def test_threepass_outer_chunks(real, n, batch):
    """the outer loop of exec_bigpow2 (2 GiB of intermediate per chunk): every transform equals its batch-1 result"""
    p = make_plan(real, n)
    row = n * ESIZE[real]
    chunk = max(1, BIG_CHUNK // row)
    assert batch > chunk
    require((4 * batch + 1) * row + BIG_CHUNK, f"{real} N=2^{log2(n)} batch {batch}")
    x = device_input(real, batch, n, FIRST)
    out = run(p, x, T.Fft, device_input(real, batch, n, DECOY))
    got = p.info()["last_launches"]
    failures = []
    bad = torch.isnan(torch.view_as_real(out)).flatten(1).any(dim=1).nonzero().flatten().tolist()
    failures += [f"rows {bad} hold NaN (never stored)"] if bad else []
    single = torch.empty((1, n), dtype=TDT[real], device="cuda")
    one = None
    for b in range(batch):
        single.fill_(complex(float("nan"), float("nan")))
        p.transform(x[b:b + 1], single, T.Fft)
        one = p.info()["last_launches"]
        failures += [m for m in [check_bits(out[b:b + 1], single, real, P, f"row {b}: batch {batch} vs 1")] if m]
    full, rest = divmod(batch, chunk)
    want = full * launches(p, x[:chunk]) + (one if rest else 0) if chunk > 1 else batch * one
    assert got == want, f"{got} launches for {-(-batch // chunk)} chunks of {chunk}, expected {want}"
    print(f"\n{real} N=2^{log2(n)}: batch {batch} in chunks of {chunk}, {got} launches", end="")
    p.close()
    assert not failures, "\n  ".join(failures)


# ---- 5. host-pointer pipeline ---------------------------------------------------------------------------------------

def host_path(n, real, batch):
    b = batch * n * ESIZE[real]
    return "zero-copy" if b <= ZERO_COPY else "single stream" if b <= SINGLE else "pipeline"


def expected_host_launches(p, x, real, n):
    """launches of a host call on x: the pipeline's chunks, each run as a device call of its size"""
    batch = x.shape[0]
    if host_path(n, real, batch) != "pipeline":
        return launches(p, x)
    chunk = min(batch, max(1, HOST_CHUNK // (n * ESIZE[real])))
    return sum(launches(p, x[b0:b0 + chunk]) for b0 in range(0, batch, chunk))


def _bits_equal(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return np.array_equal(a.view(np.uint8), b.view(np.uint8))


# (precision, N, batches in call order): a large call first, then the batches on both sides of the zero-copy (64 KiB)
# and single-stream (1 MiB) thresholds on the same plan
HOST_CASES = [
    ("f32", 1 << 20, [59]),                     # 8 chunks of 8 through 3 slots, the last one partial
    ("f32", 4099, [4 * 2046 + 1, 1, 2, 31, 32]),   # unfused Bluestein: 5 chunks of 2046, the fifth holds one transform
    ("f32", 1 << 13, [1, 2, 16, 17]),           # batch 1: the persistent kernel's TMA on a mapped host buffer
    ("f64", 1536, [3000, 2, 3, 42, 43]),
    ("f64", 1 << 16, [9, 1]),
]


@pytest.mark.parametrize("real,n,batches", HOST_CASES, ids=[f"{r}-{n}" for r, n, _ in HOST_CASES])
def test_host_pipeline(real, n, batches):
    p = make_plan(real, n)
    top = max(batches)
    require(4 * top * n * ESIZE[real], f"{real} N={n} batch {top}")
    x, base = periodic_input(real, n, top, FIRST)
    refs = Refs(base)
    failures = []
    for batch in batches:
        xb = x[:batch]
        path = host_path(n, real, batch)
        for code in (T.Fft, T.SqrtScaledIfft):
            what = f"{code.name} batch {batch} ({path})"
            if batch == top:
                _, f, _ = check_batch(p, real, n, xb, refs, code, bound(real, n), what, single=False, in_place=False)
                failures += f
            want = run(p, xb, code).cpu().numpy()
            calls = expected_host_launches(p, xb, real, n)
            pinned = xb.cpu().pin_memory()
            sources = {"pinned torch": (pinned, poisoned_like(pinned).pin_memory()),
                       "pageable numpy": (xb.cpu().numpy(), poisoned_like(xb.cpu().numpy()))}
            for kind, (src, dst) in sources.items():
                p.transform(src, dst, code)
                got = p.info()["last_launches"]
                ok = _bits_equal(dst.numpy() if torch.is_tensor(dst) else dst, want)
                failures += [] if ok else [f"{what}, {kind} out of place: differs from the device call"]
                failures += [] if got == calls else [f"{what}, {kind}: {got} launches, expected {calls}"]
                z = src.clone() if torch.is_tensor(src) else src.copy()
                if torch.is_tensor(z):
                    z = z.pin_memory()
                p.transform_in_place(z, code)
                ok = _bits_equal(z.numpy() if torch.is_tensor(z) else z, want)
                failures += [] if ok else [f"{what}, {kind} in place: differs from the device call"]
    torch.cuda.synchronize()
    print(f"\n{real} N={n} {p.kernel_name()}: host batches {[(b, host_path(n, real, b)) for b in batches]}", end="")
    p.close()
    assert not failures, f"{real} N={n}:\n  " + "\n  ".join(failures)

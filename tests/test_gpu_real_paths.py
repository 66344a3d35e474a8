"""Every real-input path checked transform by transform: the fused on-chip kernels (N = 2L) at batches that wrap their
grid, the half-length path (other even N) over every inner complex plan, the full-length path (odd N) over every inner
plan with an exact oracle, the scratch chunk loops and grid caps of both, the host staging of rfft, irfft, convolve
and dct, and every fused family kernel (conv, lconv, stft, dct, mel, mfcc, welch, csd, coherence) past one grid sweep.

Every case runs the method of test_gpu_complex_paths.py on a periodic batch: row b is 2^s(b) * base[b mod 97], s(b)
cycling over -24 .. 24, for the linear operations (rfft, irfft, conv, lconv, stft, dct), and base[b mod 97] for the
others.  So

  1. only the base rows need a reference: numpy in long double for rfft / irfft (the family's own reference function
     elsewhere), held to the bound of the path;
  2. every other row is checked bit for bit against its base row, after unscaling;
  3. outputs start as NaN and a decoy call on other input runs first;
  4. the base rows of the batch equal the same rows run one at a time from a fresh allocation, bit for bit;
  5. the plan runs the path the case is meant for (path_name, inner_path_name, kernel_name()), with the launch count
     of that path: one launch fused, and per scratch chunk the inner plan's launches plus 1 (half) or 2 (full).

Per-transform bounds: fused 2e-6 (f32) / 5e-15 (f64); half the inner complex path's bound plus 1e-6 / 5e-15 for the
untangle; full the inner complex path's bound, as the full path is exactly the complex transform of x + 0i.  Transforms
too large for a long-double reference are checked on closed-form inputs.  Cases that do not fit the free device memory
are skipped with the reason."""
import math

import numpy as np
import pytest
import torch

import fourier_b200 as fb
import test_gpu_conv as conv_mod
import test_gpu_csd as csd_mod
import test_gpu_dct as dct_mod
import test_gpu_lconv as lconv_mod
import test_gpu_mel as mel_mod
import test_gpu_mfcc as mfcc_mod
import test_gpu_stft as stft_mod
import test_gpu_welch as welch_mod
from helpers import per_transform_err
from test_gpu_complex_paths import (BLUE_M, ESIZE, HOST_CHUNK, LD_LIMIT, MIB, ONCHIP, ONCHIP_TP, P, SCRATCH,
                                    SMOOTH, TDT, THREEPASS, TWOPASS, bluestein_m, bound, expected_path, exponents, log2,
                                    pow2, require, smooth)
from test_gpu_real import scale_code, truth_irfft, truth_rfft

pytestmark = pytest.mark.gpu

T = fb.Transform
RDT = {"f32": torch.float32, "f64": torch.float64}
NPR = {"f32": np.float32, "f64": np.float64}
NPC = {"f32": np.complex64, "f64": np.complex128}
FUSED_BOUND = {"f32": 2e-6, "f64": 5e-15}
UNTANGLE = {"f32": 1e-6, "f64": 5e-15}   # the half path's allowance for the untangle / tangle step
WARPS = 8                                # warps per CTA of every on-chip size class (onchip_configs.cuh)
FUSED_N = {"f32": [2 * l for l in sorted(ONCHIP["f32"])], "f64": [2 * l for l in sorted(ONCHIP["f64"])]}
REF_SAMPLES = 1 << 22                    # long-double references on at most this many samples (at least 2 rows)

WORST = {}   # (precision, path) -> (worst per-transform error, bound) over the cases run


def note(prec, path, worst, tol):
    w, t = WORST.get((prec, path), (0.0, tol))
    WORST[(prec, path)] = (max(w, worst), min(t, tol))


# ---- the real plan's selection rules (RealPlan<T>::init) -----------------------------------------------------------

def expected_real_path(prec, n):
    """-> (path_name, inner size, inner_path_name, kernel_name() prefix, inner kernel fragment)"""
    if n % 2 == 0 and n // 2 in ONCHIP[prec]:
        return "real_fused", 0, "trivial", "onchip::onchip_real_kernel", ""
    if n % 2 == 0:
        path, _, kernel = expected_path(prec, n // 2)
        return "real_half", n // 2, path, "real::untangle_kernel / real::tangle_kernel + ", kernel
    path, _, kernel = expected_path(prec, n)
    return "real_full", n, path, "real::widen_kernel / real::hermitian_kernel + ", kernel


def real_plan(prec, n):
    p = fb.create_rfft_f32(n) if prec == "f32" else fb.create_rfft_f64(n)
    path, inner, inner_path, prefix, fragment = expected_real_path(prec, n)
    info, name = p.info(), p.kernel_name()
    got = (info["path_name"], info["inner_size"], info["inner_path_name"])
    assert got == (path, inner, inner_path) and name.startswith(prefix) and fragment in name, \
        f"{prec} N={n}: plan runs {got} / {name!r}, expected {(path, inner, inner_path)} / {prefix}...{fragment!r}"
    return p


def real_bound(prec, n):
    path, inner = expected_real_path(prec, n)[:2]
    if path == "real_fused":
        return FUSED_BOUND[prec]
    return bound(prec, inner) + (UNTANGLE[prec] if path == "real_half" else 0.0)


def scratch_chunk(total, item_bytes):
    """real.cu scratch_chunk: items of item_bytes in one chunk of plan scratch"""
    return min(total, max(1, SCRATCH // item_bytes))


def chunks(total, size):
    return [min(size, total - b0) for b0 in range(0, total, size)]


_INNER = {}


def inner_launches(prec, n, batch, code, in_place):
    """launches of the complex plan of length n on `batch` rows, as the real paths call it"""
    key = (prec, n, batch, int(code), in_place)
    if key not in _INNER:
        c = fb.create_fft_f32(n) if prec == "f32" else fb.create_fft_f64(n)
        z = torch.zeros((batch, n), dtype=TDT[prec], device="cuda")
        if in_place:
            c.transform_in_place(z, code)
        else:
            c.transform(z, torch.empty_like(z), code)
        _INNER[key] = c.info()["last_launches"]
        c.close()
        del z
    return _INNER[key]


def expected_launches(prec, n, fwd, batch, code):
    """rfft / irfft: 1 fused; per scratch chunk the inner plan's launches + 1 (half: Fft or UnscaledIfft, out of place)
    or + 2 (full: the call's code, in place)"""
    path, inner = expected_real_path(prec, n)[:2]
    if path == "real_fused":
        return 1
    total = 0
    for nb in chunks(batch, scratch_chunk(batch, inner * ESIZE[prec])):
        if path == "real_half":
            total += inner_launches(prec, inner, nb, T.Fft if fwd else T.UnscaledIfft, False) + 1
        else:
            total += inner_launches(prec, inner, nb, code, True) + 2
    return total


def conv_launches(prec, n, batch):
    """convolve: 1 fused; the inner Fft, the pair step and the inner UnscaledIfft over the whole batch (half); per
    scratch chunk the inner Fft and UnscaledIfft in place + 3 (full)"""
    path, inner = expected_real_path(prec, n)[:2]
    if path == "real_fused":
        return 1
    if path == "real_half":
        return inner_launches(prec, inner, batch, T.Fft, False) + inner_launches(prec, inner, batch, T.UnscaledIfft,
                                                                                  True) + 1
    return sum(inner_launches(prec, n, nb, T.Fft, True) + inner_launches(prec, n, nb, T.UnscaledIfft, True) + 3
               for nb in chunks(batch, scratch_chunk(batch, n * ESIZE[prec])))


def fused_wrap(prec, n):
    """(C, grid) of the fused class of real length n (onchip.cu launch): groups of C = WARPS*32 / (L/E) transforms,
    at most sms * MINB * 4 CTAs; and the number of transforms of about 1.3 grid sweeps, ending in a partial group"""
    l = n // 2
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    c = WARPS * 32 // ONCHIP_TP[l]
    grid = sms * ONCHIP[prec][l] * 4
    return c, grid, int(1.3 * grid) * c + c // 2


# ---- periodic, scaled batches ---------------------------------------------------------------------------------------

def as_real(t):
    return torch.view_as_real(t) if t.is_complex() else t


def _step(t):
    """rows of t per temporary of about 64 MiB"""
    return max(1, (64 * MIB) // max(1, t[0].numel() * t.element_size() * 2))


def periodic(base, batch, prec, scale=True):
    """row b = 2^s(b) * base[b mod q] (q = rows of base), or base[b mod q] unscaled, on the device"""
    base = torch.as_tensor(base).cuda()
    q = base.shape[0]
    x = torch.empty((batch,) + tuple(base.shape[1:]), dtype=base.dtype, device="cuda")
    xr, br = as_real(x), as_real(base)
    for r0 in range(0, batch, _step(x)):
        rows = torch.arange(r0, min(batch, r0 + _step(x)), device="cuda")
        src = br[rows % q]
        if scale:
            src = src * pow2(exponents(rows), prec).view((-1,) + (1,) * (br.dim() - 1))
        xr[r0:r0 + rows.numel()] = src
    return x


def unscaled(y, prec, r0, r1, scale=True):
    v = as_real(y[r0:r1])
    if not scale:
        return v
    rows = torch.arange(r0, r1, device="cuda")
    return v * pow2(-exponents(rows), prec).view((-1,) + (1,) * (v.dim() - 1))


def bits(t):
    r = as_real(t).contiguous()
    return r.view(torch.int32 if r.element_size() == 4 else torch.int64)


def differing_rows(a, b):
    return torch.nonzero((bits(a) != bits(b)).flatten(1).any(dim=1)).flatten().tolist()


def periodic_mismatch(y, prec, q=P, scale=True):
    """-> the rows b >= q whose unscaled bits differ from those of row b mod q"""
    batch = y.shape[0]
    if batch <= q:
        return []
    base = bits(unscaled(y, prec, 0, q, scale)).flatten(1)
    bad = []
    for r0 in range(q, batch, _step(y)):
        r1 = min(batch, r0 + _step(y))
        u = bits(unscaled(y, prec, r0, r1, scale)).flatten(1)
        diff = (u != base[torch.arange(r0, r1, device="cuda") % q]).any(dim=1)
        bad += (torch.nonzero(diff).flatten() + r0).tolist()
    return bad


def host_rows(y, prec, rows, scale=True):
    """the first `rows` rows of y, unscaled, as a numpy array of y's kind"""
    u = unscaled(y, prec, 0, rows, scale).contiguous()
    return (torch.view_as_complex(u) if y.is_complex() else u).cpu().numpy()


def nan(shape, dtype):
    return torch.full(shape, complex(float("nan"), float("nan")) if dtype.is_complex else float("nan"), dtype=dtype,
                      device="cuda")


def ref_rows(q, n):
    """base rows that get a reference: all q, or as many as REF_SAMPLES allows (at least 2)"""
    return min(q, max(2, REF_SAMPLES // max(1, n)))


def check_rows(p, prec, run, x, ref, tol, q=P, scale=True, decoy=None, single=True, absolute=False, what=""):
    """The standard check of one call: run(x, first) -> a fresh output whose row b is the result of row b of x (row
    first + b of the whole batch).  `ref` holds the reference of the first ref.shape[0] unscaled base rows.
    -> (worst error, failures, launches of the call, output)"""
    batch = x.shape[0]
    rows = min(q, batch)
    if decoy is not None:
        run(decoy, 0)
    y = run(x, 0)
    launched = p.info()["last_launches"]
    failures = []
    nref = min(rows, ref.shape[0])
    got = host_rows(y, prec, nref, scale).reshape(nref, -1)
    want = np.asarray(ref[:nref]).reshape(nref, -1)
    if absolute:
        e = np.abs(got.astype(np.float64) - want.astype(np.float64)).max(axis=1)
        err = np.where(np.isnan(e), np.inf, e)
    else:
        err = per_transform_err(got, want)
    worst = float(err.max())
    bad = np.nonzero(~(err <= tol))[0]
    if bad.size:
        failures.append(f"{what}: {bad.size} of {nref} base rows off the reference (tol {tol:.0e}, worst {worst:.2e}): "
                        f"rows {bad[:8].tolist()}")
    bad = periodic_mismatch(y, prec, q, scale)
    if bad:
        failures.append(f"{what}: {len(bad)} of {batch - q} rows beyond the base rows differ from their base row: rows "
                        f"{bad[:8]}, b mod {q} = {[b % q for b in bad[:8]]}")
    if single:
        alone = [b for b in range(rows) if differing_rows(run(x[b:b + 1].clone(), b), y[b:b + 1])]
        if alone:
            failures.append(f"{what}: base rows {alone[:8]} differ from the same row run alone")
    return worst, failures, launched, y


# ---- rfft / irfft ---------------------------------------------------------------------------------------------------

def rfft_run(p, prec, code):
    def run(x, first):
        y = nan((x.shape[0], p.size() // 2 + 1), TDT[prec])
        p.rfft(x, y, code)
        return y
    return run


def irfft_run(p, prec, code):
    def run(x, first):
        y = nan((x.shape[0], p.size()), RDT[prec])
        p.irfft(x, y, code)
        return y
    return run


def base_reals(prec, rows, n, seed):
    return np.random.default_rng(seed).standard_normal((rows, n)).astype(NPR[prec])


def base_spectra(prec, rows, n, seed):
    """random bins, imaginary parts of bins 0 and N/2 included (the transform ignores them, as numpy's irfft does)"""
    rng = np.random.default_rng(seed)
    b = n // 2 + 1
    return (rng.standard_normal((rows, b)) + 1j * rng.standard_normal((rows, b))).astype(NPC[prec])


def full_oracle(prec, n, fwd, x, code):
    """The full path computed by the complex plan of length n: forward, bins 0 .. N/2 of the transform of x + 0i (bin
    0's imaginary part stored as +0); inverse, the real parts of the transform of the Hermitian extension (real::
    hermitian: bin 0 with its imaginary part ignored, bins k <= N/2 as given, bins k > N/2 conj(x[N-k]))."""
    c = fb.create_fft_f32(n) if prec == "f32" else fb.create_fft_f64(n)
    bins = n // 2 + 1
    if fwd:
        z = torch.complex(x, torch.zeros_like(x))
    else:
        z = torch.empty((x.shape[0], n), dtype=TDT[prec], device="cuda")
        z[:, 0] = torch.complex(x[:, 0].real, torch.zeros_like(x[:, 0].real))
        z[:, 1:bins] = x[:, 1:bins]
        z[:, bins:] = torch.conj_physical(x[:, 1:n - bins + 1].flip(-1))
    y = nan(z.shape, TDT[prec])
    c.transform(z, y, code)
    c.close()
    if fwd:
        want = y[:, :bins].clone()
        want[:, 0] = torch.complex(want[:, 0].real, torch.zeros_like(want[:, 0].real))
        return want
    return y.real.contiguous()


def check_real_size(prec, n, batches, codes_at=(P,), tag=""):
    """The standard check of rfft and irfft of length n at each batch: Fft and Ifft, every code at the batches in
    codes_at; on the full path also the exact oracle of the complex plan."""
    p = real_plan(prec, n)
    path = expected_real_path(prec, n)[0]
    tol = real_bound(prec, n)
    top = max(batches)
    bins = n // 2 + 1
    require(4 * top * n * ESIZE[prec] + (top * n * ESIZE[prec] * 2 if path == "real_full" else 0),
            f"{prec} N={n} batch {top}")
    q = min(P, top)
    nref = ref_rows(q, n)
    xf_base, xi_base = base_reals(prec, q, n, n), base_spectra(prec, q, n, n + 1)
    refs = {True: truth_rfft(xf_base[:nref], 0), False: truth_irfft(xi_base[:nref], n, 2)}
    xs = {True: periodic(torch.from_numpy(xf_base), top, prec), False: periodic(torch.from_numpy(xi_base), top, prec)}
    failures, worst = [], 0.0
    for batch in batches:
        codes = list(T) if batch in codes_at else [T.Fft, T.Ifft]
        for code in codes:
            fwd = code.is_forward()
            x = xs[fwd][:batch]
            run = (rfft_run if fwd else irfft_run)(p, prec, code)
            what = f"{code.name} batch {batch}"
            decoy = torch.randn_like(x)
            w, f, launched, y = check_rows(p, prec, run, x, scale_code(refs[fwd], int(code), n), tol, decoy=decoy,
                                           what=what)
            del decoy
            worst, failures = max(worst, w), failures + f
            want = expected_launches(prec, n, fwd, batch, code)
            if launched != want:
                failures.append(f"{what}: {launched} launches, expected {want}")
            if path == "real_full":
                rows = differing_rows(y, full_oracle(prec, n, fwd, x, code))
                if rows:
                    failures.append(f"{what}: rows {rows[:8]} differ from the complex plan's transform")
            del y
    torch.cuda.synchronize()
    note(prec, path, worst, tol)
    print(f"\n{prec} N={n} {path} / {p.info()['inner_path_name']} {p.kernel_name()}{tag}: batches {batches}, worst "
          f"per-transform error {worst:.2e} (bound {tol:.0e})", end="")
    p.close()
    assert not failures, f"{prec} N={n}:\n  " + "\n  ".join(failures)


# ---- 1. fused classes at grid-wrapping batches ----------------------------------------------------------------------

FUSED_CASES = [(r, n) for r in ("f32", "f64") for n in FUSED_N[r]]


@pytest.mark.parametrize("prec,n", FUSED_CASES, ids=[f"{r}-{n}" for r, n in FUSED_CASES])
def test_fused_class(prec, n):
    c, grid, wrap = fused_wrap(prec, n)
    check_real_size(prec, n, [1, 3, P, wrap], tag=f", {wrap} rows = {-(-wrap // c)} groups of {c} on {grid} CTAs")


# ---- 2. half-length path over every inner plan -----------------------------------------------------------------------

def half_bluestein_sizes(m_inner):
    """one odd and one even non-smooth m with Bluestein inner size m_inner (none even at 16)"""
    span = range(m_inner // 4 + 1, m_inner // 2 + 1)
    odd = [m for m in span if m % 2 and not smooth(m)][:1]
    even = [m for m in span if m % 2 == 0 and not smooth(m)][:1]
    return odd + even


HALF_SMOOTH = [(r, m) for r in ("f32", "f64") for m in SMOOTH if m not in ONCHIP[r]]
HALF_BLUE = [(r, mi) for r in ("f32", "f64") for mi in BLUE_M[r]]
POW2_TOP = {"f32": 26, "f64": 23}
HALF_POW2 = [(r, k) for r in ("f32", "f64") for k in sorted(set(TWOPASS[r]) | set(THREEPASS[r]))
             if (1 << k) > max(SMOOTH) and k <= POW2_TOP[r]]


def small_batches(n):
    return [1, 3, P] if n * P <= 8 * MIB else [2]


@pytest.mark.parametrize("prec,m", HALF_SMOOTH, ids=[f"{r}-M{m}" for r, m in HALF_SMOOTH])
def test_half_smooth(prec, m):
    check_real_size(prec, 2 * m, small_batches(2 * m))


@pytest.mark.parametrize("prec,m_inner", HALF_BLUE, ids=[f"{r}-B{mi}" for r, mi in HALF_BLUE])
def test_half_bluestein(prec, m_inner):
    for m in half_bluestein_sizes(m_inner):
        assert bluestein_m(m) == m_inner
        check_real_size(prec, 2 * m, small_batches(2 * m))


def closed_form(prec, n):
    """-> device reals (2, n): an impulse at an odd n0 and three cosines a cos(2 pi f j / n) with integer f < n/2, and
    the spectrum (1, n/2+1) of the cosines (n a / 2 at bin f, 0 elsewhere)"""
    n0 = (n - n // 3) | 1
    tones = [(3, 0.5), (n // 4 + 12345, -0.25), (n // 2 - 7, 0.125)]
    x = torch.zeros((2, n), dtype=RDT[prec], device="cuda")
    x[0, n0] = 1
    step = 1 << 24
    for j0 in range(0, n, step):
        x[1, j0:j0 + step] = tone_signal(n, tones, j0, min(n, j0 + step)).to(RDT[prec])
    spec = torch.zeros((1, n // 2 + 1), dtype=TDT[prec], device="cuda")
    for f, a in tones:
        spec[0, f] = n * a / 2
    return x, spec, n0, tones


def tone_signal(n, tones, j0, j1):
    j = torch.arange(j0, j1, device="cuda", dtype=torch.int64)
    acc = torch.zeros(j.numel(), dtype=torch.float64, device="cuda")
    for f, a in tones:
        acc += a * torch.cos((2 * math.pi / n) * ((j * f) % n).to(torch.float64))
    return acc


def closed_form_errors(prec, n, y, r, n0, tones):
    """per-transform errors of the impulse's and the tones' spectra (y), and of the tones' inverse (r)"""
    step = 1 << 24
    bins = n // 2 + 1
    peak = max(abs(n * a / 2) for _, a in tones)
    e_imp = e_tone = e_inv = 0.0
    for k0 in range(0, bins, step):
        k = torch.arange(k0, min(bins, k0 + step), device="cuda", dtype=torch.int64)
        d = y[1, k0:k0 + k.numel()].to(torch.complex128)
        for f, a in tones:
            if k0 <= f < k0 + k.numel():
                d[f - k0] -= n * a / 2
        e_tone = max(e_tone, d.abs().max().item() / peak)
        ang_i = (k * n0) % n
        if prec == "f32":
            ang = (-2 * math.pi / n) * ang_i.to(torch.float64)
            e_imp = max(e_imp, (y[0, k0:k0 + k.numel()].to(torch.complex128) - torch.polar(torch.ones_like(ang), ang))
                        .abs().max().item())
        else:
            ang = np.longdouble(-2) * np.arccos(np.longdouble(-1)) * ang_i.cpu().numpy().astype(np.longdouble) / n
            got = y[0, k0:k0 + k.numel()].cpu().numpy().astype(np.clongdouble)
            e_imp = max(e_imp, float(np.abs(got - (np.cos(ang) + 1j * np.sin(ang))).max()))
    amp = sum(abs(a) for _, a in tones)
    for j0 in range(0, n, step):
        j1 = min(n, j0 + step)
        e_inv = max(e_inv, (r[0, j0:j1].to(torch.float64) - tone_signal(n, tones, j0, j1)).abs().max().item() / amp)
    return e_imp, e_tone, e_inv


@pytest.mark.parametrize("prec,k", HALF_POW2, ids=[f"{r}-M2^{k}" for r, k in HALF_POW2])
def test_half_power_of_two(prec, k):
    n = 2 << k
    if n <= LD_LIMIT[prec]:
        check_real_size(prec, n, small_batches(n))
        return
    p = real_plan(prec, n)
    tol = real_bound(prec, n)
    require(8 * n * ESIZE[prec], f"{prec} N=2^{log2(n)}")
    x, spec, n0, tones = closed_form(prec, n)
    failures = []
    y = rfft_run(p, prec, T.Fft)(x, 0)
    want = expected_launches(prec, n, True, 2, T.Fft)
    failures += [] if p.info()["last_launches"] == want else [f"forward: {p.info()['last_launches']} launches, "
                                                              f"expected {want}"]
    r = irfft_run(p, prec, T.Ifft)(spec, 0)
    want = expected_launches(prec, n, False, 1, T.Ifft)
    failures += [] if p.info()["last_launches"] == want else [f"inverse: {p.info()['last_launches']} launches, "
                                                              f"expected {want}"]
    for b in range(2):
        if differing_rows(rfft_run(p, prec, T.Fft)(x[b:b + 1].clone(), b), y[b:b + 1]):
            failures.append(f"row {b}: batch 2 differs from batch 1")
    e_imp, e_tone, e_inv = closed_form_errors(prec, n, y, r, n0, tones)
    what = f"impulse at {n0}: {e_imp:.2e}, tones: {e_tone:.2e}, tones inverse: {e_inv:.2e}"
    failures += [] if max(e_imp, e_tone, e_inv) <= tol else [f"{what} (tol {tol:.0e})"]
    torch.cuda.synchronize()
    note(prec, "real_half", max(e_imp, e_tone, e_inv), tol)
    print(f"\n{prec} N=2^{log2(n)} real_half / {p.info()['inner_path_name']} {p.kernel_name()}: {what} (bound "
          f"{tol:.0e})", end="")
    p.close()
    assert not failures, f"{prec} N=2^{log2(n)}:\n  " + "\n  ".join(failures)


HALF_INNER_KINDS = {("trivial", "scale_copy_kernel"), ("onchip_cta", "cta::cta_fft_kernel"),
                    ("twopass", "twopass::tile_kernel"), ("twopass", "fused::fused_twopass_kernel"),
                    ("threepass", "outer::column_kernel"), ("threepass", "outer::radix3_column_kernel"),
                    ("global_stages", "stockham_stage_kernel"), ("bluestein_fused", "onchip::bluestein_fused_kernel"),
                    ("bluestein_fused", "cta::cta_fft_kernel (chirp mode)"), ("bluestein", "chirp / pointwise kernels")}


def test_half_path_covers_every_inner_plan():
    """the inner (path, kernel) pairs of the sizes of this section, each confirmed on a plan"""
    ms = [(r, m) for r, m in HALF_SMOOTH] + [(r, m) for r, mi in HALF_BLUE for m in half_bluestein_sizes(mi)] + \
         [(r, 1 << k) for r, k in HALF_POW2]
    seen = set()
    for prec, m in ms:
        path, _, kernel = expected_path(prec, m)
        if (path, kernel) not in seen:
            real_plan(prec, 2 * m).close()   # asserts the plan runs them
            seen.add((path, kernel))
    print(f"\nhalf path inner plans: {sorted(seen)}; worst per path so far: "
          f"{ {k: f'{w:.2e} (bound {t:.0e})' for k, (w, t) in sorted(WORST.items())} }", end="")
    assert HALF_INNER_KINDS <= seen, f"not covered: {sorted(HALF_INNER_KINDS - seen)}"


# ---- 3. full-length path over every inner plan -----------------------------------------------------------------------

FULL_CASES = [("f32", 2187), ("f64", 2187),                  # onchip_cta
              ("f32", 19683), ("f64", 19683),                # global_stages (f64 3^8 still fits the CTA kernel)
              ("f32", 37), ("f64", 37), ("f32", 1009),       # warp Bluestein
              ("f32", 67), ("f64", 1009),                    # CTA-chirp Bluestein
              ("f32", 4099), ("f64", 2053),                  # unfused Bluestein, two-pass inner plan
              ("f32", 1048577)]                              # unfused Bluestein, three-pass inner plan
FULL_INNER_KINDS = {("onchip_cta", "cta::cta_fft_kernel"), ("global_stages", "stockham_stage_kernel"),
                    ("bluestein_fused", "onchip::bluestein_fused_kernel"),
                    ("bluestein_fused", "cta::cta_fft_kernel (chirp mode)"), ("bluestein", "chirp / pointwise kernels")}


@pytest.mark.parametrize("prec,n", FULL_CASES, ids=[f"{r}-{n}" for r, n in FULL_CASES])
def test_full_path(prec, n):
    check_real_size(prec, n, small_batches(n))


def test_full_path_covers_every_inner_plan():
    seen = {(expected_path(r, n)[0], expected_path(r, n)[2]) for r, n in FULL_CASES}
    inner3 = {expected_path(r, bluestein_m(n))[0] for r, n in FULL_CASES if expected_path(r, n)[0] == "bluestein"}
    print(f"\nfull path inner plans: {sorted(seen)}, Bluestein inner plans {sorted(inner3)}; worst per path so far: "
          f"{ {k: f'{w:.2e} (bound {t:.0e})' for k, (w, t) in sorted(WORST.items())} }", end="")
    assert FULL_INNER_KINDS <= seen and {"twopass", "threepass"} <= inner3, (sorted(seen), inner3)


# ---- 4. scratch chunk loops and grid caps -----------------------------------------------------------------------------

def test_half_scratch_chunk_off_16_bytes():
    """f32 odd M: the second chunk's rows start 8 bytes off a 16-byte boundary (N = 200006, M = 100003)"""
    n = 200006
    chunk = scratch_chunk(1 << 40, (n // 2) * ESIZE["f32"])
    assert chunk == 671 and chunk % 2 == 1
    check_real_size("f32", n, [673], codes_at=(), tag=f", scratch chunks of {chunk}")


def test_half_scratch_chunks_global_stages():
    n = 39366   # M = 3^9
    chunk = scratch_chunk(1 << 40, (n // 2) * ESIZE["f32"])
    assert chunk == 3409
    check_real_size("f32", n, [2 * chunk + 7], codes_at=(), tag=f", scratch chunks of {chunk}")


def conv_run(p, prec, H, f):
    """convolve with f spectrum rows H (device, (f, bins)): row b of a batch uses row b mod f; a single row `first`
    alone uses H[first mod f]"""
    def run(x, first):
        y = nan(x.shape, RDT[prec])
        if x.shape[0] == 1:
            p.convolve(x, H[first % f].clone(), y)   # a spectrum row of an odd f32 bin count is not 16-byte aligned
        else:
            n = x.shape[-1]
            p.convolve(x.view(-1, f, n), H, y.view(-1, f, n))
        return y
    return run


def check_convolve(prec, n, batch, f, host=False, tag=""):
    """The standard check of convolve with f spectrum rows on a periodic batch (period lcm(97, f)), its launch count,
    and with host=True the same call staged from host memory (numpy and pinned torch), bit for bit"""
    assert batch % f == 0
    p = real_plan(prec, n)
    require(5 * batch * n * ESIZE[prec], f"{prec} N={n} batch {batch}")
    q = min(batch, P * f)
    xb = base_reals(prec, q, n, 7 * n)
    H = torch.from_numpy(conv_mod.spectra(prec, (f,), n, 7 * n + 1)).cuda()
    nref = ref_rows(q, n) // f * f or f
    ref = conv_mod.truth(xb[:nref].reshape(-1, f, n), H.cpu().numpy(), n).reshape(nref, n)
    x = periodic(torch.from_numpy(xb), batch, prec)
    run = conv_run(p, prec, H, f)
    tol = conv_mod.TOL[prec]
    worst, failures, launched, y = check_rows(p, prec, run, x, ref, tol, q=q, decoy=torch.randn_like(x),
                                              what=f"convolve batch {batch}, {f} spectra")
    want = conv_launches(prec, n, batch)
    failures += [] if launched == want else [f"{launched} launches, expected {want}"]
    if host:
        failures += host_calls(p, lambda src, dst: p.convolve(src.reshape(-1, f, n), H.cpu().numpy() if isinstance(
            src, np.ndarray) else H.cpu().pin_memory(), dst.reshape(-1, f, n)), x, y, n * ESIZE[prec] // 2,
            n * ESIZE[prec] // 2, lambda nb: (p.convolve(x[:nb], H[0], nan((nb, n), RDT[prec])),
                                               p.info()["last_launches"])[1], "convolve")
    torch.cuda.synchronize()
    print(f"\n{prec} N={n} {p.info()['path_name']} / {p.info()['inner_path_name']}: convolve batch {batch} with {f} "
          f"spectra, {launched} launches, worst error {worst:.2e} (tol {tol:.0e}){tag}", end="")
    p.close()
    assert not failures, f"{prec} N={n}:\n  " + "\n  ".join(failures)


def full_chunk_size(n):
    return scratch_chunk(1 << 40, n * ESIZE["f32"])


def test_full_scratch_chunks():
    """rfft, irfft and convolve with 3 spectrum rows across a scratch chunk whose size is not a multiple of 3, so the
    second chunk starts at spectrum row 1; the first chunk holds more than 65535 rows (the grid.y cap of
    hermitian_kernel and hermitian_mul_kernel)"""
    n = 1013
    chunk = full_chunk_size(n)
    assert chunk % 3 and chunk > 65535
    batch = chunk + 2 + (-(chunk + 2)) % 3
    check_real_size("f32", n, [batch], codes_at=(), tag=f", scratch chunks of {chunk}")
    check_convolve("f32", n, batch, 3, tag=f", scratch chunks of {chunk}")


@pytest.mark.parametrize("n", [9, 1009])
def test_hermitian_rows_past_the_grid_y_cap(n):
    """more than 65535 rows in one chunk (N = 1009: two chunks, the first of 66510 rows)"""
    batch = 70001
    assert min(batch, full_chunk_size(n)) > 65535
    check_real_size("f32", n, [batch], codes_at=(), tag=f", scratch chunks of {full_chunk_size(n)}")
    check_convolve("f32", n, batch, 1)


# ---- 5. host staging past 64 MiB -------------------------------------------------------------------------------------

def staging_rows(batch, in_row, out_row):
    """real.cu stage_rows: rows per host chunk"""
    return min(batch, max(1, HOST_CHUNK // max(in_row, out_row)))


def host_calls(p, call, x, want, in_row, out_row, device_launches, what):
    """call(src, dst) on numpy arrays and on pinned tensors must give the device result `want` bit for bit, with the
    launches of one device call per staging chunk -> failures"""
    batch = x.shape[0]
    rows = staging_rows(batch, in_row, out_row)
    expect = sum(device_launches(nb) for nb in chunks(batch, rows))
    wnp = want.cpu().numpy()
    failures = []
    for kind in ("numpy", "pinned"):
        if kind == "numpy":
            src = x.cpu().numpy()
            dst = np.full(wnp.shape, np.nan, dtype=wnp.dtype)
        else:
            src = x.cpu().pin_memory()
            dst = torch.full(want.shape, complex(float("nan"), float("nan")) if want.is_complex() else float("nan"),
                             dtype=want.dtype).pin_memory()
        call(src, dst)
        got = p.info()["last_launches"]
        d = dst if kind == "numpy" else dst.numpy()
        if not np.array_equal(np.ascontiguousarray(d).view(np.uint8), np.ascontiguousarray(wnp).view(np.uint8)):
            failures.append(f"{what}, {kind}: differs from the device call")
        if got != expect:
            failures.append(f"{what}, {kind}: {got} launches, expected {expect} ({len(chunks(batch, rows))} staging "
                            f"chunks of {rows})")
    return failures


HOST_SIZES = [("f32", 2048), ("f32", 4096), ("f32", 1013)]   # fused, half, full


@pytest.mark.parametrize("prec,n", HOST_SIZES, ids=[f"{r}-{n}" for r, n in HOST_SIZES])
def test_host_staging(prec, n):
    p = real_plan(prec, n)
    bins = n // 2 + 1
    rsz, csz = n * ESIZE[prec] // 2, bins * ESIZE[prec]
    batch = 2 * staging_rows(1 << 40, rsz, csz) + 5
    require(8 * batch * n * ESIZE[prec], f"{prec} N={n} batch {batch}")
    tol = real_bound(prec, n)
    failures = []
    for code in (T.Fft, T.Ifft):
        fwd = code.is_forward()
        base = base_reals(prec, P, n, 3 * n) if fwd else base_spectra(prec, P, n, 3 * n)
        x = periodic(torch.from_numpy(base), batch, prec)
        nref = ref_rows(P, n)
        ref = truth_rfft(base[:nref], int(code)) if fwd else truth_irfft(base[:nref], n, int(code))
        run = (rfft_run if fwd else irfft_run)(p, prec, code)
        _, f, _, y = check_rows(p, prec, run, x, ref, tol, single=False, what=f"{code.name} batch {batch}")
        failures += f
        method = p.rfft if fwd else p.irfft
        failures += host_calls(p, lambda s, d: method(s, d, code), x, y, rsz if fwd else csz, csz if fwd else rsz,
                               lambda nb: expected_launches(prec, n, fwd, nb, code), f"{code.name} host")
        del x, y
    for t in (2, 3):
        base = base_reals(prec, P, n, 5 * n + t)
        x = periodic(torch.from_numpy(base), batch, prec)
        ref = dct_mod.ref_dct(base[:ref_rows(P, n)], t, "backward")

        def run(xx, first):
            yy = nan(xx.shape, RDT[prec])
            p.dct(xx, yy, type=t)
            return yy
        _, f, _, y = check_rows(p, prec, run, x, ref, dct_mod.TOL[prec], single=False, what=f"dct {t} batch {batch}")
        failures += f
        failures += host_calls(p, lambda s, d: p.dct(s, d, type=t), x, y, rsz, rsz,
                               lambda nb: (run(x[:nb], 0), p.info()["last_launches"])[1], f"dct {t} host")
        del x, y
    torch.cuda.synchronize()
    print(f"\n{prec} N={n} {p.info()['path_name']}: host rfft / irfft / dct batch {batch} in staging chunks of "
          f"{staging_rows(batch, rsz, csz)}", end="")
    p.close()
    assert not failures, f"{prec} N={n}:\n  " + "\n  ".join(failures)
    crow = staging_rows(1 << 40, rsz, rsz)
    assert crow % 3, crow
    check_convolve(prec, n, 3 * (crow + 2), 3, host=True, tag=f", host staging chunks of {crow}")


# ---- 6. every fused family kernel past one grid sweep ---------------------------------------------------------------

FAMILY_CASES = [(r, n) for r in ("f32", "f64") for n in FUSED_N[r]]
FAMILIES = ["conv", "lconv", "stft", "dct2", "dct3", "mel", "mfcc", "welch", "csd", "coherence"]
LINEAR = {"conv", "lconv", "stft", "dct2", "dct3"}
N_MELS = 40


def family(kind, p, prec, n, sms_groups):
    """-> (inputs as base rows (q, L) numpy, run(x, first), reference of base rows, tolerance, absolute, items per row,
    description) for one call whose groups span about 1.3 grid sweeps"""
    c, grid, items = sms_groups
    rng = np.random.default_rng(n + len(kind))
    if kind == "conv":
        h = torch.from_numpy(conv_mod.spectra(prec, (), n, n)).cuda()
        rows = items
        return (n, rows, conv_run(p, prec, h[None], 1), lambda xb: conv_mod.truth(xb, h.cpu().numpy(), n),
                conv_mod.TOL[prec], False, f"{rows} rows")
    if kind in ("dct2", "dct3"):
        t = int(kind[-1])

        def run(x, first):
            y = nan(x.shape, RDT[prec])
            p.dct(x, y, type=t, norm="ortho")
            return y
        return n, items, run, lambda xb: dct_mod.ref_dct(xb, t, "ortho"), dct_mod.TOL[prec], False, f"{items} rows"
    if kind == "lconv":
        k = n // 4 + 1
        length = 4 * n
        h = lconv_mod.taps((), k, n)
        hs = torch.from_numpy(lconv_mod.spectra(prec, h, n)).cuda()
        per = (length + k - 1) // (n - k + 1)   # at least this many segments per row
        rows = -(-items // per)

        def run(x, first):
            y = nan((x.shape[0], length + k - 1), RDT[prec])
            p.convolve_linear(x, hs, k, y, "full")
            return y
        return length, rows, run, lambda xb: lconv_mod.truth(xb, h, "full"), lconv_mod.TOL[prec], False, \
            f"{rows} rows of >= {per} segments"
    hop, length = n // 4, 4 * n
    if kind in ("stft", "mel", "mfcc"):
        frames = p.stft_frames(length, hop)
        rows = -(-items // frames)
        if kind == "stft":
            w = stft_mod.window(prec, n)
            wd = torch.from_numpy(w).cuda()

            def run(x, first):
                y = nan((x.shape[0], frames, n // 2 + 1), TDT[prec])
                p.stft(x, wd, hop, y)
                return y
            return length, rows, run, lambda xb: stft_mod.ref_stft(xb, w, hop, True, "reflect"), \
                stft_mod.TOL[prec], False, f"{rows} rows of {frames} frames"
        w = mel_mod.hann(prec, n)
        filt = rng.random((N_MELS, n // 2 + 1)).astype(NPR[prec])
        d = mfcc_mod.dct_matrix(prec, N_MELS, 13) if kind == "mfcc" else None
        wd, fd = torch.from_numpy(w).cuda(), torch.from_numpy(filt).cuda()
        dd = None if d is None else torch.from_numpy(d).cuda()

        def run(x, first):
            y = nan((x.shape[0], frames, N_MELS if d is None else 13), RDT[prec])
            if kind == "mel":
                p.mel_spectrogram(x, wd, hop, fd, y)
            else:
                p.mfcc(x, wd, hop, fd, dd, y, top_db=None)
            return y
        if kind == "mel":
            ref = lambda xb: mel_mod.ref_mel(xb, w, hop, True, "reflect", filt, 2)   # noqa: E731
        else:
            ref = lambda xb: mfcc_mod.ref_mfcc(xb, w, hop, filt, d, top_db=None)   # noqa: E731
        return length, rows, run, ref, mel_mod.TOL[prec], False, f"{rows} rows of {frames} frames"
    # welch: rows of C frames, csd / coherence: rows of C/2 frame pairs -- one item per group, so groups = rows
    frames = c if kind == "welch" else c // 2
    hop = n // 2
    length = welch_mod.row_len(n, hop, frames)
    rows = int(1.3 * grid) + 1
    w = welch_mod.hann(prec, n) + NPR[prec](0.25)
    wd = torch.from_numpy(w).cuda()
    if kind == "welch":
        def run(x, first):
            y = nan((x.shape[0], n // 2 + 1), RDT[prec])
            p.welch(x, wd, hop, y)
            return y
        return length, rows, run, lambda xb: welch_mod.ref_welch(xb, w, hop, 1.0, "density", "constant"), \
            welch_mod.TOL[prec], False, f"{rows} rows of {frames} frames"
    # the y rows travel as the second half of each input row
    def run(x, first):
        xs, ys = x[:, :length].contiguous(), x[:, length:].contiguous()
        y = nan((x.shape[0], n // 2 + 1), TDT[prec] if kind == "csd" else RDT[prec])
        getattr(p, kind)(xs, ys, wd, hop, y)
        return y
    if kind == "csd":
        ref = lambda xb: csd_mod.ref_csd(xb[:, :length], xb[:, length:], w, hop)   # noqa: E731
    else:
        ref = lambda xb: csd_mod.ref_coherence(xb[:, :length], xb[:, length:], w, hop)   # noqa: E731
    return 2 * length, rows, run, ref, csd_mod.TOL[prec], kind == "coherence", f"{rows} rows of {frames} frame pairs"


@pytest.mark.parametrize("kind", FAMILIES)
@pytest.mark.parametrize("prec,n", FAMILY_CASES, ids=[f"{r}-{n}" for r, n in FAMILY_CASES])
def test_family_kernel_past_one_grid_sweep(prec, n, kind):
    p = real_plan(prec, n)
    c, grid, items = fused_wrap(prec, n)
    length, rows, run, ref_fn, tol, absolute, what = family(kind, p, prec, n, (c, grid, items))
    require(6 * rows * length * ESIZE[prec], f"{kind} {prec} N={n} {what}")
    scale = kind in LINEAR
    xb = base_reals(prec, P, length, 11 * n + len(kind))
    x = periodic(torch.from_numpy(xb), rows, prec, scale)
    ref = ref_fn(xb)
    run(x[:1].clone(), 0)
    one = p.info()["last_launches"]
    worst, failures, launched, _ = check_rows(p, prec, run, x, ref, tol, scale=scale, decoy=torch.randn_like(x),
                                              absolute=absolute, what=f"{kind} {what}")
    failures += [] if launched == one else [f"{launched} launches, batch 1 takes {one}"]
    torch.cuda.synchronize()
    print(f"\n{prec} N={n} {kind}: {what} (groups of {c} transforms on at most {grid} CTAs), {launched} launches, "
          f"worst error of the base rows {worst:.2e} (tol {tol:.0e})", end="")
    p.close()
    assert not failures, f"{kind} {prec} N={n}:\n  " + "\n  ".join(failures)

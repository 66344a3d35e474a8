"""The schedule of the persistent two-pass kernel (fused_twopass_kernel), checked transform by transform.

A race in its work queue, ring or readiness counters does not change the arithmetic: it makes a few transforms of a
long batch wrong (stale data from transform b - RING, a tile read before it was stored, a slot overwritten early, a tile
never stored).  So every configuration runs a batch that wraps its ring at least twice under full load, and the same
batch on the smallest ring (RING=2, LAG=1: every pass-1 tile waits for the slot of transform b - 2), and every
transform of it is checked

  1. against numpy's FFT in long double, per transform, within the bounds tools/emulate.cu enforces on the same tile
     arithmetic (2e-6 f32, 5e-15 f64);
  2. bit for bit against the same plan run on that transform alone (batch 1): the per-tile arithmetic does not depend
     on the schedule, so any difference is a scheduling bug;
  3. bit for bit against the same call in place.

Every output buffer starts as NaN (a tile never stored shows), and a decoy call on other input runs first (the ring
then holds wrong but plausible data).  A failure names the transforms, their ring slots and the first bad bins.
The tile kernels that replace the persistent kernel with FOURIER_B200_FUSED=0, and their chunk loop, are checked the
same way."""
import re

import numpy as np
import pytest
import torch

import fourier_b200 as fb
from oracle import oracle as O
from helpers import per_transform_err, poisoned_like, scale_ld, truth_ld

pytestmark = pytest.mark.gpu

T = fb.Transform
NP = {"f32": np.complex64, "f64": np.complex128}
TDT = {"f32": torch.complex64, "f64": torch.complex128}
BITS = {"f32": torch.int32, "f64": torch.int64}
TOL = {"f32": 2e-6, "f64": 5e-15}
FIRST, DECOY = 5, 100003          # first_transform of the checked input and of the decoy input
KNOBS = ("FOURIER_B200_FUSED", "FOURIER_B200_CHUNK_MB", "FOURIER_B200_RING", "FOURIER_B200_LAG")

SIZES = [("f32", 1 << k) for k in range(13, 21)] + [("f64", 1 << k) for k in (12, 13, 14, 16)]
CONFIGS = [(r, n, False) for r, n in SIZES] + [(r, n, True) for r, n in SIZES]   # True: RING=2, LAG=1
SMALLEST_RING = {"FOURIER_B200_RING": 2, "FOURIER_B200_LAG": 1}
DESC = re.compile(r"^fused::fused_twopass_kernel \[(\d+)x(\d+), (\d+) groups x (\d+), (TMA staging|direct loads), "
                  r"ring (\d+), lag (\d+)\]$")


def _id(c):
    return f"{c[0]}-2^{c[1].bit_length() - 1}-{'ring2' if c[2] else 'default'}"


def make_plan(monkeypatch, real, n, **env):
    """A plan created under the given FOURIER_B200_* settings (read at creation) and no others."""
    for k in KNOBS:
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, str(v))
    p = fb.create_fft_f32(n) if real == "f32" else fb.create_fft_f64(n)
    for k in env:
        monkeypatch.delenv(k)
    return p


def persistent_plan(monkeypatch, real, n, **env):
    """-> plan, its configuration parsed from kernel_name()"""
    p = make_plan(monkeypatch, real, n, **env)
    name = p.kernel_name()
    m = DESC.match(name)
    assert m, f"not a persistent-kernel description: {name!r}"
    n1, n2, groups, gt, loads, ring, lag = m.groups()
    assert int(n1) * int(n2) == n
    return p, {"name": name, "groups": int(groups), "group_threads": int(gt), "direct": loads == "direct loads",
               "ring": int(ring), "lag": int(lag)}


def device_input(real, batch, n, first):
    x = torch.empty((batch, n), dtype=TDT[real], device="cuda")
    return fb.fill_input(x, first_transform=first)


def host_input(real, batch, n, first, x_dev):
    """The same values rebuilt on the host (the counter hash is bit-identical on both)."""
    xh = O.fill_input(batch, n, NP[real], first_transform=first)
    assert np.array_equal(xh.view(np.uint8), x_dev.cpu().numpy().view(np.uint8)), "device and host input differ"
    return xh


def run(plan, x, code, decoy=None):
    """Out-of-place call into a NaN-filled buffer; with `decoy`, a call on that input (into another NaN-filled buffer)
    runs first."""
    if decoy is not None:
        plan.transform(decoy, poisoned_like(decoy), code)
    out = poisoned_like(x)
    plan.transform(x, out, code)
    return out


def one_by_one(plan, x, code):
    """Every transform of `x` on its own (a device slice of batch 1)."""
    out = poisoned_like(x)
    for b in range(x.shape[0]):
        plan.transform(x[b:b + 1], out[b:b + 1], code)
    return out


def _slots(rows, ring):
    rows = [int(b) for b in rows]
    more = f" (+{len(rows) - 8} more)" if len(rows) > 8 else ""
    return f"transforms {rows[:8]}{more}, b % {ring} = {[b % ring for b in rows[:8]]}"


def check_reference(y, ref, real, ring, what):
    """Check 1 on every transform; returns (worst error, failure text or None)."""
    err = per_transform_err(y, ref)
    bad = np.nonzero(~(err < TOL[real]))[0]
    if bad.size == 0:
        return float(err.max()), None
    bins = []
    for b in bad[:3]:
        scale = np.abs(ref[b]).max()
        k = np.nonzero(~(np.abs(y[b].astype(ref.dtype) - ref[b]) <= TOL[real] * scale))[0]
        bins.append(f"b={b}: bins {k[:6].tolist()} of {k.size}")
    return float(err.max()), (f"{what}: {bad.size} of {len(err)} transforms off the long-double reference "
                              f"(tol {TOL[real]:.0e}, worst {err.max():.2e}): {_slots(bad, ring)}; "
                              f"first bad bins {'; '.join(bins)}")


def check_bits(got, want, real, ring, what):
    """Checks 2 and 3: bit identity of two device results; returns failure text or None."""
    a = torch.view_as_real(got).view(BITS[real]).view(got.shape[0], -1)
    b = torch.view_as_real(want).view(BITS[real]).view(got.shape[0], -1)
    diff = (a != b).view(got.shape[0], got.shape[1], 2).any(dim=2)
    rows = torch.nonzero(diff.any(dim=1)).flatten().tolist()
    if not rows:
        return None
    bins = [f"b={r}: bins {torch.nonzero(diff[r]).flatten()[:6].tolist()}" for r in rows[:3]]
    return f"{what}: {len(rows)} of {got.shape[0]} transforms differ: {_slots(rows, ring)}; first bins {'; '.join(bins)}"


# ---- 1. every persistent configuration, at a batch that wraps its ring under full load ---------------------------

@pytest.mark.parametrize("real,n,smallest", CONFIGS, ids=[_id(c) for c in CONFIGS])
def test_every_transform_of_a_ring_wrapping_batch(monkeypatch, real, n, smallest):
    p, cfg = persistent_plan(monkeypatch, real, n)
    batch = 2 * cfg["ring"] + cfg["lag"] + 3     # wraps the default ring at least twice; prologue and epilogue run
    if smallest:
        p.close()
        p, cfg = persistent_plan(monkeypatch, real, n, **SMALLEST_RING)
        assert (cfg["ring"], cfg["lag"]) == (2, 1), cfg["name"]
    ring = cfg["ring"]
    window = 2 * cfg["groups"] * torch.cuda.get_device_properties(0).multi_processor_count
    x = device_input(real, batch, n, FIRST)
    decoy = device_input(real, batch, n, DECOY)
    xh = host_input(real, batch, n, FIRST, x)
    codes = list(T) if not smallest else [T.Fft, T.SqrtScaledIfft]
    bit_codes = (T.Fft, T.SqrtScaledIfft)
    failures, worst = [], {}
    unscaled, direction = None, None
    for code in sorted(codes, key=lambda c: not c.is_forward()):   # one long-double reference alive at a time
        if direction != code.is_forward():
            direction, unscaled = code.is_forward(), None
            unscaled = truth_ld(xh, int(T.Fft if direction else T.UnscaledIfft))
        out = run(p, x, code, decoy)
        ref = scale_ld(unscaled, int(code))
        worst[code.name], msg = check_reference(out.cpu().numpy(), ref, real, ring, f"{code.name} batch {batch}")
        del ref
        failures += [msg] if msg else []
        z = x.clone()
        p.transform_in_place(z, code)
        failures += [m for m in [check_bits(z, out, real, ring, f"{code.name} in place vs out of place")] if m]
        if code in bit_codes:
            single = one_by_one(p, x, code)
            failures += [m for m in [check_bits(out, single, real, ring, f"{code.name} batch {batch} vs batch 1")] if m]
    torch.cuda.synchronize()
    print(f"\n{real} N=2^{n.bit_length() - 1} {cfg['name']}: B={batch} "
          f"({batch / ring:.2f} rings), ~{window} work items in flight; worst per-transform error "
          + " ".join(f"{c} {e:.2e}" for c, e in worst.items()))
    p.close()
    assert not failures, f"{cfg['name']}:\n  " + "\n  ".join(failures)


# ---- 2. batches on both sides of the ring-shrink rule ---------------------------------------------------------------

def _sweep(ring, lag):
    return sorted({1, 2, 3, lag - 1, lag, lag + 1, ring // 2, ring // 2 + 1, ring - 1, ring, ring + 1, 2 * ring + 1})


@pytest.mark.parametrize("real,n", [("f32", 1 << 13), ("f32", 1 << 20), ("f64", 1 << 16)])
def test_batches_across_the_ring_shrink_rule(monkeypatch, real, n):
    p, cfg = persistent_plan(monkeypatch, real, n)
    ring, lag = cfg["ring"], cfg["lag"]
    if ring <= 8:
        batches = list(range(1, 2 * ring + 2))
    else:
        batches = [b for b in _sweep(ring, lag) if b >= 1 and (real == "f32" or b <= 80)]
    top = max(batches)
    x = device_input(real, top, n, FIRST)
    decoy = device_input(real, top, n, DECOY)
    ref = truth_ld(host_input(real, top, n, FIRST, x), int(T.Fft))
    single = one_by_one(p, x, T.Fft)
    failures, worst = [], 0.0
    for batch in batches:
        out = run(p, x[:batch], T.Fft, decoy[:batch])
        err, msg = check_reference(out.cpu().numpy(), ref[:batch], real, ring, f"batch {batch}")
        worst = max(worst, err)
        failures += [m for m in [msg, check_bits(out, single[:batch], real, ring, f"batch {batch} vs batch 1")] if m]
    print(f"\n{cfg['name']}: batches {batches}, worst per-transform error {worst:.2e}")
    p.close()
    assert not failures, f"{cfg['name']}:\n  " + "\n  ".join(failures)


# ---- 3. the tile kernels (FOURIER_B200_FUSED=0 and the sizes without a persistent kernel) and their chunk loop -------

TWO_PASS = [("f32", 1 << k) for k in range(11, 21)] + [("f64", 1 << k) for k in range(9, 17)]


def _check_tile_path(p, real, n, batch, chunk):
    assert p.info()["path_name"] == "twopass" and "tile_kernel" in p.kernel_name(), p.kernel_name()
    x = device_input(real, batch, n, FIRST)
    xh = host_input(real, batch, n, FIRST, x)
    chunks = -(-batch // chunk)
    failures = []
    for code in (T.Fft, T.SqrtScaledIfft):
        out = run(p, x, code)
        assert p.info()["last_launches"] == 2 * chunks, (code, p.info()["last_launches"], chunks)
        err, msg = check_reference(out.cpu().numpy(), truth_ld(xh, int(code)), real, chunk,
                                   f"{code.name} batch {batch}, {chunks} chunks of {chunk}")
        failures += [msg] if msg else []
        print(f"\n{real} N=2^{n.bit_length() - 1} tile kernels: batch {batch} in {chunks} chunks of {chunk}, "
              f"{code.name} worst per-transform error {err:.2e}", end="")
    assert not failures, "\n  ".join(failures)


@pytest.mark.parametrize("real,n", TWO_PASS, ids=[f"{r}-2^{n.bit_length() - 1}" for r, n in TWO_PASS])
def test_tile_kernels_in_one_megabyte_chunks(monkeypatch, real, n):
    p = make_plan(monkeypatch, real, n, FOURIER_B200_FUSED=0, FOURIER_B200_CHUNK_MB=1)
    chunk = max(1, (1 << 20) // (n * np.dtype(NP[real]).itemsize))
    _check_tile_path(p, real, n, 2 * chunk + max(1, chunk // 2), chunk)    # several chunks, the last one partial
    p.close()


@pytest.mark.parametrize("real,n,batch", [("f64", 1 << 15, 133), ("f32", 1 << 11, 4100), ("f32", 1 << 12, 2050)])
def test_tile_kernels_beyond_one_default_chunk(monkeypatch, real, n, batch):
    p = make_plan(monkeypatch, real, n)
    _check_tile_path(p, real, n, batch, (32 << 20) // (n * np.dtype(NP[real]).itemsize))
    p.close()

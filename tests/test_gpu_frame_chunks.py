"""The frame-chunk loops and host staging of the framed real transforms, pinned by exact launch counts and bits.

A real plan runs the frames of stft, mel, mfcc, welch, csd and coherence off the fused path in chunks through its
512 MB scratch: per chunk a gather, the plan's own rfft and the operation's consumer kernels.  Host memory goes through
64 MB staging chunks of rows, each running the device call's steps on its rows, plus the kernels a call runs once (the
mel bands, the Welch scale).  So a call's launches are

  once + sum over staging chunks of (sum over scratch chunks of (kernels per chunk + the rfft's launches)),

with one staging chunk for device memory, and rows cut by a scratch or staging chunk equal the same rows run alone,
bit for bit.  Every case runs f32 N = 400 (real_half) with hop 160, as Whisper does."""
import numpy as np
import pytest
import torch

from test_gpu_csd import dev_call, partner
from test_gpu_mel import bank, hann, launches, plan, reals, rfft_launches
from test_gpu_mfcc import dct_matrix, dev_mfcc

pytestmark = pytest.mark.gpu

SCRATCH = 512 << 20             # kScratchTargetBytes
HOST_CHUNK = 64 << 20           # kHostChunkBytes
N, HOP, BINS = 400, 160, 201
FRAME, SPEC = N * 4, BINS * 8   # bytes of one f32 frame and of one spectrum
N_MELS, N_OUT = 80, 13


def chunks(total, size):
    return [min(size, total - q0) for q0 in range(0, total, size)]


def frame_launches(p, total, item_bytes, per_chunk, k=1):
    """launches of the scratch chunks of `total` frames (or frame pairs, k = 2) of item_bytes each: per chunk
    per_chunk kernels and the plan's rfft of its k * nq frames"""
    size = min(total, max(1, SCRATCH // item_bytes))
    return sum(per_chunk + rfft_launches(p, k * nq) for nq in chunks(total, size))


def bits(a):
    a = a.cpu().numpy() if isinstance(a, torch.Tensor) else a
    return np.ascontiguousarray(a).view(np.uint8)


def test_stft_two_scratch_chunks():
    """112 rows of 3001 frames: 335544 frames of 1600 bytes fill the scratch, so the cut falls inside row 111"""
    p = plan("f32", N)
    assert p.info()["path_name"] == "real_half"
    rows = 112
    x = torch.from_numpy(reals("f32", (rows, 480000), 61)).cuda()
    w = torch.from_numpy(hann("f32", N)).cuda()
    frames = p.stft_frames(480000, HOP)
    out = torch.full((rows, frames, BINS), complex(float("nan"), float("nan")), dtype=torch.complex64, device="cuda")
    p.stft(x, w, HOP, out)
    got = launches(p)
    chunk = SCRATCH // FRAME
    assert (frames, chunk, chunk // frames) == (3001, 335544, 111) and chunk < rows * frames
    assert got == frame_launches(p, rows * frames, FRAME, 1)
    for r in (0, chunk // frames, rows - 1):
        alone = torch.empty((1, frames, BINS), dtype=torch.complex64, device="cuda")
        p.stft(x[r:r + 1], w, HOP, alone)
        assert np.array_equal(bits(out[r:r + 1]), bits(alone)), r


@pytest.mark.parametrize("top_db_rows", (None, 4))
def test_mfcc_two_scratch_chunks(top_db_rows):
    """60 rows of 3001 frames: a frame, its spectrum and its 80 mels take 3528 bytes, so 152174 frames fill the
    scratch and the cut falls inside row 50, within the clamp group of rows 48 .. 51"""
    p = plan("f32", N)
    rows = 60
    x = reals("f32", (rows, 480000), 62)
    x[49] *= 1e-3
    w = hann("f32", N)
    f = bank("f32", N, N_MELS, "slaney")
    d = dct_matrix("f32", N_MELS, N_OUT)
    kw = dict(top_db=None) if top_db_rows is None else dict(top_db_rows=top_db_rows)
    got, frames = dev_mfcc(p, x, w, HOP, f, d, **kw)
    n = launches(p)
    item = FRAME + SPEC + N_MELS * 4
    chunk = SCRATCH // item
    assert (chunk, chunk // frames) == (152174, 50)
    sweeps = 1 if top_db_rows is None else 2
    assert n == 1 + sweeps * frame_launches(p, rows * frames, item, 3)   # bands; per chunk gather, mels, mfcc
    g0, g1 = (50, 51) if top_db_rows is None else (48, 52)
    alone, _ = dev_mfcc(p, np.ascontiguousarray(x[g0:g1]), w, HOP, f, d, **kw)
    assert np.array_equal(bits(got[g0:g1]), bits(alone))


def test_coherence_two_row_chunks_of_partials():
    """702 rows of 1024 frames at hop 1: 256 items of 4 frames per row, whose 4 planes of partials take 823296 bytes,
    so 652 rows fill the partials; within each such chunk 83676 frame pairs fill the scratch"""
    p = plan("f32", N)
    length, frames, items = N + 1023, 1024, 256
    x = reals("f32", (234, 3, length), 63) + np.float32(0.5)
    y = partner("f32", x[0], 64)
    w = hann("f32", N)
    got = dev_call(p, "coherence", x, y, w, 1).reshape(702, BINS)
    n = launches(p)
    rows = SCRATCH // (items * 4 * BINS * 4)
    pair = 2 * (FRAME + SPEC)
    assert (rows, SCRATCH // pair) == (652, 83676)
    # per row chunk: per scratch chunk the gather and the accumulate, then the finish
    assert n == sum(frame_launches(p, nr * frames, pair, 2, k=2) + 1 for nr in chunks(702, rows))
    xr = x.reshape(702, length)
    for r in (0, 83676 // frames, rows - 1, rows, 701):
        alone = dev_call(p, "coherence", xr[r:r + 1], y[r % 3], w, 1)
        assert np.array_equal(bits(got[r:r + 1]), bits(alone)), r


# ---- host memory over several staging chunks -------------------------------------------------------------------------

LENGTH, TAPS = 48000, 101


def cases():
    """kind -> (output shape of one row, output dtype, in_row bytes, out_row bytes, launches once per call, sweeps over
    the rows, run(p, src, dst, consts))"""
    framed = 1 + LENGTH // HOP                 # 301 frames with center
    real_row = LENGTH * 4

    def stft(p, s, d, c):
        p.stft(s, c["w"], HOP, d)

    def istft(p, s, d, c):
        p.istft(s, c["w"], HOP, d)

    def mel(p, s, d, c):
        p.mel_spectrogram(s, c["w"], HOP, c["f"], d)

    def mfcc(p, s, d, c, **kw):
        p.mfcc(s, c["w"], HOP, c["f"], c["d"], d, **kw)

    def welch(p, s, d, c):
        p.welch(s, c["w"], HOP, d)

    def cross(kind):
        def run(p, s, d, c):
            # the rows in pairs of three with y's three rows, when they come in threes; one y row otherwise
            if s.shape[0] % 3 == 0:
                getattr(p, kind)(s.reshape(-1, 3, LENGTH), c["y"], c["w"], HOP, d.reshape(-1, 3, BINS))
            else:
                getattr(p, kind)(s, c["y"][0], c["w"], HOP, d)
        return run

    def lconv(p, s, d, c):
        p.convolve_linear(s, c["h"], TAPS, d, "full")

    return {
        "stft": ((framed, BINS), torch.complex64, real_row, framed * SPEC, 0, 1, stft),
        "istft": ((LENGTH,), torch.float32, framed * SPEC, real_row, 0, 1, istft),
        "mel": ((framed, N_MELS), torch.float32, real_row, framed * N_MELS * 4, 1, 1, mel),
        "mfcc": ((framed, N_OUT), torch.float32, real_row, framed * N_OUT * 4, 1, 1,
                 lambda p, s, d, c: mfcc(p, s, d, c, top_db=None)),
        "mfcc-clamp": ((framed, N_OUT), torch.float32, real_row, framed * N_OUT * 4, 1, 2,
                       lambda p, s, d, c: mfcc(p, s, d, c, top_db_rows=2)),
        "welch": ((BINS,), torch.float32, real_row, BINS * 4, 1, 1, welch),
        "csd": ((BINS,), torch.complex64, real_row, BINS * 8, 1, 1, cross("csd")),
        "coherence": ((BINS,), torch.float32, real_row, BINS * 4, 0, 1, cross("coherence")),
        "lconv": ((LENGTH + TAPS - 1,), torch.float32, real_row, (LENGTH + TAPS - 1) * 4, 0, 1, lconv),
    }


def consts(seed):
    """the operands besides the rows, as numpy arrays and as device tensors"""
    rng = np.random.default_rng(seed)
    h = np.zeros(N)
    h[:TAPS] = rng.standard_normal(TAPS)
    c = {"w": hann("f32", N), "f": bank("f32", N, N_MELS, "slaney"), "d": dct_matrix("f32", N_MELS, N_OUT),
         "y": reals("f32", (3, LENGTH), seed + 1),
         "h": np.fft.rfft(h).astype(np.complex64)}
    return c, {k: torch.from_numpy(v).cuda() for k, v in c.items()}


@pytest.mark.parametrize("kind", ["stft", "istft", "mel", "mfcc", "mfcc-clamp", "welch", "csd", "coherence", "lconv"])
def test_host_staging_chunks(kind):
    """numpy buffers over at least two staging chunks (the last one short and, for the clamp, cutting a group of two
    rows) give the device call's bits, with the once-per-call kernels plus each chunk's device launches"""
    shape, dtype, in_row, out_row, once, sweeps, run = cases()[kind]
    p = plan("f32", N)
    per = max(1, HOST_CHUNK // max(in_row, out_row))
    batch = (2 * per // 6 + 1) * 6             # a multiple of 6, in three staging chunks
    rng = np.random.default_rng(70 + len(kind))
    if kind == "istft":
        x = (rng.standard_normal((batch,) + (1 + LENGTH // HOP, BINS))
             + 1j * rng.standard_normal((batch, 1 + LENGTH // HOP, BINS))).astype(np.complex64)
    else:
        x = rng.standard_normal((batch, LENGTH)).astype(np.float32)
    ch, cd = consts(80 + len(kind))
    xd = torch.from_numpy(x).cuda()
    dev = torch.full((batch,) + shape, float("nan"), dtype=dtype, device="cuda")
    run(p, xd, dev, cd)
    torch.cuda.synchronize()
    host = np.full(dev.shape, np.nan, dtype=dev.cpu().numpy().dtype)
    run(p, x, host, ch)
    got = launches(p)
    assert np.array_equal(bits(host), bits(dev))

    # each sweep of the clamp launches the kernels of the call without it
    count = cases()["mfcc"][-1] if kind == "mfcc-clamp" else run

    def device_launches(nb):
        count(p, xd[:nb], torch.empty((nb,) + shape, dtype=dtype, device="cuda"), cd)
        return launches(p) - once

    staged = chunks(batch, per)
    assert len(staged) == 3 and (kind != "mfcc-clamp" or per % 2 == 1)   # an odd chunk cuts a clamp group
    assert got == once + sweeps * sum(device_launches(nb) for nb in staged), (got, staged)


def test_host_linear_convolution_in_runs_of_segments():
    """rows of 35 * 2^19 samples (70 MB) go through the host path in runs of segments of one row, each run the device
    steps on its segments: 55922 segments of 300 outputs a run, so a row of 61168 segments takes two runs"""
    p = plan("f32", N)
    length = 35 << 19
    s = N - TAPS + 1
    x = reals("f32", (2, length), 90)
    ch, cd = consts(91)
    out = length + TAPS - 1
    host = np.full((2, out), np.nan, np.float32)
    p.convolve_linear(x, ch["h"], TAPS, host, "full")
    got = launches(p)
    dev = torch.empty((2, out), dtype=torch.float32, device="cuda")
    p.convolve_linear(torch.from_numpy(x).cuda(), cd["h"], TAPS, dev, "full")
    assert np.array_equal(bits(host), bits(dev))
    per = -(-out // s)
    run = (HOST_CHUNK // 4 - N) // s
    assert (per, run) == (61168, 55922)

    def segments(nseg):
        # one device row of exactly nseg segments ("valid": L - K + 1 = nseg * s outputs)
        z = torch.zeros((1, TAPS - 1 + nseg * s), dtype=torch.float32, device="cuda")
        p.convolve_linear(z, cd["h"], TAPS, torch.empty((1, nseg * s), dtype=torch.float32, device="cuda"), "valid")
        return launches(p)

    assert got == 2 * sum(segments(n) for n in chunks(per, run))

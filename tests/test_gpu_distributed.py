"""The distributed six-step transform on the GPU backend with ONE rank (all-to-all degenerates to the
local transposes): checks the CUDA transpose / twiddle kernels and the batched local FFTs inside the
six-step flow against the oracle and against the single-plan path.  The multi-rank exchange logic is
covered on CPU (tests/test_distributed_host_logic.py) and by tools/dist_check.py under torchrun."""
import os

import numpy as np
import pytest

from oracle import oracle as O
from helpers import rel_err

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("real,n1,n2", [("f32", 256, 256), ("f32", 1024, 1024), ("f32", 2048, 1024),
                                        ("f32", 96, 243), ("f64", 256, 256), ("f64", 512, 128)])
@pytest.mark.parametrize("forward", [True, False])
def test_six_step_single_rank_vs_oracle(real, n1, n2, forward):
    import torch
    from fourier_b200.distributed import CudaBackend, DistributedFft
    dt = np.complex64 if real == "f32" else np.complex128
    x = O.fill_input(1, n1 * n2, dt)[0]
    xd = torch.from_numpy(x.copy()).cuda()
    out = DistributedFft(n1, n2, 0, 1, CudaBackend(real)).transform(xd, torch.empty_like(xd), forward=forward)
    torch.cuda.synchronize()
    want = O.transform(x, O.FFT if forward else O.UNSCALED_IFFT)
    assert rel_err(out.cpu().numpy(), want) < (1e-5 if real == "f32" else 1e-12)


def test_transpose_and_swap_kernels():
    import torch
    from fourier_b200.distributed import CudaBackend
    be = CudaBackend("f32")
    a = torch.randn(3 * 70 * 45, dtype=torch.complex64, device="cuda")
    out = torch.empty_like(a)
    be._call("transpose", a.data_ptr(), out.data_ptr(), 3, 70, 45, be._stream(a))
    assert torch.equal(out.view(3, 45, 70), a.view(3, 70, 45).transpose(1, 2))
    be.swap_leading(a, out, 3, 70, 45)
    assert torch.equal(out.view(70, 3, 45), a.view(3, 70, 45).transpose(0, 1))


@pytest.mark.parametrize("real", ["f32", "f64"])
@pytest.mark.parametrize("twiddle", [None, (True, 37, 1 << 30), (False, 5, 3 * 70 * 96)])
def test_pack_kernel_matches_numpy_backend(real, twiddle):
    """Strided batched transpose (+ fused inter-step twiddle) against the CPU stand-in of the host tests."""
    import torch
    from fourier_b200.distributed import CudaBackend, NumpyBackend
    dt = torch.complex64 if real == "f32" else torch.complex128
    batch, rows, cols, ld, col0 = 3, 70, 20, 96, 9          # column blocks [9, 29), [41, 61), [73, 93) of 96
    torch.manual_seed(5)
    a = torch.randn(rows * ld, dtype=dt)
    want = torch.empty(batch * cols * rows, dtype=dt)
    NumpyBackend().pack(a, want, batch, rows, cols, ld, col0, twiddle)
    got = torch.empty_like(want).cuda()
    CudaBackend(real).pack(a.cuda(), got, batch, rows, cols, ld, col0, twiddle)
    torch.cuda.synchronize()
    assert rel_err(got.cpu().numpy(), want.numpy()) < (5e-7 if real == "f32" else 4e-15)


@pytest.mark.parametrize("real", ["f32", "f64"])
@pytest.mark.parametrize("forward", [None, True, False])
def test_peer_exchange_kernel_layout(real, forward):
    """The one-kernel exchange with the P destination buffers all on this GPU: rank by rank it must build, in
    every destination, that rank's rows of the transposed (and twiddled) global matrix."""
    import ctypes
    import torch
    from fourier_b200.distributed import CudaBackend
    P, rows_loc, cb = 4, 40, 24
    cols, n_total = P * cb, P * rows_loc * P * cb
    dt = torch.complex64 if real == "f32" else torch.complex128
    torch.manual_seed(11)
    g = torch.randn(P * rows_loc, cols, dtype=torch.complex128)
    if forward is not None:
        idx = (torch.arange(P * rows_loc)[:, None] * torch.arange(cols)[None, :]) % n_total
        w = torch.exp((-2j if forward else 2j) * np.pi * idx.to(torch.float64) / n_total)
    else:
        w = torch.ones_like(g)
    outs = [torch.zeros(cb * P * rows_loc, dtype=dt, device="cuda") for _ in range(P)]
    table = (ctypes.c_void_p * P)(*[o.data_ptr() for o in outs])
    be = CudaBackend(real)
    for me in range(P):
        src = g[me * rows_loc:(me + 1) * rows_loc].to(dt).contiguous().cuda()
        be.exchange(src, table, P, me, rows_loc, cb, None if forward is None else (forward, me * rows_loc, n_total))
    torch.cuda.synchronize()
    for q in range(P):
        want = (g * w)[:, q * cb:(q + 1) * cb].t().contiguous().numpy().ravel()
        assert rel_err(outs[q].cpu().numpy(), want) < (5e-7 if real == "f32" else 4e-15)


@pytest.mark.parametrize("real,n,P,rows_loc", [("f32", 1 << 14, 4, 64), ("f32", 1 << 11, 2, 96), ("f32", 1 << 16, 8, 48),
                                               ("f32", 1 << 20, 2, 16), ("f64", 1 << 12, 4, 32), ("f64", 1 << 16, 2, 24),
                                               # 64 / 32 rows: tiles of 32 (f32) / 16 (f64) transforms, 256-byte store runs
                                               ("f32", 1 << 16, 4, 64), ("f64", 1 << 16, 4, 32), ("f32", 1 << 14, 2, 48)])
@pytest.mark.parametrize("forward", [True, False])
@pytest.mark.parametrize("twiddle", [False, True])
def test_rows_fft_with_fused_exchange_matches_fft_then_exchange(real, n, P, rows_loc, forward, twiddle):
    """fft_rows_exchange (the exchange folded into the last register stage of the row FFT, csrc/dist_kernels.cuh)
    against the two-kernel formulation it replaces (batched FFT, then the exchange kernel) and against numpy-f64,
    with the P destination buffers all on this GPU and every rank played in turn."""
    import ctypes
    import torch
    from fourier_b200.distributed import CudaBackend
    dt = torch.complex64 if real == "f32" else torch.complex128
    cb, n_total = n // P, n * 4096
    torch.manual_seed(3)
    be = CudaBackend(real)
    fused = [torch.zeros(cb * P * rows_loc, dtype=dt, device="cuda") for _ in range(P)]
    plain = [torch.zeros(cb * P * rows_loc, dtype=dt, device="cuda") for _ in range(P)]
    tf = (ctypes.c_void_p * P)(*[o.data_ptr() for o in fused])
    tp = (ctypes.c_void_p * P)(*[o.data_ptr() for o in plain])
    srcs = []
    for me in range(P):
        src = torch.randn(rows_loc * n, dtype=dt, device="cuda")
        srcs.append(src.clone())
        tw = (forward, me * rows_loc, n_total) if twiddle else None
        be.fft_rows_exchange(src, tf, P, me, rows_loc, n, forward, tw)
        assert torch.equal(src, srcs[-1])                      # the input is left intact
        be.fft_rows(src, n, forward)
        be.exchange(src, tp, P, me, rows_loc, cb, tw)
    torch.cuda.synchronize()
    tol = 2e-6 if real == "f32" else 1e-14
    for q in range(P):
        assert rel_err(fused[q].cpu().numpy(), plain[q].cpu().numpy()) < tol
    # numpy-f64 reference of destination 0
    g = torch.cat([s.view(rows_loc, n) for s in srcs]).cpu().numpy().astype(np.complex128)
    spec = np.fft.fft(g, axis=1) if forward else np.fft.ifft(g, axis=1) * n
    if twiddle:
        idx = (np.arange(P * rows_loc, dtype=np.int64)[:, None] * np.arange(cb, dtype=np.int64)[None, :]) % n_total
        spec = spec[:, :cb] * np.exp((-2j if forward else 2j) * np.pi * idx / n_total)
    assert rel_err(fused[0].cpu().numpy(), spec[:, :cb].T.ravel()) < tol


def test_rows_fft_with_fused_exchange_chunks_and_streams(monkeypatch):
    """More rows than one L2-resident chunk: the chunks alternate between two streams (default) or run on one
    (FOURIER_B200_DIST_OVERLAP=0); both must equal the single-chunk result bit for bit."""
    import ctypes
    import torch
    from fourier_b200.distributed import CudaBackend
    n, P, rows_loc = 1 << 14, 2, 96
    src = torch.randn(rows_loc * n, dtype=torch.complex64, device="cuda")
    results = []
    for chunk_mb, overlap in (("64", "1"), ("2", "1"), ("2", "0"), ("4", "1")):
        monkeypatch.setenv("FOURIER_B200_CHUNK_MB", chunk_mb)      # 2 MB = 16 transforms per chunk -> 6 chunks
        monkeypatch.setenv("FOURIER_B200_DIST_OVERLAP", overlap)
        be = CudaBackend("f32")
        outs = [torch.zeros(n // P * rows_loc, dtype=torch.complex64, device="cuda") for _ in range(P)]
        table = (ctypes.c_void_p * P)(*[o.data_ptr() for o in outs])
        be.fft_rows_exchange(src, table, 1, 0, rows_loc, n, True, (True, 7, 1 << 30))
        torch.cuda.synchronize()
        results.append(torch.cat(outs))
    for r in results[1:]:
        assert torch.equal(r, results[0])


def test_rows_exchange_rejects_what_it_cannot_do():
    import ctypes
    import torch
    from fourier_b200 import Fft
    x = torch.zeros(32 * 243, dtype=torch.complex64, device="cuda")
    table = (ctypes.c_void_p * 1)(x.data_ptr())
    with pytest.raises(NotImplementedError):
        Fft(243, "f32").fft_rows_exchange(x.view(32, 243), table, 32, 0)            # not a two-pass plan
    y = torch.zeros(8 * 4096, dtype=torch.complex64, device="cuda")
    with pytest.raises(RuntimeError):
        Fft(4096, "f32").fft_rows_exchange(y.view(8, 4096), table, 8, 0)            # not whole tiles of rows
    table3 = (ctypes.c_void_p * 3)(y.data_ptr(), y.data_ptr(), y.data_ptr())
    with pytest.raises(RuntimeError):
        Fft(4096, "f32").fft_rows_exchange(torch.zeros(32, 4096, dtype=torch.complex64, device="cuda"), table3, 32, 0)

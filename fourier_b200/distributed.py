"""One huge 1-D complex FFT distributed over the GPUs of a box (BASELINE.json configs[4]: N = 2^30 over 8
GPUs): the six-step algorithm with all-to-all transposes between local batched FFTs.

The reference has no counterpart (single-threaded CPU code, SURVEY.md 5); this is the only place of the
engine where the path has a real exchange step, hence the only place a collective is used.

Layout.  N = N1*N2.  The input is block-distributed in natural order: rank r of P holds samples
[r*N/P, (r+1)*N/P), i.e. rows n1 in [r*N1/P, (r+1)*N1/P) of x[n1][n2] (n = n1*N2 + n2).  The output has the
same block distribution of natural order X[k], k = k1 + N1*k2: rank r holds rows k2 of X[k2][k1].

    1. exchange:  [n1_loc][n2]  ->  [n2_loc][n1],  N2/P local FFTs of length N1 over n1
    2. exchange:  [n2_loc][k1] * w_N^{n2*k1}  ->  [k1_loc][n2],  N1/P local FFTs of length N2 over n2
    3. exchange:  [k1_loc][k2]  ->  [k2_loc][k1]      (natural order)

One exchange = the transpose of a row-distributed matrix, pipelined in `chunks` pieces over the rows of the
RESULT (each piece holds complete result rows, so the work that follows can start on it):

    pack     local transpose of the piece's column blocks, so that what goes to rank q is contiguous
             (fourier_b200_pack_*; in exchange 2 the inter-step twiddle is applied on the way)
    send     one asynchronous all_to_all_single per piece: N/P/chunks samples per rank, (P-1)/P of them
             over NVLink; the collective of piece k runs while piece k+1 is packed and piece k-1 is
             unpacked and transformed
    unpack   swap of the two leading axes of the received [source rank][my rows][their rows]
             (fourier_b200_swap_leading_*) straight into the piece's rows of the result
    then     the local FFTs of those rows (fourier_b200_transform_batch_async_*)

With exchange="peer" (CudaBackend only) the three sweeps of an exchange collapse into ONE kernel
(fourier_b200_exchange_*, csrc/exchange.cu): the transposing kernel stores its tiles straight into the
destination rank's buffer over NVLink, already in the final layout, with the twiddle applied on the way;
a stream-ordered barrier (a one-element all_reduce) separates it from the FFTs that follow.  The two
work buffers then come from `plan.buffers()`: they are cudaMalloc'ed by the library and opened by every
peer through CUDA IPC (one process per GPU).

The local pieces are this library's kernels; torch provides memory, streams and the collective.

`backend` abstracts the local compute so that the exchange logic is tested on CPU with gloo + numpy
(tests/test_distributed_host_logic.py); the product backend is `CudaBackend` (no CPU fallback).
"""
import numpy as np

from . import _lib


class CudaBackend:
    """Local compute on the rank's GPU through the C ABI."""

    def __init__(self, real):
        import torch
        self.torch = torch
        self.real = real
        self.t = "float" if real == "f32" else "double"
        self.dtype = torch.complex64 if real == "f32" else torch.complex128
        self._plans = {}
        self.launches = None   # set to 0 to have the methods below count the kernels they launch (bench.py)

    def _count(self, n):
        if self.launches is not None:
            self.launches += n

    def _stream(self, x):
        return self.torch.cuda.current_stream(x.device).cuda_stream

    def _call(self, name, *args):
        rc = getattr(_lib.load(), f"fourier_b200_{name}_{self.t}")(*args)
        self._count(1)
        if rc != 0:
            raise RuntimeError(f"fourier_b200_{name}_{self.t} failed: {_lib.last_error()}")

    def empty_like(self, x):
        return self.torch.empty_like(x)

    def empty(self, samples):
        return self.torch.empty(samples, dtype=self.dtype, device="cuda")

    def _plan(self, x, n):
        from . import Fft
        key = (x.device.index, n)
        plan = self._plans.get(key)
        if plan is None:
            plan = self._plans[key] = Fft(n, self.real)
        return plan

    def fft_rows(self, x, n, forward):
        """In-place batched FFT over rows of length n (unscaled in both directions)."""
        from . import Transform
        self._plan(x, n).transform_in_place(x.view(-1, n), Transform.Fft if forward else Transform.UnscaledIfft)
        if self.launches is not None:
            self._count(self._plan(x, n).info()["last_launches"])

    def can_fuse(self, x, n, rows):
        """True if fft_rows_exchange() exists for rows of length n (two-pass plans, whole tiles of up to 32 rows)."""
        return self._plan(x, n).info()["path_name"] == "twopass" and rows % 32 == 0

    def fft_rows_exchange(self, src, table, world, rank, rows_loc, n, forward, twiddle):
        """The FFTs of the rows_loc rows of length n of `src` and the exchange() of the result in one pass: the last
        register stage of the transform stores straight into the peers' buffers (csrc/dist_kernels.cuh)."""
        tw = None if twiddle is None else (twiddle[1], twiddle[2])
        self._plan(src, n).fft_rows_exchange(src.view(rows_loc, n), table, world * rows_loc, rank * rows_loc, forward, tw)
        if self.launches is not None:
            self._count(self._plan(src, n).info()["last_launches"])

    def transpose(self, src, dst, rows, cols):
        self._call("transpose", src.data_ptr(), dst.data_ptr(), 1, rows, cols, self._stream(src))

    def pack(self, src, dst, batch, rows, cols, ld, col0, twiddle):
        """dst[b][c][r] = src[r][col0 + b*(ld/batch) + c] (* twiddle), src row-major with `ld` columns.
        twiddle = None or (forward, row0, n_total): factor w_N^{(row0 + r) * column}."""
        mode, row0, n_total = (0, 0, 0) if twiddle is None else (1 if twiddle[0] else 2, twiddle[1], twiddle[2])
        item = src.element_size()
        self._call("pack", src.data_ptr() + col0 * item, dst.data_ptr(), batch, rows, cols, ld, ld // batch,
                   cols * rows, mode, row0, col0, n_total, self._stream(src))

    def swap_leading(self, src, dst, a, b, inner):
        self._call("swap_leading", src.data_ptr(), dst.data_ptr(), a, b, inner, self._stream(src))

    def twiddle_rows(self, x, rows, cols, row0, n_total, forward):
        self._call("twiddle_rows", x.data_ptr(), rows, cols, row0, n_total, int(forward), self._stream(x))

    # ---- exchange over NVLink peer memory ------------------------------------------------------------------
    def peer_buffers(self, samples, count, rank, world, group):
        """Collective.  Allocates `count` buffers of `samples` complex values that every rank of the group can
        store into; returns (tensors, tables): tables[i][q] is the address of rank q's buffer i on this GPU."""
        import ctypes
        import torch.distributed as dist
        L = _lib.load()
        item = 8 if self.real == "f32" else 16
        mine = []
        for _ in range(count):
            ptr, handle = ctypes.c_void_p(), ctypes.create_string_buffer(64)
            if L.fourier_b200_peer_alloc(samples * item, ctypes.byref(ptr), handle) != 0:
                raise RuntimeError(f"fourier_b200_peer_alloc failed: {_lib.last_error()}")
            mine.append((ptr.value, handle.raw))
        everyone = [None] * world
        dist.all_gather_object(everyone, [h for _, h in mine], group=group)
        tensors, tables = [], []
        for i, (ptr, _) in enumerate(mine):
            table = (ctypes.c_void_p * world)()
            for q in range(world):
                if q == rank:
                    table[q] = ptr
                else:
                    peer = ctypes.c_void_p()
                    if L.fourier_b200_peer_open(everyone[q][i], ctypes.byref(peer)) != 0:
                        raise RuntimeError(f"fourier_b200_peer_open failed: {_lib.last_error()}")
                    table[q] = peer.value
            tensors.append(_as_complex_tensor(self.torch, ptr, samples, self.real))
            tables.append(table)
        self._token = self.torch.zeros(1, device="cuda")
        return tensors, tables

    def peer_release(self, tensors, tables, rank):
        """Closes the peers' mappings and frees this rank's buffers (the tensors must not be used afterwards)."""
        L = _lib.load()
        self.torch.cuda.synchronize()
        for t, table in zip(tensors, tables):
            for q in range(len(table)):
                if q != rank and table[q]:
                    L.fourier_b200_peer_close(table[q])
            L.fourier_b200_peer_free(t.data_ptr())

    def exchange(self, src, table, world, rank, rows_loc, cb, twiddle, first=0, count=None):
        """Rows [first, first + count) of this rank's rows_loc x (world * cb) matrix `src` go, transposed, into
        the peers' buffers (table[q]); twiddle = None or (forward, global index of local row 0, N)."""
        count = rows_loc - first if count is None else count
        mode, row0, n_total = (0, 0, 0) if twiddle is None else (1 if twiddle[0] else 2, twiddle[1], twiddle[2])
        ld = world * cb
        self._call("exchange", src.data_ptr() + first * ld * src.element_size(), table, world, rank, count, cb, ld,
                   world * rows_loc, rank * rows_loc + first, mode, row0 + first, n_total, self._stream(src))

    def side_stream(self):
        if getattr(self, "_side", None) is None:
            self._side = self.torch.cuda.Stream()
        return self._side

    def barrier(self, group):
        """Stream-ordered (no host synchronisation): every rank's earlier kernels have completed, and with them
        their stores into peer memory, before any rank's later kernels start."""
        import torch.distributed as dist
        dist.all_reduce(self._token, group=group)

    def all_to_all(self, dst, src, group):
        """Asynchronous: ordered after the work already enqueued on the current stream; returns a handle
        whose wait() makes the current stream (not the host) wait for the collective."""
        import torch.distributed as dist
        # NCCL has no complex dtype: exchange the raw (re, im) scalars
        return dist.all_to_all_single(self.torch.view_as_real(dst), self.torch.view_as_real(src), group=group,
                                      async_op=True)


class _DeviceMemory:
    """A library-owned device allocation seen through the CUDA array interface."""

    def __init__(self, ptr, scalars, real):
        self.__cuda_array_interface__ = {"shape": (scalars,), "typestr": "<f4" if real == "f32" else "<f8",
                                         "data": (ptr, False), "version": 2}


def _as_complex_tensor(torch, ptr, samples, real):
    flat = torch.as_tensor(_DeviceMemory(ptr, 2 * samples, real), device="cuda")
    return torch.view_as_complex(flat.view(samples, 2))


class NumpyBackend:
    """CPU stand-in used ONLY by the host-logic tests (gloo): the same interface on torch CPU tensors."""

    def __init__(self):
        import torch
        self.torch = torch

    def empty_like(self, x):
        return self.torch.empty_like(x)

    def empty(self, samples):
        return self.torch.empty(samples, dtype=self.torch.complex128)

    def fft_rows(self, x, n, forward):
        a = x.view(-1, n).numpy()
        a[...] = np.fft.fft(a, axis=-1) if forward else np.fft.ifft(a, axis=-1) * n

    def transpose(self, src, dst, rows, cols):
        dst.view(cols, rows).copy_(src.view(rows, cols).t())

    def pack(self, src, dst, batch, rows, cols, ld, col0, twiddle):
        a = src.view(rows, ld).numpy()
        out = dst.view(batch, cols, rows).numpy()
        for b in range(batch):
            c = col0 + b * (ld // batch) + np.arange(cols, dtype=np.int64)
            blk = a[:, c]
            if twiddle is not None:
                forward, row0, n_total = twiddle
                idx = (np.arange(rows, dtype=np.int64)[:, None] + row0) * c[None, :] % n_total
                blk = blk * np.exp((-2j if forward else 2j) * np.pi * idx / n_total).astype(a.dtype)
            out[b] = blk.T

    def swap_leading(self, src, dst, a, b, inner):
        dst.view(b, a, inner).copy_(src.view(a, b, inner).transpose(0, 1))

    def twiddle_rows(self, x, rows, cols, row0, n_total, forward):
        idx = (np.arange(rows, dtype=np.int64)[:, None] + row0) * np.arange(cols, dtype=np.int64)[None, :] % n_total
        w = np.exp((-2j if forward else 2j) * np.pi * idx / n_total)
        a = x.view(rows, cols).numpy()
        a *= w.astype(a.dtype)

    def all_to_all(self, dst, src, group):
        import torch.distributed as dist
        return dist.all_to_all_single(self.torch.view_as_real(dst), self.torch.view_as_real(src), group=group,
                                      async_op=True)


class DistributedFft:
    """Plan for one length-N transform over `world` ranks (N = n1 * n2, both divisible by world).
    `chunks` pieces per exchange (reduced to a divisor of the rows each rank receives; None = the default
    of the exchange mode)."""

    def __init__(self, n1, n2, rank, world, backend, group=None, chunks=None, exchange="nccl"):
        if n1 % world or n2 % world:
            raise ValueError("n1 and n2 must be divisible by the number of ranks")
        if exchange not in ("nccl", "peer", "fused"):
            raise ValueError("exchange must be 'nccl', 'peer' or 'fused'")
        self.n1, self.n2, self.n = n1, n2, n1 * n2
        self.rank, self.world, self.backend, self.group = rank, world, backend, group
        self.exchange = exchange if world > 1 else "nccl"
        # the NCCL formulation is pipelined in 8 pieces; the peer-memory path is not pipelined (1 piece)
        self.chunks = max(1, int(chunks)) if chunks else (8 if self.exchange == "nccl" else 1)
        self._send = self._recv = None
        self._bufs, self._tables = None, {}
        # "fused": peer memory as well, and the exchanges that follow row FFTs are folded into the FFTs' last stage
        self.fused, self.exchange = self.exchange == "fused", ("peer" if self.exchange == "fused" else self.exchange)
        if self.exchange == "peer":      # collective: every rank of the group constructs the plan
            self._bufs, tables = backend.peer_buffers(self.local_samples(), 2, rank, world, group)
            self._tables = {b.data_ptr(): t for b, t in zip(self._bufs, tables)}
            backend.barrier(group)

    def close(self):
        """Collective, exchange="peer" only: unmaps the peers' buffers and frees this rank's.  The tensors
        returned by buffers() are dead afterwards.  (Process exit releases everything as well.)"""
        if self.exchange == "peer" and self._bufs is not None:
            self.backend.barrier(self.group)          # nobody is still storing into a buffer that goes away
            self.backend.peer_release(self._bufs, [self._tables[b.data_ptr()] for b in self._bufs], self.rank)
            self._bufs, self._tables = None, {}

    def buffers(self):
        """The two work buffers to pass to transform(): peer-visible memory with exchange="peer"."""
        if self._bufs is None:
            self._bufs = [self.backend.empty(self.local_samples()) for _ in range(2)]
        return self._bufs

    def local_samples(self):
        return self.n // self.world

    def wire_bytes_per_exchange(self, itemsize):
        """Bytes each rank sends over NVLink per exchange."""
        return self.local_samples() * itemsize * (self.world - 1) // self.world

    def _pieces(self, rows_out):
        k = min(self.chunks, rows_out)
        while rows_out % k:
            k -= 1
        return k

    def _exchange(self, src, dst, rows_loc, cols, twiddle=None, then=None):
        """Transpose of the row-distributed global matrix [rows_loc * P][cols] (times the twiddle, if given):
        on return `dst` holds this rank's cols / P rows of the transposed matrix, each rows_loc * P long,
        and `then(rows, first_row)` has been applied to every piece of them.  `src` is left intact."""
        P, be = self.world, self.backend
        cb = cols // P                                  # result rows of this rank
        if P == 1:
            if twiddle is None:
                be.transpose(src, dst, rows_loc, cols)
            else:
                be.pack(src, dst, 1, rows_loc, cols, cols, 0, twiddle)
            if then:
                then(dst, 0)
            return dst
        if self._send is None or self._send.numel() != src.numel() or self._send.dtype != src.dtype:
            self._send, self._recv = be.empty_like(src), be.empty_like(src)
        K = self._pieces(cb)
        cbk = cb // K
        piece = P * cbk * rows_loc                      # samples per piece, on every side
        work = []
        for k in range(K):
            s = self._send[k * piece:(k + 1) * piece]
            be.pack(src, s, P, rows_loc, cbk, cols, k * cbk, twiddle)          # [P][cbk][rows_loc]
            work.append(be.all_to_all(self._recv[k * piece:(k + 1) * piece], s, self.group))
        for k in range(K):
            work[k].wait()
            d = dst[k * piece:(k + 1) * piece]                                 # rows k*cbk .. of the result
            be.swap_leading(self._recv[k * piece:(k + 1) * piece], d, P, cbk, rows_loc)   # [cbk][P * rows_loc]
            if then:
                then(d, k * cbk)
        return dst

    def _fft_then_exchange(self, src, dst, rows_loc, cols, fft_len, forward, twiddle):
        """Peer mode: the local FFTs over the rows of `src` and the exchange that follows them, software-
        pipelined over `chunks` row blocks: while block k travels over NVLink (side stream) block k+1 is being
        transformed (current stream).  A row of `src` is a complete FFT, so its exchange can start as soon as
        its block is done; the receivers need every block of every rank, hence one barrier at the end."""
        be, torch = self.backend, self.backend.torch
        table = self._table(dst)
        if fft_len and self.fused and be.can_fuse(src, fft_len, rows_loc):
            be.fft_rows_exchange(src, table, self.world, self.rank, rows_loc, fft_len, forward, twiddle)
            be.barrier(self.group)
            return dst
        K = self._pieces(rows_loc) if fft_len else 1
        rows_k = rows_loc // K
        main, side = (torch.cuda.current_stream(), be.side_stream()) if K > 1 else (None, None)
        for k in range(K):
            if fft_len:
                be.fft_rows(src[k * rows_k * cols:(k + 1) * rows_k * cols], fft_len, forward)
            if K == 1:
                be.exchange(src, table, self.world, self.rank, rows_loc, cols // self.world, twiddle)
                break
            side.wait_stream(main)
            with torch.cuda.stream(side):
                be.exchange(src, table, self.world, self.rank, rows_loc, cols // self.world, twiddle,
                            first=k * rows_k, count=rows_k)
        if K > 1:
            main.wait_stream(side)
        be.barrier(self.group)
        return dst

    def _table(self, dst):
        table = self._tables.get(dst.data_ptr())
        if table is None:
            raise ValueError("exchange='peer': transform() needs the plan's own buffers (plan.buffers())")
        return table

    def transform(self, x, scratch, forward=True, natural_order=True):
        """x: this rank's N/P samples (its block of the natural order), scratch: same size.  Both are
        clobbered; returns the one holding this rank's block of the result (unscaled in both directions:
        Transform.Fft / Transform.UnscaledIfft).

        natural_order=False skips the third exchange (a third of the NVLink traffic): the result stays
        transposed, rank r holding rows k1 in [r*N1/P, (r+1)*N1/P) of Y[k1][k2] = X[k1 + N1*k2] -- enough for
        callers that can consume the spectrum in that order."""
        P, be = self.world, self.backend
        n1, n2 = self.n1, self.n2
        r1, r2 = n1 // P, n2 // P
        if self.exchange == "peer":
            # Entry barrier: step 1 stores straight into every peer's `scratch`, which may hold the peer's previous
            # result (natural order) that its stream is still reading: no rank may start storing before every rank's
            # stream has reached this call.  Stream-ordered, one element: negligible next to the transform.
            be.barrier(self.group)
            a = self._fft_then_exchange(x, scratch, r1, n2, 0, forward, None)                          # [n2_loc][n1]
            b = self._fft_then_exchange(a, x, r2, n1, n1, forward, (forward, self.rank * r2, self.n))  # [k1_loc][n2]
            if not natural_order:
                be.fft_rows(b, n2, forward)
                return b                                                                               # [k1_loc][k2]
            return self._fft_then_exchange(b, scratch, r1, n2, n2, forward, None)                      # [k2_loc][k1]
        a = self._exchange(x, scratch, r1, n2, then=lambda rows, first: be.fft_rows(rows, n1, forward))   # [n2_loc][k1]
        b = self._exchange(a, x, r2, n1, twiddle=(forward, self.rank * r2, self.n),
                           then=lambda rows, first: be.fft_rows(rows, n2, forward))                       # [k1_loc][k2]
        if not natural_order:
            return b
        return self._exchange(b, scratch, r1, n2)                                                         # [k2_loc][k1]

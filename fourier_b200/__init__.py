"""fourier_b200 -- Python mirror of the `fourier` crate's public surface over libfourier.so.

The product is the C-ABI library (include/fourier.h, include/fourier_b200.h; hand-written sm_90a
CUDA).  This module is the thin host-side binding used by the tests and the benchmark; it mirrors the
reference's operator interface name for name:

    reference (Rust)                                      here
    fourier::Transform {Fft, Ifft, UnscaledIfft,          Transform (IntEnum, same C codes,
      SqrtScaledFft, SqrtScaledIfft}  fft.rs:5-16           is_forward / inverse: fft.rs:20-36)
    fourier::Fft trait  fft.rs:40-82                      class Fft: size, transform_in_place,
                                                            transform, fft_in_place, ifft_in_place, fft, ifft
    fourier::create_fft_f32 / create_fft_f64              create_fft_f32 / create_fft_f64
      fourier/src/lib.rs:31-60
    (no counterpart)                                      RealFft, create_rfft_f32 / create_rfft_f64:
                                                            batched rfft / irfft of real rows
    (no counterpart)                                      RealFft.convolve: y = irfft(rfft(x) * H) of real
                                                            rows, one or several spectra H, one call
    (no counterpart)                                      RealFft.convolve_linear: linear convolution of real
                                                            rows of any length with K <= N taps (scipy's
                                                            full / same / valid), overlap-save in one call
    (no counterpart)                                      RealFft.stft / istft / stft_frames: short-time Fourier
                                                            transform of real rows and its overlap-add inverse
                                                            (torch.stft / istft, frames frame-major)
    (no counterpart)                                      RealFft.mel_spectrogram: |stft|^p through a caller's
                                                            mel filter bank (torchaudio's MelSpectrogram,
                                                            frames frame-major), the spectrum kept on chip
    (no counterpart)                                      RealFft.mfcc: log mels, a top_db clamp and a DCT matrix
                                                            (torchaudio's MFCC, librosa's mfcc, Whisper's
                                                            log-mel), the mels kept on chip
    (no counterpart)                                      RealFft.welch: Welch's power spectral density of real
                                                            rows (scipy.signal.welch), frames summed on chip
    (no counterpart)                                      RealFft.csd / coherence: cross-spectral density and
                                                            magnitude-squared coherence of real row pairs
                                                            (scipy.signal.csd / coherence), frames summed on chip
    (no counterpart)                                      RealFft.dct / idct: discrete cosine transforms of real
                                                            rows, types 2 and 3 (scipy.fft.dct / idct; torch has
                                                            none)
    (no counterpart)                                      RealFft.hilbert: analytic signal of real rows
                                                            (scipy.signal.hilbert; torch has none)
    (no counterpart)                                      RealFft.envelope: its modulus, the amplitude envelope
                                                            (numpy.abs(scipy.signal.hilbert))
    (no counterpart)                                      RealFft.dct4: the type-IV DCT of real rows
                                                            (scipy.fft.dct(type=4))
    (no counterpart)                                      RealFft.mdct / imdct / mdct_frames: the modified discrete
                                                            cosine transform of real rows and its overlap-add inverse
                                                            (tf.signal.mdct / inverse_mdct; torch has none)

Buffers are numpy arrays (host memory: staged over PCIe by the library) or torch CUDA tensors
(device memory: transformed in HBM on torch's current stream).  A leading batch dimension is
allowed: shape (..., size) means prod(...) independent transforms.  There is no CPU fallback.
"""
import ctypes
import enum
import math

import numpy as np

from . import _lib

__all__ = ["Transform", "Fft", "create_fft_f32", "create_fft_f64", "RealFft", "create_rfft_f32", "create_rfft_f64",
           "set_device", "fill_input", "lib_path"]


class Transform(enum.IntEnum):
    """fourier-algorithms/src/fft.rs:5-16; integer values are the C codes of fourier.h:30-36."""
    Fft = 0
    Ifft = 1
    UnscaledIfft = 2
    SqrtScaledFft = 3
    SqrtScaledIfft = 4

    def is_forward(self):
        return self in (Transform.Fft, Transform.SqrtScaledFft)

    def inverse(self):
        return {Transform.Fft: Transform.Ifft, Transform.Ifft: Transform.Fft,
                Transform.SqrtScaledFft: Transform.SqrtScaledIfft,
                Transform.SqrtScaledIfft: Transform.SqrtScaledFft,
                Transform.UnscaledIfft: None}[self]


def _is_torch(x):
    return type(x).__module__.startswith("torch")


class Fft:
    """A plan for one transform size: the `Box<dyn Fft<Real = T> + Send>` of the reference."""

    def __init__(self, size, real, general=False):
        if real not in ("f32", "f64"):
            raise ValueError("real must be 'f32' or 'f64'")
        self.real = real
        self._t = "float" if real == "f32" else "double"
        self._np_dtype = np.dtype(np.complex64 if real == "f32" else np.complex128)
        L = _lib.load()
        ctor = getattr(L, f"fourier_b200_create_general_{self._t}" if general else f"fourier_create_{self._t}")
        self._plan = ctor(int(size))
        if not self._plan:
            raise RuntimeError(f"fourier_create_{self._t}({size}) returned NULL: {_lib.last_error()}")
        self._size = int(size)
        self._device = self.info()["device"]

    # -- lifetime -------------------------------------------------------------------------------
    def close(self):
        p, self._plan = getattr(self, "_plan", None), None
        if p:
            getattr(_lib.load(), f"fourier_destroy_{self._t}")(p)

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # -- Fft trait --------------------------------------------------------------------------------
    def size(self):
        return self._size

    def info(self):
        i = _lib.PlanInfo()
        getattr(_lib.load(), f"fourier_b200_plan_info_{self._t}")(self._plan, ctypes.byref(i))
        d = {f: getattr(i, f) for f, _ in i._fields_}
        d["path_name"] = _lib.load().fourier_b200_path_name(i.path).decode()
        d["inner_path_name"] = _lib.load().fourier_b200_path_name(i.inner_path).decode()
        return d

    def kernel_name(self):
        """The kernel that moves (nearly) all of this plan's bytes, as a profiler lists it."""
        return getattr(_lib.load(), f"fourier_b200_plan_kernel_{self._t}")(self._plan).decode()

    def _describe(self, x):
        """-> (pointer, batch, is_device, stream)"""
        if _is_torch(x):
            import torch
            want = torch.complex64 if self.real == "f32" else torch.complex128
            if x.dtype != want:
                raise TypeError(f"expected {want}, got {x.dtype}")
            if not x.is_contiguous():
                raise ValueError("buffers must be contiguous")
            if x.shape[-1] != self._size:
                raise ValueError(f"last dimension must be {self._size}")  # assert_eq!, fft.rs:57-58
            batch = x.numel() // self._size
            if x.is_cuda:
                if x.device.index != self._device:
                    raise ValueError(f"plan lives on cuda:{self._device}, buffer on {x.device}")
                return x.data_ptr(), batch, True, torch.cuda.current_stream(x.device).cuda_stream
            return x.data_ptr(), batch, False, None
        if not isinstance(x, np.ndarray):
            raise TypeError("buffers must be numpy arrays or torch tensors")
        if x.dtype != self._np_dtype:
            raise TypeError(f"expected {self._np_dtype}, got {x.dtype}")
        if not x.flags.c_contiguous:
            raise ValueError("buffers must be C-contiguous")
        if x.shape[-1] != self._size:
            raise ValueError(f"last dimension must be {self._size}")
        return x.ctypes.data, x.size // self._size, False, None

    def _run(self, src, dst, transform):
        code = int(Transform(transform))
        pi, bi, di, si = self._describe(src)
        po, bo, do_, so = self._describe(dst)
        if bi != bo:
            raise ValueError("input and output hold a different number of transforms")
        if di != do_:
            raise ValueError("input and output must both be host or both be device buffers")
        L = _lib.load()
        if di:
            rc = getattr(L, f"fourier_b200_transform_batch_async_{self._t}")(self._plan, pi, po, bi, code, si)
        else:
            rc = getattr(L, f"fourier_b200_transform_batch_{self._t}")(self._plan, pi, po, bi, code)
        if rc != 0:
            raise RuntimeError(f"transform failed (cuda error {rc}): {_lib.last_error()}")

    def transform_in_place(self, input, transform):
        """Fft::transform_in_place (fft.rs:48)."""
        self._run(input, input, transform)

    def transform(self, input, output, transform):
        """Fft::transform (fft.rs:51-61): out of place, input untouched."""
        self._run(input, output, transform)

    def fft_in_place(self, input):
        self.transform_in_place(input, Transform.Fft)

    def ifft_in_place(self, input):
        self.transform_in_place(input, Transform.Ifft)

    def fft(self, input, output):
        self.transform(input, output, Transform.Fft)

    def ifft(self, input, output):
        self.transform(input, output, Transform.Ifft)

    # -- distributed six-step transform: row FFTs + exchange in one pass (csrc/dist_fft.cu) -----------------
    def fft_rows_exchange(self, rows, outs, out_ld, out_off, forward=True, twiddle=None):
        """FFT of the contiguous rows of the CUDA tensor `rows` (unscaled) whose last register stage stores the result
        transposed into the buffers `outs` (a ctypes array of device pointers, one per destination rank):
        outs[q][c*out_ld + out_off + r] = FFT(rows[r])[q*cb + c] * w_Ntot^{(row0 + r)*(q*cb + c)}, cb = size / len(outs);
        twiddle = None or (row0, Ntot).  Two-pass plans only (raises NotImplementedError otherwise)."""
        ptr, count, on_device, stream = self._describe(rows)
        if not on_device:
            raise ValueError("fft_rows_exchange needs CUDA tensors")
        mode, row0, n_total = (0, 0, 0) if twiddle is None else ((1 if forward else 2), int(twiddle[0]), int(twiddle[1]))
        rc = getattr(_lib.load(), f"fourier_b200_fft_rows_exchange_{self._t}")(
            self._plan, ptr, count, int(bool(forward)), outs, len(outs), int(out_ld), int(out_off), mode, row0,
            n_total, stream)
        if rc == 801:
            raise NotImplementedError(_lib.last_error())
        if rc != 0:
            raise RuntimeError(f"fft_rows_exchange failed (cuda error {rc}): {_lib.last_error()}")

    # -- the raw single-transform reference ABI (for the boundary tests) ------------------------------
    def c_transform(self, input, output, transform):
        pi, _, _, _ = self._describe(input)
        po, _, _, _ = self._describe(output)
        getattr(_lib.load(), f"fourier_transform_{self._t}")(self._plan, pi, po, int(transform))

    def c_transform_in_place(self, input, transform):
        pi, _, _, _ = self._describe(input)
        getattr(_lib.load(), f"fourier_transform_in_place_{self._t}")(self._plan, pi, int(transform))


def create_fft_f32(size, general=False):
    """fourier::create_fft_f32 (fourier/src/lib.rs:31-43)."""
    return Fft(size, "f32", general=general)


def create_fft_f64(size, general=False):
    """fourier::create_fft_f64 (fourier/src/lib.rs:49-60)."""
    return Fft(size, "f64", general=general)


class RealFft:
    """A plan for real-input transforms of one length N (numpy's rfft / irfft, batched): reals of shape (..., N) and
    spectra of shape (..., N//2+1), with equal leading dimensions.  rfft / irfft are out of place only; convolve
    (irfft(rfft(x) * H) in one call) may run in place; convolve_linear filters rows of any length, out of place."""

    def __init__(self, size, real):
        if real not in ("f32", "f64"):
            raise ValueError("real must be 'f32' or 'f64'")
        self.real = real
        self._t = "float" if real == "f32" else "double"
        self._np = {"real": np.dtype(np.float32 if real == "f32" else np.float64),
                    "spec": np.dtype(np.complex64 if real == "f32" else np.complex128)}
        self._plan = getattr(_lib.load(), f"fourier_b200_rfft_create_{self._t}")(int(size))
        if not self._plan:
            raise RuntimeError(f"fourier_b200_rfft_create_{self._t}({size}) returned NULL: {_lib.last_error()}")
        self._size = int(size)
        self._device = self.info()["device"]

    def close(self):
        p, self._plan = getattr(self, "_plan", None), None
        if p:
            getattr(_lib.load(), f"fourier_b200_rfft_destroy_{self._t}")(p)

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def size(self):
        return self._size

    def info(self):
        i = _lib.PlanInfo()
        getattr(_lib.load(), f"fourier_b200_rfft_info_{self._t}")(self._plan, ctypes.byref(i))
        d = {f: getattr(i, f) for f, _ in i._fields_}
        d["path_name"] = _lib.load().fourier_b200_path_name(i.path).decode()
        d["inner_path_name"] = _lib.load().fourier_b200_path_name(i.inner_path).decode()
        return d

    def kernel_name(self):
        """The real kernel of the plan, and for the half-length and full-length paths the inner plan's kernel."""
        return getattr(_lib.load(), f"fourier_b200_rfft_kernel_{self._t}")(self._plan).decode()

    def _describe(self, x, kind, last=None):
        """kind 'real' (last dimension N, or `last`) or 'spec' (N//2+1) -> (pointer, leading shape, is_device,
        stream)"""
        if last is None:
            last = self._size if kind == "real" else self._size // 2 + 1
        if _is_torch(x):
            import torch
            want = {("real", "f32"): torch.float32, ("real", "f64"): torch.float64,
                    ("spec", "f32"): torch.complex64, ("spec", "f64"): torch.complex128}[(kind, self.real)]
            if x.dtype != want:
                raise TypeError(f"expected {want}, got {x.dtype}")
            if not x.is_contiguous():
                raise ValueError("buffers must be contiguous")
            if x.dim() == 0 or x.shape[-1] != last:
                raise ValueError(f"last dimension must be {last}")
            if x.is_cuda:
                if x.device.index != self._device:
                    raise ValueError(f"plan lives on cuda:{self._device}, buffer on {x.device}")
                return x.data_ptr(), tuple(x.shape[:-1]), True, torch.cuda.current_stream(x.device).cuda_stream
            return x.data_ptr(), tuple(x.shape[:-1]), False, None
        if not isinstance(x, np.ndarray):
            raise TypeError("buffers must be numpy arrays or torch tensors")
        if x.dtype != self._np[kind]:
            raise TypeError(f"expected {self._np[kind]}, got {x.dtype}")
        if not x.flags.c_contiguous:
            raise ValueError("buffers must be C-contiguous")
        if x.ndim == 0 or x.shape[-1] != last:
            raise ValueError(f"last dimension must be {last}")
        return x.ctypes.data, tuple(x.shape[:-1]), False, None

    def _run(self, direction, src, dst, transform):
        code = int(Transform(transform))
        kinds = ("real", "spec") if direction == "forward" else ("spec", "real")
        pi, li, di, si = self._describe(src, kinds[0])
        po, lo, do_, _ = self._describe(dst, kinds[1])
        if li != lo:
            raise ValueError(f"leading dimensions differ: {li} and {lo}")
        if di != do_:
            raise ValueError("input and output must both be host or both be device buffers")
        batch = int(np.prod(li, dtype=np.int64))
        self._call(f"rfft_{direction}", f"real {direction} transform", di, si, pi, po, batch, code)

    def _call(self, symbol, what, on_device, stream, *args):
        """fourier_b200_<symbol>_<t>(plan, *args), or on device buffers fourier_b200_<symbol>_async_<t>(plan, *args,
        stream); RuntimeError naming `what` if it fails."""
        L = _lib.load()
        if on_device:
            rc = getattr(L, f"fourier_b200_{symbol}_async_{self._t}")(self._plan, *args, stream)
        else:
            rc = getattr(L, f"fourier_b200_{symbol}_{self._t}")(self._plan, *args)
        if rc != 0:
            raise RuntimeError(f"{what} failed (cuda error {rc}): {_lib.last_error()}")

    @staticmethod
    def _check_resolved(*buffers):
        for x in buffers:
            if _is_torch(x) and (x.is_conj() or x.is_neg()):
                raise ValueError("torch tensors with the conj or neg bit set hold unconjugated data: "
                                 "pass x.resolve_conj() (and resolve_neg()) instead")

    def convolve(self, input, spectrum, output):
        """output = numpy.fft.irfft(numpy.fft.rfft(input) * spectrum, n=N): circular convolution of every row of
        `input` (shape (..., N)) with the filter whose rfft is `spectrum` (shape (..., N//2+1), this plan's rfft
        layout).  The spectrum's leading shape must equal a trailing part of the input's leading shape and is
        broadcast over the rest: () means one filter for all rows, (C,) one per channel for input (B, C, N), the
        input's whole leading shape one per row.  `output` has the input's shape and may be `input`
        itself.  Correlation: pass conj(H), resolved (spectrum.conj().resolve_conj() for torch)."""
        self._check_resolved(input, spectrum, output)
        pi, li, di, si = self._describe(input, "real")
        ps, ls, ds, _ = self._describe(spectrum, "spec")
        po, lo, do_, _ = self._describe(output, "real")
        if li != lo:
            raise ValueError(f"input and output shapes differ: {li} and {lo}")
        if len(ls) > len(li) or tuple(li[len(li) - len(ls):]) != ls:
            raise ValueError(f"spectrum leading shape {ls} is not a trailing part of the input's {li}")
        if not (di == ds == do_):
            raise ValueError("input, spectrum and output must all be host or all be device buffers")
        batch = int(np.prod(li, dtype=np.int64))
        rows = int(np.prod(ls, dtype=np.int64))
        self._call("convolve_real", "real convolution", di, si, pi, ps, rows, po, batch)

    LINEAR_MODES = {"full": 0, "same": 1, "valid": 2}

    def convolve_linear(self, input, spectrum, taps, output, mode="full"):
        """output = scipy.signal.convolve(input, h, mode) for every row of `input` (shape (..., L), any L >= 1), where
        `spectrum` (shape (..., N//2+1), this plan's rfft layout) is rfft(h, n=N) of `taps` = K <= N taps h.  `output`
        has shape (..., out_len): out_len = L + K - 1 (mode "full"), L ("same") or L - K + 1 ("valid", L >= K).  The
        spectrum broadcasts over the input's leading shape as in convolve.  Rows are filtered by overlap-save in
        segments of N - K + 1 outputs, so N should be a few times K.  If irfft(spectrum) has non-zero samples beyond
        the first K, the result is unspecified.  Out of place only; correlation: pass conj(H), resolved."""
        self._check_resolved(input, spectrum, output)
        if mode not in self.LINEAR_MODES:
            raise ValueError(f"mode must be one of {sorted(self.LINEAR_MODES)}, got {mode!r}")
        taps = int(taps)
        if not 1 <= taps <= self._size:
            raise ValueError(f"taps must be in [1, {self._size}], got {taps}")
        in_len = input.shape[-1] if getattr(input, "ndim", 0) > 0 else 0
        if in_len < 1:
            raise ValueError("input rows must hold at least one sample")
        if mode == "valid" and in_len < taps:
            raise ValueError(f"mode 'valid' needs rows of at least taps = {taps} samples, got {in_len}")
        out_len = {"full": in_len + taps - 1, "same": in_len, "valid": in_len - taps + 1}[mode]
        pi, li, di, si = self._describe(input, "real", last=in_len)
        ps, ls, ds, _ = self._describe(spectrum, "spec")
        if getattr(output, "ndim", 0) == 0 or output.shape[-1] != out_len:
            raise ValueError(f"output rows must hold out_len = {out_len} samples for mode {mode!r} "
                             f"(L = {in_len}, taps = {taps})")
        po, lo, do_, _ = self._describe(output, "real", last=out_len)
        if li != lo:
            raise ValueError(f"input and output leading shapes differ: {li} and {lo}")
        if len(ls) > len(li) or tuple(li[len(li) - len(ls):]) != ls:
            raise ValueError(f"spectrum leading shape {ls} is not a trailing part of the input's {li}")
        if not (di == ds == do_):
            raise ValueError("input, spectrum and output must all be host or all be device buffers")
        batch = int(np.prod(li, dtype=np.int64))
        rows = int(np.prod(ls, dtype=np.int64))
        self._call("linear_convolve_real", "linear convolution", di, si, pi, in_len, ps, rows, taps,
                   self.LINEAR_MODES[mode], po, batch)

    STFT_PAD_MODES = {"constant": 1, "reflect": 2}

    def stft_frames(self, in_len, hop, center=True):
        """F, the number of frames `stft` makes of rows of in_len samples: 1 + (in_len + 2 pad - N) // hop with
        pad = N//2 if center else 0."""
        pad = self._size // 2 if center else 0
        return 1 + (int(in_len) + 2 * pad - self._size) // int(hop)

    def _framing(self, input, window, hop, center, pad_mode):
        """The framing of stft and mel_spectrogram: checks pad_mode, hop and the row length against N, and describes
        the input and the window -> (hop, boundary, in_len, frames, (pointer, leading shape, is_device, stream) of the
        input, (pointer, is_device) of the window)"""
        if center and pad_mode not in self.STFT_PAD_MODES:
            raise ValueError(f"pad_mode must be one of {sorted(self.STFT_PAD_MODES)}, got {pad_mode!r}")
        hop = int(hop)
        if hop < 1:
            raise ValueError(f"hop must be at least 1, got {hop}")
        boundary = self.STFT_PAD_MODES[pad_mode] if center else 0
        n = self._size
        in_len = input.shape[-1] if getattr(input, "ndim", 0) > 0 else 0
        if in_len < 1:
            raise ValueError("input rows must hold at least one sample")
        if boundary == 0 and in_len < n:
            raise ValueError(f"center=False needs rows of at least N = {n} samples, got {in_len}")
        if boundary == 2 and in_len <= n // 2:
            raise ValueError(f"pad_mode 'reflect' needs rows of more than N//2 = {n // 2} samples, got {in_len}")
        frames = self.stft_frames(in_len, hop, center)
        src = self._describe(input, "real", last=in_len)
        pw, lw, dw, _ = self._describe(window, "real")
        if lw != ():
            raise ValueError(f"window must hold exactly N = {n} reals, got shape {tuple(window.shape)}")
        return hop, boundary, in_len, frames, src, (pw, dw)

    def stft(self, input, window, hop, output, center=True, pad_mode="reflect"):
        """Short-time Fourier transform of every row of `input` (shape (..., L)): frames of N = size() samples every
        `hop`, times `window` (N reals; zero-pad a shorter one), through rfft.  `output` has shape (..., F, N//2+1),
        F = stft_frames(L, hop, center), frame-major: this is torch.stft(x, N, hop, window=window, center=center,
        pad_mode=pad_mode, return_complex=True).transpose(-1, -2).  With center the rows are padded by N//2 on both
        sides, with zeros (pad_mode "constant") or mirrored without repeating the edge ("reflect", needs L > N//2);
        pad_mode is ignored without center, which needs L >= N.  Out of place only."""
        self._check_resolved(input, window, output)
        hop, boundary, in_len, frames, (pi, li, di, si), (pw, dw) = self._framing(input, window, hop, center, pad_mode)
        n = self._size
        if getattr(output, "ndim", 0) < 2 or output.shape[-2] != frames:
            raise ValueError(f"output must have shape (..., {frames}, {n // 2 + 1}) (F = {frames} frames)")
        po, lo, do_, _ = self._describe(output, "spec")
        if li != lo[:-1]:
            raise ValueError(f"input and output leading shapes differ: {li} and {lo[:-1]}")
        if not (di == dw == do_):
            raise ValueError("input, window and output must all be host or all be device buffers")
        batch = int(np.prod(li, dtype=np.int64))
        self._call("stft", "stft", di, si, pi, in_len, pw, hop, boundary, po, batch)

    def mel_spectrogram(self, input, window, hop, filters, output, power=2, center=True, pad_mode="reflect"):
        """Mel spectrogram of every row of `input` (shape (..., L)) with stft's framing: output[..., f, m] =
        sum_k filters[m, k] * |X_f[k]|**power, X_f the stft of frame f (same window, hop, center and pad_mode), power 1
        or 2, no log.  `filters` has shape (n_mels, N//2+1) (librosa's and Whisper's layout; pass torchaudio's
        melscale_fbanks(...).T.contiguous()), any n_mels >= 1 and any real weights.  `output` has shape
        (..., F, n_mels), F = stft_frames(L, hop, center): with power 2 and torchaudio's own window and bank this is
        torchaudio.transforms.MelSpectrogram(...)(x).transpose(-1, -2).  The spectrum stays on chip where the plan's
        path allows.  Out of place only."""
        self._check_resolved(input, window, filters, output)
        if power not in (1, 2):
            raise ValueError(f"power must be 1 or 2, got {power!r}")
        hop, boundary, in_len, frames, (pi, li, di, si), (pw, dw) = self._framing(input, window, hop, center, pad_mode)
        n = self._size
        if getattr(filters, "ndim", 0) != 2:
            raise ValueError(f"filters must have shape (n_mels, {n // 2 + 1})")
        pf, lf, df, _ = self._describe(filters, "real", last=n // 2 + 1)
        n_mels = lf[0]
        if n_mels < 1:
            raise ValueError("filters must hold at least one mel row")
        if getattr(output, "ndim", 0) < 2 or output.shape[-2] != frames:
            raise ValueError(f"output must have shape (..., {frames}, {n_mels}) (F = {frames} frames)")
        po, lo, do_, _ = self._describe(output, "real", last=n_mels)
        if li != lo[:-1]:
            raise ValueError(f"input and output leading shapes differ: {li} and {lo[:-1]}")
        if not (di == dw == df == do_):
            raise ValueError("input, window, filters and output must all be host or all be device buffers")
        batch = int(np.prod(li, dtype=np.int64))
        if batch == 0:
            return   # nothing to do; an empty torch tensor has no data pointer for the C entry point
        self._call("mel_spectrogram", "mel spectrogram", di, si, pi, in_len, pw, hop, boundary, int(power), pf, n_mels,
                   po, batch)

    def mfcc(self, input, window, hop, filters, dct, output, power=2, center=True, pad_mode="reflect",
             log_scale=10.0 / math.log(10.0), log_floor=1e-10, log_offset=0.0, top_db=80.0, top_db_rows=1, bias=0.0):
        """MFCC or log-mel spectrogram of every row of `input` (shape (..., L)), from mel_spectrogram's mels
        mel[..., f, m] (same framing, window, power and filters), all in the plan's precision:
        lm = log_scale * ln(max(mel + log_offset, log_floor)); with top_db not None, lc = max(lm, max_g(lm) - top_db)
        where max_g is taken over clamp group g, top_db_rows consecutive rows of the flattened leading shape (their
        count must be a multiple of it), all their frames and mels; else lc = lm.  Then output[..., f, j] = bias +
        sum_m lc[..., f, m] * dct[m, j] (ascending m), or lc + bias with dct None (the log-mel spectrogram).  `dct` has
        shape (n_mels, n_out): torchaudio's create_dct(n_mfcc, n_mels, "ortho"), or librosa's
        scipy.fft.dct(np.eye(n_mels), norm="ortho")[:, :n_mfcc]; fold a lifter into its columns.  `output` has shape
        (..., F, n_out), frame-major: the transpose of torchaudio's layout.
        The defaults are torchaudio.transforms.MFCC(log_mels=False) for one-channel input; for input (..., C, L) pass
        top_db_rows = C, as torchaudio takes the max over each item's channels.  MFCC(log_mels=True): log_scale=1,
        log_floor = the smallest normal of the dtype, log_offset=1e-6, top_db=None.  librosa.feature.mfcc: top_db_rows
        = all rows.  Whisper's log-mel: log_scale=1/(4 ln 10), log_floor=1e-10, top_db=2, dct=None, bias=1; Whisper
        drops the last frame before its max and this takes the max over all F frames, so the two agree on frames
        0 .. F-2 unless the last frame holds the row's maximum.  The mels stay on chip where the plan's path allows.
        Out of place only."""
        self._check_resolved(input, window, filters, dct, output)
        if power not in (1, 2):
            raise ValueError(f"power must be 1 or 2, got {power!r}")
        log_scale, log_floor, log_offset, bias = float(log_scale), float(log_floor), float(log_offset), float(bias)
        if not math.isfinite(log_offset):
            raise ValueError(f"log_offset must be finite, got {log_offset!r}")
        if not math.isfinite(bias):
            raise ValueError(f"bias must be finite, got {bias!r}")
        if not (math.isfinite(log_floor) and log_floor > 0):
            raise ValueError(f"log_floor must be finite and positive, got {log_floor!r}")
        if not (math.isfinite(log_scale) and log_scale > 0):
            raise ValueError(f"log_scale must be finite and positive, got {log_scale!r}")
        top_db = math.inf if top_db is None else float(top_db)
        if not top_db >= 0:
            raise ValueError(f"top_db must be None or >= 0, got {top_db!r}")
        top_db_rows = int(top_db_rows)
        if top_db_rows < 1:
            raise ValueError(f"top_db_rows must be at least 1, got {top_db_rows}")
        hop, boundary, in_len, frames, (pi, li, di, si), (pw, dw) = self._framing(input, window, hop, center, pad_mode)
        n = self._size
        if getattr(filters, "ndim", 0) != 2:
            raise ValueError(f"filters must have shape (n_mels, {n // 2 + 1})")
        pf, lf, df, _ = self._describe(filters, "real", last=n // 2 + 1)
        n_mels = lf[0]
        if n_mels < 1:
            raise ValueError("filters must hold at least one mel row")
        if dct is None:
            n_out, pd, dd = n_mels, None, di
        else:
            if getattr(dct, "ndim", 0) != 2 or dct.shape[0] != n_mels or dct.shape[1] < 1:
                raise ValueError(f"dct must have shape ({n_mels}, n_out) with n_out >= 1")
            n_out = int(dct.shape[1])
            pd, _, dd, _ = self._describe(dct, "real", last=n_out)
        if getattr(output, "ndim", 0) < 2 or output.shape[-2] != frames:
            raise ValueError(f"output must have shape (..., {frames}, {n_out}) (F = {frames} frames)")
        po, lo, do_, _ = self._describe(output, "real", last=n_out)
        if li != lo[:-1]:
            raise ValueError(f"input and output leading shapes differ: {li} and {lo[:-1]}")
        if not (di == dw == df == dd == do_):
            raise ValueError("input, window, filters, dct and output must all be host or all be device buffers")
        batch = int(np.prod(li, dtype=np.int64))
        if math.isfinite(top_db) and batch % top_db_rows:
            raise ValueError(f"{batch} rows do not form whole clamp groups of top_db_rows = {top_db_rows}")
        if batch == 0:
            return   # nothing to do; an empty torch tensor has no data pointer for the C entry point
        self._call("mfcc", "mfcc", di, si, pi, in_len, pw, hop, boundary, int(power), pf, n_mels, log_offset,
                   log_floor, log_scale, top_db, top_db_rows, pd, n_out, bias, po, batch)

    DCT_NORMS = {"backward": 0, "ortho": 1, "forward": 2}

    def dct(self, input, output, type=2, norm="backward"):
        """output = scipy.fft.dct(input, type=type, norm=norm) along the last axis: the discrete cosine transform of
        type 2 or 3 of every row of `input` (shape (..., N), real dtype), with scipy's norms "backward", "ortho" and
        "forward" (orthogonalize=True).  `output` has the input's shape and may be `input` itself."""
        self._check_resolved(input, output)
        if type not in (2, 3) or isinstance(type, bool):
            raise ValueError(f"type must be 2 or 3, got {type!r}")
        if not isinstance(norm, str) or norm not in self.DCT_NORMS:
            raise ValueError(f"norm must be one of {sorted(self.DCT_NORMS)}, got {norm!r}")
        pi, li, di, si = self._describe(input, "real")
        po, lo, do_, _ = self._describe(output, "real")
        if li != lo:
            raise ValueError(f"input and output shapes differ: {li} and {lo}")
        if di != do_:
            raise ValueError("input and output must both be host or both be device buffers")
        batch = int(np.prod(li, dtype=np.int64))
        if batch == 0:
            return   # nothing to do; an empty torch tensor has no data pointer for the C entry point
        self._call("dct", "dct", di, si, pi, po, batch, int(type), self.DCT_NORMS[norm])

    def idct(self, input, output, type=2, norm="backward"):
        """output = scipy.fft.idct(input, type=type, norm=norm): the dct of type 5 - type with the norms "backward" and
        "forward" swapped, so that idct(dct(x, type, norm), type, norm) is x."""
        if not isinstance(norm, str) or norm not in self.DCT_NORMS:
            raise ValueError(f"norm must be one of {sorted(self.DCT_NORMS)}, got {norm!r}")
        if type not in (2, 3) or isinstance(type, bool):
            raise ValueError(f"type must be 2 or 3, got {type!r}")
        swapped = {"backward": "forward", "forward": "backward", "ortho": "ortho"}[norm]
        self.dct(input, output, type=5 - type, norm=swapped)

    def hilbert(self, input, output):
        """output = scipy.signal.hilbert(input, axis=-1): the analytic signal x + i y of every row of `input` (shape
        (..., N), real dtype), y = irfft(G * rfft(x), n=N) with G = -i on the bins 0 < k < N/2 and 0 at k = 0 and
        (N even) N/2.  `output` is complex with the input's shape and must not overlap it.  Its real part is a copy of
        the input, bit for bit."""
        self._hilbert(input, output, "spec", 0)

    def envelope(self, input, output):
        """output = numpy.abs(scipy.signal.hilbert(input, axis=-1)): the amplitude envelope sqrt(x^2 + y^2) of every
        row of `input` (shape (..., N), real dtype).  `output` is real with the input's shape and may be `input`."""
        self._hilbert(input, output, "real", 1)

    def _hilbert(self, input, output, out_kind, code):
        self._check_resolved(input, output)
        pi, li, di, si = self._describe(input, "real")
        po, lo, do_, _ = self._describe(output, out_kind, last=self._size)
        if li != lo:
            raise ValueError(f"input and output shapes differ: {li} and {lo}")
        if di != do_:
            raise ValueError("input and output must both be host or both be device buffers")
        batch = int(np.prod(li, dtype=np.int64))
        if batch == 0:
            return   # nothing to do; an empty torch tensor has no data pointer for the C entry point
        self._call("hilbert", "hilbert" if code == 0 else "envelope", di, si, pi, po, batch, code)

    def _check_norm(self, norm):
        if not isinstance(norm, str) or norm not in self.DCT_NORMS:
            raise ValueError(f"norm must be one of {sorted(self.DCT_NORMS)}, got {norm!r}")
        if self._size % 2:
            raise ValueError(f"the type-IV DCT and the MDCT need an even plan length, got N = {self._size}")
        return self.DCT_NORMS[norm]

    def dct4(self, input, output, norm="backward"):
        """output = scipy.fft.dct(input, type=4, norm=norm) along the last axis: the type-IV DCT y[k] = 2 h sum_n x[n]
        cos(pi (2n+1)(2k+1) / (4N)) of every row of `input` (shape (..., N), real dtype, N even), h = 1, 1/sqrt(2N) or
        1/(2N) for the norms "backward", "ortho" and "forward".  `output` has the input's shape and may be `input`
        itself.  The inverse is dct4 with "backward" and "forward" swapped (scipy.fft.idct(type=4)); "ortho" is its own
        inverse."""
        self._check_resolved(input, output)
        code = self._check_norm(norm)
        pi, li, di, si = self._describe(input, "real")
        po, lo, do_, _ = self._describe(output, "real")
        if li != lo:
            raise ValueError(f"input and output shapes differ: {li} and {lo}")
        if di != do_:
            raise ValueError("input and output must both be host or both be device buffers")
        batch = int(np.prod(li, dtype=np.int64))
        if batch == 0:
            return   # nothing to do; an empty torch tensor has no data pointer for the C entry point
        self._call("dct4", "dct4", di, si, pi, po, batch, code)

    def mdct_frames(self, in_len, center=True):
        """F, the number of frames `mdct` makes of rows of in_len samples: ceil(in_len / N) + 1 with center, else
        1 + (in_len - 2N) // N (in_len >= 2N)."""
        n, in_len = self._size, int(in_len)
        return -(-in_len // n) + 1 if center else 1 + (in_len - 2 * n) // n

    def _mdct_window(self, window):
        pw, lw, dw, _ = self._describe(window, "real", last=2 * self._size)
        if lw != ():
            raise ValueError(f"window must hold exactly 2N = {2 * self._size} reals, got shape {tuple(window.shape)}")
        return pw, dw

    def mdct(self, input, window, output, center=True, norm="backward"):
        """The modified discrete cosine transform of every row of `input` (shape (..., L)): N = size() coefficients per
        frame of 2N samples every N, X_f[k] = 2 h sum_s w[s] x[fN - pad + s] cos(pi/N (s + 1/2 + N/2)(k + 1/2)), h as
        for dct4, `window` 2N reals.  center=True pads N zeros at both ends, so every sample lies in two frames
        (F = ceil(L/N) + 1); center=False needs L >= 2N (F = 1 + (L - 2N) // N) and is tf.signal.mdct(x, 2N,
        window_fn, pad_end=False).  `output` has shape (..., F, N), F = mdct_frames(L, center).  Out of place only."""
        self._check_resolved(input, window, output)
        code = self._check_norm(norm)
        n = self._size
        in_len = input.shape[-1] if getattr(input, "ndim", 0) > 0 else 0
        if in_len < 1:
            raise ValueError("input rows must hold at least one sample")
        if not center and in_len < 2 * n:
            raise ValueError(f"center=False needs rows of at least 2N = {2 * n} samples, got {in_len}")
        frames = self.mdct_frames(in_len, center)
        pi, li, di, si = self._describe(input, "real", last=in_len)
        pw, dw = self._mdct_window(window)
        if getattr(output, "ndim", 0) < 2 or output.shape[-2] != frames:
            raise ValueError(f"output must have shape (..., {frames}, {n}) for rows of {in_len} samples")
        po, lo, do_, _ = self._describe(output, "real")
        if lo[:-1] != li:
            raise ValueError(f"input and output leading shapes differ: {li} and {lo[:-1]}")
        if not (di == dw == do_):
            raise ValueError("input, window and output must all be host or all be device buffers")
        batch = int(np.prod(li, dtype=np.int64))
        if batch == 0:
            return
        self._call("mdct", "mdct", di, si, pi, in_len, pw, int(bool(center)), code, po, batch)

    def imdct(self, input, window, output, center=True, norm="backward"):
        """Inverse of mdct: `input` (shape (..., F, N)) -> `output` (shape (..., out_len), any out_len >= 1).  Output i
        is the overlap-add of window * v_f over the frames covering padded position t = i + pad (pad = N if center),
        v_f the unfolded dct4 of frame f with the norm's backward and forward swapped, with no division: the aliasing
        cancels between frames.  With center, out_len = L and a Princen-Bradley window (w[s]^2 + w[s+N]^2 = 1, w
        symmetric), imdct(mdct(x)) = x in every norm.  Without center and out_len = (F + 1) N this is
        tf.signal.inverse_mdct.  Out of place only."""
        self._check_resolved(input, window, output)
        code = self._check_norm(norm)
        n = self._size
        if getattr(input, "ndim", 0) < 2 or input.shape[-2] < 1:
            raise ValueError(f"input must have shape (..., F, {n}) with F >= 1")
        frames = int(input.shape[-2])
        out_len = output.shape[-1] if getattr(output, "ndim", 0) > 0 else 0
        if out_len < 1:
            raise ValueError("output rows must hold at least one sample")
        pi, li, di, si = self._describe(input, "real")
        pw, dw = self._mdct_window(window)
        po, lo, do_, _ = self._describe(output, "real", last=out_len)
        if li[:-1] != lo:
            raise ValueError(f"input and output leading shapes differ: {li[:-1]} and {lo}")
        if not (di == dw == do_):
            raise ValueError("input, window and output must all be host or all be device buffers")
        batch = int(np.prod(lo, dtype=np.int64))
        if batch == 0:
            return
        self._call("imdct", "imdct", di, si, pi, frames, pw, int(bool(center)), code, po, out_len, batch)

    WELCH_SCALINGS = {"density": 0, "spectrum": 1}
    WELCH_DETRENDS = {False: 0, "constant": 1}

    def welch(self, input, window, hop, output, fs=1.0, scaling="density", detrend="constant"):
        """Welch's power spectral density of every row of `input` (shape (..., L), L >= N): the F = stft_frames(L, hop,
        center=False) frames of N = size() samples every `hop`, each with its mean taken off (detrend "constant"; False
        keeps it) and then times `window` (N reals), averaged as |rfft|**2, one-sided and scaled to a density
        (1 / (fs * sum(window**2))) or a spectrum (1 / sum(window)**2).  `output` has shape (..., N//2+1) in the real
        dtype: this is scipy.signal.welch(x, fs, window=window, nperseg=N, noverlap=N-hop, detrend=detrend,
        scaling=scaling)[1], at the frequencies numpy.fft.rfftfreq(N, 1/fs).  The frames stay on chip where the plan's
        path allows.  Out of place only."""
        self._check_resolved(input, window, output)
        if not isinstance(scaling, str) or scaling not in self.WELCH_SCALINGS:
            raise ValueError(f"scaling must be 'density' or 'spectrum', got {scaling!r}")
        if not (detrend is False or (isinstance(detrend, str) and detrend == "constant")):
            raise ValueError(f"detrend must be 'constant' or False, got {detrend!r}")
        fs = float(fs)
        if not (np.isfinite(fs) and fs > 0):
            raise ValueError(f"fs must be finite and positive, got {fs!r}")
        hop, _, in_len, _, (pi, li, di, si), (pw, dw) = self._framing(input, window, hop, False, "reflect")
        po, lo, do_, _ = self._describe(output, "real", last=self._size // 2 + 1)
        if li != lo:
            raise ValueError(f"input and output leading shapes differ: {li} and {lo}")
        if not (di == dw == do_):
            raise ValueError("input, window and output must all be host or all be device buffers")
        batch = int(np.prod(li, dtype=np.int64))
        if batch == 0:
            return   # nothing to do; an empty torch tensor has no data pointer for the C entry point
        self._call("welch", "welch", di, si, pi, in_len, pw, hop, self.WELCH_DETRENDS[detrend],
                   self.WELCH_SCALINGS[scaling], fs, po, batch)

    def csd(self, x, y, window, hop, output, fs=1.0, scaling="density", detrend="constant"):
        """Cross-spectral density of every row of `x` (shape (..., L), L >= N) with its row of `y`: welch's frames of
        both, detrended and windowed alike, averaged as conj(rfft(x frame)) * rfft(y frame), one-sided and scaled as
        welch does.  `y` has rows of the same L, and its leading shape must equal a trailing part of x's and is
        broadcast over the rest, as convolve's spectrum is.  `output` has shape (..., N//2+1) in the complex dtype and
        x's leading shape: this is scipy.signal.csd(x, y, fs, window=window, nperseg=N, noverlap=N-hop,
        detrend=detrend, scaling=scaling)[1].  The frames stay on chip where the plan's path allows.  Out of place
        only."""
        if not isinstance(scaling, str) or scaling not in self.WELCH_SCALINGS:
            raise ValueError(f"scaling must be 'density' or 'spectrum', got {scaling!r}")
        fs = float(fs)
        if not (np.isfinite(fs) and fs > 0):
            raise ValueError(f"fs must be finite and positive, got {fs!r}")
        self._cross("csd", x, y, window, hop, output, detrend, self.WELCH_SCALINGS[scaling], fs)

    def coherence(self, x, y, window, hop, output, detrend="constant"):
        """Magnitude-squared coherence of every row of `x` with its row of `y` (framed and broadcast as in csd):
        |sum conj(X) Y|**2 / (sum |X|**2 * sum |Y|**2) over the frames, per bin.  `output` has shape (..., N//2+1) in
        the real dtype: this is scipy.signal.coherence(x, y, fs, window=window, nperseg=N, noverlap=N-hop,
        detrend=detrend)[1] for any fs.  NaN where a denominator is 0, as scipy gives.  Out of place only."""
        self._cross("coherence", x, y, window, hop, output, detrend, None, None)

    def _cross(self, kind, x, y, window, hop, output, detrend, scaling, fs):
        self._check_resolved(x, y, window, output)
        if not (detrend is False or (isinstance(detrend, str) and detrend == "constant")):
            raise ValueError(f"detrend must be 'constant' or False, got {detrend!r}")
        hop, _, in_len, _, (pi, li, di, si), (pw, dw) = self._framing(x, window, hop, False, "reflect")
        if getattr(y, "ndim", 0) == 0 or y.shape[-1] != in_len:
            raise ValueError(f"y rows must hold the {in_len} samples of the x rows")
        py, ly, dy, _ = self._describe(y, "real", last=in_len)
        po, lo, do_, _ = self._describe(output, "spec" if kind == "csd" else "real", last=self._size // 2 + 1)
        if li != lo:
            raise ValueError(f"x and output leading shapes differ: {li} and {lo}")
        if len(ly) > len(li) or tuple(li[len(li) - len(ly):]) != ly:
            raise ValueError(f"y leading shape {ly} is not a trailing part of x's {li}")
        if not (di == dy == dw == do_):
            raise ValueError("x, y, window and output must all be host or all be device buffers")
        batch = int(np.prod(li, dtype=np.int64))
        if batch == 0:
            return   # nothing to do; an empty torch tensor has no data pointer for the C entry point
        y_rows = int(np.prod(ly, dtype=np.int64))
        if kind == "csd":
            self._call("csd", "csd", di, si, pi, py, y_rows, in_len, pw, hop, self.WELCH_DETRENDS[detrend], scaling,
                       fs, po, batch)
        else:
            self._call("coherence", "coherence", di, si, pi, py, y_rows, in_len, pw, hop, self.WELCH_DETRENDS[detrend],
                       po, batch)

    def istft(self, input, window, hop, output, center=True):
        """Inverse of stft: `input` (shape (..., F, N//2+1), stft's frame-major layout) -> `output` (shape
        (..., out_len), any out_len >= 1).  Output i is the overlap-add of window * irfft(frame) over the frames that
        cover padded position t = i + pad (pad = N//2 if center), divided by the sum of window^2 there; 0 where that
        sum is below 1e-11, including positions no frame covers (torch.istft raises instead).  With out_len =
        hop * (F - 1) + N - 2 pad this is torch.istft(input.transpose(-1, -2), N, hop, window=window, center=center,
        length=out_len).  Out of place only."""
        self._check_resolved(input, window, output)
        hop = int(hop)
        if hop < 1:
            raise ValueError(f"hop must be at least 1, got {hop}")
        n = self._size
        if getattr(input, "ndim", 0) < 2 or input.shape[-2] < 1:
            raise ValueError(f"input must have shape (..., F, {n // 2 + 1}) with F >= 1")
        frames = int(input.shape[-2])
        out_len = output.shape[-1] if getattr(output, "ndim", 0) > 0 else 0
        if out_len < 1:
            raise ValueError("output rows must hold at least one sample")
        pi, li, di, si = self._describe(input, "spec")
        pw, lw, dw, _ = self._describe(window, "real")
        if lw != ():
            raise ValueError(f"window must hold exactly N = {n} reals, got shape {tuple(window.shape)}")
        po, lo, do_, _ = self._describe(output, "real", last=out_len)
        if li[:-1] != lo:
            raise ValueError(f"input and output leading shapes differ: {li[:-1]} and {lo}")
        if not (di == dw == do_):
            raise ValueError("input, window and output must all be host or all be device buffers")
        batch = int(np.prod(lo, dtype=np.int64))
        self._call("istft", "istft", di, si, pi, frames, pw, hop, int(bool(center)), po, out_len, batch)

    def rfft(self, input, output, transform=Transform.Fft):
        """output[..., :N//2+1] = numpy.fft.rfft(input) (Fft) or that times 1/sqrt(N) (SqrtScaledFft)."""
        self._run("forward", input, output, transform)

    def irfft(self, input, output, transform=Transform.Ifft):
        """output = numpy.fft.irfft(input, n=N) (Ifft), N times that (UnscaledIfft) or sqrt(N) times (SqrtScaledIfft)."""
        self._run("inverse", input, output, transform)


def create_rfft_f32(size):
    """Real-input transforms of length `size` in single precision."""
    return RealFft(size, "f32")


def create_rfft_f64(size):
    """Real-input transforms of length `size` in double precision."""
    return RealFft(size, "f64")


def set_device(device):
    rc = _lib.load().fourier_b200_set_device(int(device))
    if rc != 0:
        raise RuntimeError(f"fourier_b200_set_device({device}) failed: {_lib.last_error()}")


def fill_input(tensor, first_transform=0, seed=0xDEADBEEF):
    """Fill a torch CUDA complex tensor of shape (..., size) with the synthetic benchmark input
    (same counter-hash stream as the oracle's fill_input), on torch's current stream."""
    import torch
    if not tensor.is_cuda or not tensor.is_contiguous():
        raise ValueError("fill_input needs a contiguous CUDA tensor")
    t = {torch.complex64: "float", torch.complex128: "double"}[tensor.dtype]
    n = tensor.shape[-1]
    count = 2 * tensor.numel()
    stream = torch.cuda.current_stream(tensor.device).cuda_stream
    rc = getattr(_lib.load(), f"fourier_b200_fill_input_{t}")(
        tensor.data_ptr(), 2 * n * int(first_transform), count, seed, stream)
    if rc != 0:
        raise RuntimeError(f"fill_input failed: {_lib.last_error()}")
    return tensor


def lib_path():
    return _lib.LIB_PATH

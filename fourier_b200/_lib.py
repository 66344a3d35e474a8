"""Loads libfourier.so (the C-ABI product library) through ctypes.  No fallback: if the library is
missing or no CUDA device is usable, the error is raised to the caller."""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libfourier.so.0.1.0")


class PlanInfo(ctypes.Structure):
    _fields_ = [
        ("size", ctypes.c_size_t), ("path", ctypes.c_int), ("inner_size", ctypes.c_size_t),
        ("inner_path", ctypes.c_int), ("n1", ctypes.c_size_t), ("n2", ctypes.c_size_t),
        ("precision_bytes", ctypes.c_int), ("device", ctypes.c_int), ("table_bytes", ctypes.c_size_t),
        ("last_launches", ctypes.c_ulonglong),
    ]


_lib = None

# every symbol include/fourier.h and include/fourier_b200.h declare
REFERENCE_SYMBOLS = [f"fourier_{op}_{t}" for t in ("float", "double")
                     for op in ("create", "destroy", "transform_in_place", "transform")]
EXTENSION_SYMBOLS = (
    ["fourier_b200_set_device", "fourier_b200_get_device", "fourier_b200_device_count",
     "fourier_b200_peer_alloc", "fourier_b200_peer_open", "fourier_b200_peer_close", "fourier_b200_peer_free",
     "fourier_b200_path_name", "fourier_b200_last_error", "fourier_b200_version"]
    + [f"fourier_b200_{op}_{t}" for t in ("float", "double")
       for op in ("transform_batch", "transform_batch_async", "plan_info", "create_general", "fill_input",
                  "transpose", "pack", "exchange", "fft_rows_exchange", "swap_leading", "twiddle_rows", "plan_kernel")]
    + [f"fourier_b200_rfft_{op}_{t}" for t in ("float", "double")
       for op in ("create", "destroy", "forward", "forward_async", "inverse", "inverse_async", "info", "kernel")]
    + [f"fourier_b200_convolve_real_{op}{t}" for t in ("float", "double") for op in ("", "async_")]
    + [f"fourier_b200_linear_convolve_real_{op}{t}" for t in ("float", "double") for op in ("", "async_")]
    + [f"fourier_b200_{fn}_{op}{t}" for fn in ("stft", "istft") for t in ("float", "double") for op in ("", "async_")]
    + [f"fourier_b200_mel_spectrogram_{op}{t}" for t in ("float", "double") for op in ("", "async_")]
    + [f"fourier_b200_mfcc_{op}{t}" for t in ("float", "double") for op in ("", "async_")]
    + [f"fourier_b200_welch_{op}{t}" for t in ("float", "double") for op in ("", "async_")]
    + [f"fourier_b200_{fn}_{op}{t}" for fn in ("csd", "coherence") for t in ("float", "double") for op in ("", "async_")]
    + [f"fourier_b200_dct_{op}{t}" for t in ("float", "double") for op in ("", "async_")]
    + [f"fourier_b200_hilbert_{op}{t}" for t in ("float", "double") for op in ("", "async_")]
    + [f"fourier_b200_{fn}_{op}{t}" for fn in ("dct4", "mdct", "imdct") for t in ("float", "double")
       for op in ("", "async_")])


def load():
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            f"{LIB_PATH} is missing: build it with `python -m fourier_b200.build` "
            "(nvcc, sm_90a). fourier_b200 has no CPU or PyTorch fallback.")
    L = ctypes.CDLL(LIB_PATH)
    vp, sz, ci, dbl = ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int, ctypes.c_double
    for t in ("float", "double"):
        getattr(L, f"fourier_create_{t}").restype = vp
        getattr(L, f"fourier_create_{t}").argtypes = [sz]
        getattr(L, f"fourier_destroy_{t}").restype = None
        getattr(L, f"fourier_destroy_{t}").argtypes = [vp]
        getattr(L, f"fourier_transform_in_place_{t}").restype = None
        getattr(L, f"fourier_transform_in_place_{t}").argtypes = [vp, vp, ci]
        getattr(L, f"fourier_transform_{t}").restype = None
        getattr(L, f"fourier_transform_{t}").argtypes = [vp, vp, vp, ci]
        getattr(L, f"fourier_b200_transform_batch_{t}").argtypes = [vp, vp, vp, sz, ci]
        getattr(L, f"fourier_b200_transform_batch_async_{t}").argtypes = [vp, vp, vp, sz, ci, vp]
        getattr(L, f"fourier_b200_plan_info_{t}").argtypes = [vp, ctypes.POINTER(PlanInfo)]
        getattr(L, f"fourier_b200_plan_kernel_{t}").restype = ctypes.c_char_p
        getattr(L, f"fourier_b200_plan_kernel_{t}").argtypes = [vp]
        getattr(L, f"fourier_b200_create_general_{t}").restype = vp
        getattr(L, f"fourier_b200_create_general_{t}").argtypes = [sz]
        getattr(L, f"fourier_b200_fill_input_{t}").argtypes = [vp, ctypes.c_ulonglong, sz, ctypes.c_ulonglong, vp]
        getattr(L, f"fourier_b200_transpose_{t}").argtypes = [vp, vp, sz, sz, sz, vp]
        getattr(L, f"fourier_b200_pack_{t}").argtypes = [vp, vp, sz, sz, sz, sz, sz, sz, ci, ctypes.c_ulonglong,
                                                       ctypes.c_ulonglong, ctypes.c_ulonglong, vp]
        getattr(L, f"fourier_b200_exchange_{t}").argtypes = [vp, ctypes.POINTER(vp), ci, ci, sz, sz, sz, sz, sz, ci,
                                                           ctypes.c_ulonglong, ctypes.c_ulonglong, vp]
        getattr(L, f"fourier_b200_fft_rows_exchange_{t}").argtypes = [vp, vp, sz, ci, ctypes.POINTER(vp), ci, sz, sz, ci,
                                                                    ctypes.c_ulonglong, ctypes.c_ulonglong, vp]
        getattr(L, f"fourier_b200_swap_leading_{t}").argtypes = [vp, vp, sz, sz, sz, vp]
        getattr(L, f"fourier_b200_twiddle_rows_{t}").argtypes = [vp, sz, sz, ctypes.c_ulonglong, ctypes.c_ulonglong, ci, vp]
        getattr(L, f"fourier_b200_rfft_create_{t}").restype = vp
        getattr(L, f"fourier_b200_rfft_create_{t}").argtypes = [sz]
        getattr(L, f"fourier_b200_rfft_destroy_{t}").restype = None
        getattr(L, f"fourier_b200_rfft_destroy_{t}").argtypes = [vp]
        for d in ("forward", "inverse"):
            getattr(L, f"fourier_b200_rfft_{d}_{t}").argtypes = [vp, vp, vp, sz, ci]
            getattr(L, f"fourier_b200_rfft_{d}_async_{t}").argtypes = [vp, vp, vp, sz, ci, vp]
        getattr(L, f"fourier_b200_rfft_info_{t}").argtypes = [vp, ctypes.POINTER(PlanInfo)]
        getattr(L, f"fourier_b200_rfft_kernel_{t}").restype = ctypes.c_char_p
        getattr(L, f"fourier_b200_rfft_kernel_{t}").argtypes = [vp]
        getattr(L, f"fourier_b200_convolve_real_{t}").argtypes = [vp, vp, vp, sz, vp, sz]
        getattr(L, f"fourier_b200_convolve_real_async_{t}").argtypes = [vp, vp, vp, sz, vp, sz, vp]
        getattr(L, f"fourier_b200_linear_convolve_real_{t}").argtypes = [vp, vp, sz, vp, sz, sz, ci, vp, sz]
        getattr(L, f"fourier_b200_linear_convolve_real_async_{t}").argtypes = [vp, vp, sz, vp, sz, sz, ci, vp, sz, vp]
        getattr(L, f"fourier_b200_stft_{t}").argtypes = [vp, vp, sz, vp, sz, ci, vp, sz]
        getattr(L, f"fourier_b200_stft_async_{t}").argtypes = [vp, vp, sz, vp, sz, ci, vp, sz, vp]
        getattr(L, f"fourier_b200_istft_{t}").argtypes = [vp, vp, sz, vp, sz, ci, vp, sz, sz]
        getattr(L, f"fourier_b200_istft_async_{t}").argtypes = [vp, vp, sz, vp, sz, ci, vp, sz, sz, vp]
        getattr(L, f"fourier_b200_mel_spectrogram_{t}").argtypes = [vp, vp, sz, vp, sz, ci, ci, vp, sz, vp, sz]
        getattr(L, f"fourier_b200_mel_spectrogram_async_{t}").argtypes = [vp, vp, sz, vp, sz, ci, ci, vp, sz, vp, sz, vp]
        mfcc = [vp, vp, sz, vp, sz, ci, ci, vp, sz, dbl, dbl, dbl, dbl, sz, vp, sz, dbl, vp, sz]
        getattr(L, f"fourier_b200_mfcc_{t}").argtypes = mfcc
        getattr(L, f"fourier_b200_mfcc_async_{t}").argtypes = mfcc + [vp]
        getattr(L, f"fourier_b200_welch_{t}").argtypes = [vp, vp, sz, vp, sz, ci, ci, ctypes.c_double, vp, sz]
        getattr(L, f"fourier_b200_welch_async_{t}").argtypes = [vp, vp, sz, vp, sz, ci, ci, ctypes.c_double, vp, sz, vp]
        getattr(L, f"fourier_b200_csd_{t}").argtypes = [vp, vp, vp, sz, sz, vp, sz, ci, ci, ctypes.c_double, vp, sz]
        getattr(L, f"fourier_b200_csd_async_{t}").argtypes = [vp, vp, vp, sz, sz, vp, sz, ci, ci, ctypes.c_double, vp,
                                                              sz, vp]
        getattr(L, f"fourier_b200_coherence_{t}").argtypes = [vp, vp, vp, sz, sz, vp, sz, ci, vp, sz]
        getattr(L, f"fourier_b200_coherence_async_{t}").argtypes = [vp, vp, vp, sz, sz, vp, sz, ci, vp, sz, vp]
        getattr(L, f"fourier_b200_dct_{t}").argtypes = [vp, vp, vp, sz, ci, ci]
        getattr(L, f"fourier_b200_dct_async_{t}").argtypes = [vp, vp, vp, sz, ci, ci, vp]
        getattr(L, f"fourier_b200_hilbert_{t}").argtypes = [vp, vp, vp, sz, ci]
        getattr(L, f"fourier_b200_hilbert_async_{t}").argtypes = [vp, vp, vp, sz, ci, vp]
        getattr(L, f"fourier_b200_dct4_{t}").argtypes = [vp, vp, vp, sz, ci]
        getattr(L, f"fourier_b200_dct4_async_{t}").argtypes = [vp, vp, vp, sz, ci, vp]
        getattr(L, f"fourier_b200_mdct_{t}").argtypes = [vp, vp, sz, vp, ci, ci, vp, sz]
        getattr(L, f"fourier_b200_mdct_async_{t}").argtypes = [vp, vp, sz, vp, ci, ci, vp, sz, vp]
        getattr(L, f"fourier_b200_imdct_{t}").argtypes = [vp, vp, sz, vp, ci, ci, vp, sz, sz]
        getattr(L, f"fourier_b200_imdct_async_{t}").argtypes = [vp, vp, sz, vp, ci, ci, vp, sz, sz, vp]
    L.fourier_b200_peer_alloc.argtypes = [sz, ctypes.POINTER(vp), ctypes.c_char_p]
    L.fourier_b200_peer_open.argtypes = [ctypes.c_char_p, ctypes.POINTER(vp)]
    L.fourier_b200_peer_close.argtypes = [vp]
    L.fourier_b200_peer_free.argtypes = [vp]
    L.fourier_b200_set_device.argtypes = [ci]
    L.fourier_b200_path_name.restype = ctypes.c_char_p
    L.fourier_b200_path_name.argtypes = [ci]
    L.fourier_b200_last_error.restype = ctypes.c_char_p
    L.fourier_b200_version.restype = ctypes.c_char_p
    _lib = L
    return L


def last_error():
    return load().fourier_b200_last_error().decode()

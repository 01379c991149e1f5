"""ctypes binding of the test-only probe of the regression head's training kernels, tests/libthmr_head_train_probe.so
(tests/csrc/head_train_probe.cu).  Every wrapper returns a THMR status, except head_probe_hl_gemm, which returns the
split count it launched with; `call` and `hl_gemm` raise on a failure."""
from __future__ import annotations

import ctypes
from ctypes import POINTER, Structure, c_char_p, c_float, c_int, c_longlong, c_void_p
from pathlib import Path

PROBE_PATH = Path(__file__).resolve().parent / "libthmr_head_train_probe.so"
_probe = None


class HlGemm(Structure):
    """Mirror of the regression head's fp32 GEMM descriptor HlGemm (csrc/head_train.cuh)."""
    _fields_ = [("A", c_void_p), ("sAm", c_longlong), ("sAk", c_longlong), ("sAz", c_longlong),
                ("Bm", c_void_p), ("sBk", c_longlong), ("sBn", c_longlong), ("sBz", c_longlong),
                ("C", c_void_p), ("ldc", c_longlong), ("sCz", c_longlong),
                ("M", c_int), ("N", c_int), ("K", c_int), ("batch", c_int),
                ("alpha", c_float),
                ("bias", c_void_p), ("dgelu", c_void_p), ("gelu_out", c_void_p),
                ("accumulate", c_int),
                ("partial", c_void_p),
                ("splits", c_int)]


HL_ORIENT = {"xwt": 0, "dyw": 1, "dytx": 2}   # kXWt / kDyW / kDytX

P, I, F = c_void_p, c_int, c_float
SIGNATURES = {
    "head_probe_last_error": (c_char_p, []),
    "head_probe_check_device_flags": (c_int, []),
    "head_probe_hl_gemm_desc_size": (ctypes.c_size_t, []),
    "head_probe_hl_split_floats": (c_longlong, []),
    "head_probe_hl_gemm": (c_int, [POINTER(HlGemm), I, P]),
    "head_probe_rh_attn_fwd": (c_int, [P, P, I, F, I, P, P, P, P, P, P]),
    "head_probe_rh_attn_bwd": (c_int, [P, P, I, F, I, P, P, P, P, P, P, P]),
    "head_probe_rh_ln_fwd": (c_int, [P, P, P, P, P, P, I, P]),
    "head_probe_rh_ln_bwd": (c_int, [P, P, P, P, P, P, I, P]),
    "head_probe_rh_colsum": (c_int, [I, P, I, I, I, P, P, P, P, P, P, P]),
    "head_probe_rh_token0": (c_int, [P, P, P, I, P]),
    "head_probe_rh_readout_bwd": (c_int, [P, P, P, P, P, P, I, P]),
}


def lib() -> ctypes.CDLL:
    global _probe
    if _probe is None:
        if not PROBE_PATH.exists():
            raise RuntimeError(f"{PROBE_PATH} not found: it is built by tokenhmr_b200._build.build()")
        _probe = ctypes.CDLL(str(PROBE_PATH))
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(_probe, name)
            fn.restype, fn.argtypes = res, args
    return _probe


def _error() -> str:
    return lib().head_probe_last_error().decode(errors="replace")


def call(name: str, *args) -> None:
    status = getattr(lib(), name)(*args)
    if status != 0:
        raise RuntimeError(f"{name} failed ({status}): {_error()}")


def flags() -> int:
    """Reads and clears this library's device status words (bit 0 pipeline timeout, bit 1 split overflow)."""
    f = lib().head_probe_check_device_flags()
    if f < 0:
        raise RuntimeError("head_probe_check_device_flags: CUDA error")
    return f


def hl_gemm(desc: HlGemm, orient: str) -> int:
    """The regression head's fp32 GEMM (head_train.cuh hl_gemm) as the engine launches it, in orientation "xwt",
    "dyw" or "dytx"; returns the split count its planner chose."""
    if lib().head_probe_hl_gemm_desc_size() != ctypes.sizeof(HlGemm):
        raise RuntimeError("tests/head_train_probe.py HlGemm does not mirror head_train.cuh's")
    import torch
    n = lib().head_probe_hl_gemm(ctypes.byref(desc), HL_ORIENT[orient], torch.cuda.current_stream().cuda_stream)
    if n < 1:
        raise RuntimeError(f"head_probe_hl_gemm failed ({n}): {_error()}")
    return n

"""ctypes binding of the FP8 mode's test-only probe tests/libthmr_fp8_probe.so (tests/csrc/fp8_probe.cu), plus thin
torch-facing helpers.  Every wrapper returns a THMR status; `call` raises on a non-zero one."""
from __future__ import annotations

import ctypes
from ctypes import POINTER, Structure, c_char_p, c_float, c_int, c_longlong, c_void_p
from pathlib import Path

PROBE_PATH = Path(__file__).resolve().parent / "libthmr_fp8_probe.so"
_probe = None


class Fp8GemmDesc(Structure):
    """Mirror of fp8_probe_gemm_desc (fp8_probe.cu)."""
    _fields_ = [("A", c_void_p), ("lda", c_int), ("a_rows", c_longlong),
                ("B", c_void_p), ("ldb", c_int),
                ("M", c_int), ("N", c_int), ("K", c_int),
                ("bias", c_void_p),
                ("resid", c_void_p), ("ldr", c_int),
                ("act", c_int),
                ("out32", c_void_p), ("ld32", c_int),
                ("out16", c_void_p), ("ld16", c_int),
                ("alpha", c_float),
                ("force_bn", c_int),
                ("a_scale", c_void_p), ("ld_as", c_int),
                ("w_scale", c_void_p),
                ("out8", c_void_p), ("ld8", c_int), ("out8_scale", c_void_p), ("ld8s", c_int)]


P, I, F = c_void_p, c_int, c_float
SIGNATURES = {
    "fp8_probe_last_error": (c_char_p, []),
    "fp8_probe_gemm_desc_size": (ctypes.c_size_t, []),
    "fp8_probe_check_device_flags": (c_int, []),
    "fp8_probe_gemm": (c_int, [POINTER(Fp8GemmDesc), P]),
    "fp8_probe_layernorm_e4m3": (c_int, [P, P, P, P, P, I, P, I, I, F, P]),
}

ACT = {"none": 0, "gelu": 1, "relu": 2}      # kActNone / kActGelu / kActRelu


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


def call(name: str, *args) -> None:
    status = getattr(lib(), name)(*args)
    if status != 0:
        raise RuntimeError(f"{name} failed ({status}): {lib().fp8_probe_last_error().decode(errors='replace')}")


def ptr(t) -> int | None:
    return None if t is None else t.data_ptr()


def stream() -> int:
    import torch
    return torch.cuda.current_stream().cuda_stream


def flags() -> int:
    """Reads and clears the FP8 probe's pipeline-timeout flag (1 = set)."""
    f = lib().fp8_probe_check_device_flags()
    if f < 0:
        raise RuntimeError("fp8_probe_check_device_flags: CUDA error")
    return f


def gemm_fp8(A8, a_scale, B8, w_scale, M: int, N: int, K: int, *, a_rows: int | None = None, bias=None, resid=None,
             ldr: int = 0, act: str = "none", out32=None, ld32: int = 0, out16=None, ld16: int = 0, out8=None,
             out8_scale=None, alpha: float = 1.0, force_bn: int = 0) -> None:
    """FP8 GEMM: A8 [M, K] / B8 [N, K] e4m3 codes (float8_e4m3fn or uint8), a_scale [K/128, >= M padded to 128],
    w_scale [ceil(N/128), K/128]; out8 (e4m3 [M, N]) with out8_scale [N/128, >= M]."""
    d = Fp8GemmDesc(ptr(A8), A8.stride(0), a_rows if a_rows is not None else M, ptr(B8), B8.stride(0), M, N, K,
                    ptr(bias), ptr(resid), ldr, ACT[act], ptr(out32), ld32, ptr(out16), ld16, alpha, force_bn,
                    ptr(a_scale), a_scale.stride(0), ptr(w_scale),
                    ptr(out8), out8.stride(0) if out8 is not None else 0,
                    ptr(out8_scale), out8_scale.stride(0) if out8_scale is not None else 0)
    call("fp8_probe_gemm", ctypes.byref(d), stream())


def layernorm_e4m3(x, gamma, beta, eps: float, y32=None, lds: int | None = None):
    """LayerNorm -> e4m3 codes [R, C] (uint8) + scales [C/128, lds] (elementwise.cuh layernorm_e4m3_kernel)."""
    import torch
    R, C = x.shape
    y8 = torch.zeros(R, C, dtype=torch.uint8, device=x.device)
    ys = torch.full((C // 128, lds or R), float("nan"), device=x.device)
    call("fp8_probe_layernorm_e4m3", x.data_ptr(), gamma.data_ptr(), beta.data_ptr(), y8.data_ptr(), ys.data_ptr(),
         ys.stride(0), ptr(y32), R, C, eps, stream())
    return y8, ys

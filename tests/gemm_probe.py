"""ctypes binding of the test-only GEMM plan probe tests/libthmr_gemm_probe.so (tests/csrc/gemm_probe.cu): the fp16 GEMM
with a forced epilogue kind, the plan's block_n / epilogue kind / grid, and the per-tile timeline."""
from __future__ import annotations

import ctypes
from ctypes import POINTER, Structure, c_char_p, c_float, c_int, c_longlong, c_void_p
from pathlib import Path

PROBE_PATH = Path(__file__).resolve().parent / "libthmr_gemm_probe.so"
_probe = None

ACT = {"none": 0, "gelu": 1, "relu": 2}      # kActNone / kActGelu / kActRelu
EPI = {"general": 0, "f16": 1, "bias_f16": 2, "bias_gelu_f16": 3, "bias_resid_f32": 4}   # kEpi* (gemm_wgmma.cuh)


class GemmDesc(Structure):
    """Mirror of gemm_probe_desc (gemm_probe.cu)."""
    _fields_ = [("A", c_void_p), ("lda", c_int), ("a_rows", c_longlong),
                ("B", c_void_p), ("ldb", c_int),
                ("M", c_int), ("N", c_int), ("K", c_int),
                ("bias", c_void_p),
                ("resid", c_void_p), ("ldr", c_int), ("resid_mod", c_int),
                ("act", c_int), ("act32", c_int),
                ("out32", c_void_p), ("ld32", c_int),
                ("out16", c_void_p), ("ld16", c_int),
                ("seq_pitch", c_int), ("seq_lo", c_int), ("seq_hi", c_int),
                ("alpha", c_float),
                ("force_bn", c_int),
                ("force_epi", c_int)]


P, I = c_void_p, c_int
SIGNATURES = {
    "gemm_probe_last_error": (c_char_p, []),
    "gemm_probe_desc_size": (ctypes.c_size_t, []),
    "gemm_probe_check_device_flags": (c_int, []),
    "gemm_probe_run": (c_int, [POINTER(GemmDesc), P]),
    "gemm_probe_plan": (c_int, [POINTER(GemmDesc), POINTER(c_int), POINTER(c_int), POINTER(c_int)]),
    "gemm_probe_timeline": (c_int, [POINTER(GemmDesc), P, I, P, P]),
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


def call(name: str, *args) -> None:
    status = getattr(lib(), name)(*args)
    if status != 0:
        raise RuntimeError(f"{name} failed ({status}): {lib().gemm_probe_last_error().decode(errors='replace')}")


def flags() -> int:
    """Reads and clears this library's pipeline-timeout flag (1 = a wait timed out)."""
    f = lib().gemm_probe_check_device_flags()
    if f < 0:
        raise RuntimeError("gemm_probe_check_device_flags: CUDA error")
    return f


def _ptr(t) -> int | None:
    return None if t is None else t.data_ptr()


def _stream() -> int:
    import torch
    return torch.cuda.current_stream().cuda_stream


def desc(A, B, M: int, N: int, K: int, *, bias=None, resid=None, ldr: int = 0, resid_mod: int = 0, act: str = "none",
         act32: int = 0, out32=None, ld32: int = 0, out16=None, ld16: int = 0, seq=(0, 0, 0), alpha: float = 1.0,
         force_bn: int = 0, epi: str | None = None) -> GemmDesc:
    """fp16 GEMM descriptor; epi names a forced epilogue kind (EPI), None leaves the choice to the plan."""
    return GemmDesc(_ptr(A), A.stride(0), M, _ptr(B), B.stride(0), M, N, K, _ptr(bias), _ptr(resid), ldr, resid_mod,
                    ACT[act], act32, _ptr(out32), ld32, _ptr(out16), ld16, seq[0], seq[1], seq[2], alpha, force_bn,
                    0 if epi is None else 1 + EPI[epi])


def gemm(A, B, M: int, N: int, K: int, **kw) -> None:
    call("gemm_probe_run", ctypes.byref(desc(A, B, M, N, K, **kw)), _stream())


def plan(A, B, M: int, N: int, K: int, **kw) -> tuple[int, str, int]:
    """(block_n, epilogue kind, grid) of the plan gemm_make_plan makes, without a launch."""
    bn, epi, grid = c_int(), c_int(), c_int()
    call("gemm_probe_plan", ctypes.byref(desc(A, B, M, N, K, **kw)), ctypes.byref(bn), ctypes.byref(epi),
         ctypes.byref(grid))
    return bn.value, {v: k for k, v in EPI.items()}[epi.value], grid.value


def timeline(A, B, M: int, N: int, K: int, slots: int, **kw):
    """gemm with the per-tile timeline: (stamps int64 [grid, slots, 2, 4] in ns, 0 where no tile ran; smid int32
    [grid]).  Stamps: tile start, first full barrier passed, last wgmma retired, epilogue done."""
    import torch
    _, _, grid = plan(A, B, M, N, K, **kw)
    tl = torch.zeros(grid, slots, 2, 4, dtype=torch.int64, device=A.device)
    sm = torch.full((grid,), -1, dtype=torch.int32, device=A.device)
    call("gemm_probe_timeline", ctypes.byref(desc(A, B, M, N, K, **kw)), tl.data_ptr(), slots, sm.data_ptr(),
         _stream())
    return tl, sm

"""ctypes binding of the test-only probe of the two heads' training kernels, tests/libthmr_head_train_probe.so
(tests/csrc/head_train_probe.cu).  Every wrapper returns a THMR status, except head_probe_hl_gemm, which returns the
split count it launched with, and head_probe_tk_colsum_chunks, which returns a count; `call` and `hl_gemm` raise on a
failure.

Also the helpers the two kernel test files share (tests/test_gpu_head_train_kernels.py,
tests/test_gpu_token_head_train_kernels.py): gamma, the NaN-filled outputs, the run-twice check, the teeth check, and
the hl_gemm call-site machinery (Site and its checks against fp64)."""
from __future__ import annotations

import ctypes
import dataclasses
import zlib
from ctypes import POINTER, Structure, c_char_p, c_float, c_int, c_longlong, c_short, c_void_p
from pathlib import Path

import probe
from probe import U32, assert_within

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

P, I, F, L = c_void_p, c_int, c_float, c_longlong
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
    "head_probe_tk_seq_map": (c_int, [I, I, POINTER(c_short), POINTER(c_short)]),
    "head_probe_tk_im2col": (c_int, [P, I, I, I, I, I, I, P, I, P]),
    "head_probe_tk_col2im": (c_int, [P, I, I, I, I, I, P, P, P, P, I, P]),
    "head_probe_tk_relu_copy": (c_int, [P, P, L, P]),
    "head_probe_tk_transpose": (c_int, [P, I, I, P, P, I, P]),
    "head_probe_tk_ln_wide_fwd": (c_int, [P, P, P, P, P, P, I, P]),
    "head_probe_tk_ln_wide_bwd": (c_int, [P, P, P, P, P, P, P, I, P]),
    "head_probe_tk_ln64_fwd": (c_int, [P, P, P, P, P, P, I, I, P]),
    "head_probe_tk_ln64_bwd": (c_int, [P, P, P, P, P, P, P, I, I, P]),
    "head_probe_tk_softmax_fwd": (c_int, [P, I, P]),
    "head_probe_tk_softmax_bwd": (c_int, [P, P, I, P]),
    "head_probe_tk_colsum": (c_int, [P, I, I, I, P, P, P, P, P, P, P, P]),
    "head_probe_tk_colsum_chunks": (c_int, [I]),
    "head_probe_tk_conv": (c_int, [P, I, I, I, I, I, I, P, P, I, P, I, I, P, P, P]),
    "head_probe_tk_conv_bwd": (c_int, [P, I, P, I, I, I, I, I, P, P, P, P, I, P, P, P]),
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


def tk_seq_map(lin: int, lout: int) -> tuple[list[int], list[int]]:
    """The token head's resize map as the kernels receive it (token_head_train.cuh tk_seq_map): (src[0 .. lout),
    lo[0 .. lin])."""
    src, lo = (c_short * 160)(), (c_short * 161)()
    call("head_probe_tk_seq_map", lin, lout, src, lo)
    return list(src[:lout]), list(lo[:lin + 1])


# ------------------------------------------------------------------------------------------------ shared test helpers
def gamma(n: int) -> float:
    """gamma_n = n u / (1 - n u): the relative error bound of n chained fp32 roundings."""
    return n * U32 / (1 - n * U32)


def _nan(*shape):
    import torch
    return torch.full(shape, float("nan"), device="cuda")


def _rejects(got, ref, bound) -> bool:
    """True when some element of got lies outside bound of the (perturbed) reference."""
    import torch
    err = (got.double() - ref.double()).abs()
    return bool((~(err <= torch.as_tensor(bound, device=err.device).double())).any())


def _twice(run):
    """Runs a launch twice; the two results must be bit-identical (no atomics, fixed reduction order)."""
    import torch
    a = run()
    b = run()
    for x, y in zip(a, b):
        assert torch.equal(x.nan_to_num(1234.5), y.nan_to_num(1234.5)) and torch.equal(x.isnan(), y.isnan())
    return a


# hl_gemm: C[z] = epilogue(alpha * sum_k A(m,k) B(k,n)).  Each output is a serial fmaf chain over its split's k range
# (at most kper = ceil(K / splits) terms), then, when split, the reduce kernel's `splits` additions in split order, so
# every product passes through at most kper + splits roundings: |acc - S| <= gamma_(kper+splits) sum_k |a||b| (= Tab).
# Then alpha (a power of two here: exact), + bias (1 rounding), * gelu'(dgelu) (1 rounding), + C0 (1 rounding): with
# G the fp64 gelu' (1 without dgelu) and eps_G the error of the fp32 gelu' itself,
#   |C - C64| <= gamma_(kper+splits+4) |G| (|alpha| Tab + |bias|) + eps_G (|alpha| Tab + |bias|) + u |C0|.
# gelu'(x) = 0.5 (1 + erff(x / sqrt 2)) + x phi(x) with expf: erff's 2 ulp and the argument's rounding (erf' <= 1.13)
# give u (2 + 0.8 |x|) on the first half; expf's 2 ulp, the rounding of -x^2/2 (relative u x^2 / 2 on the result) and
# three products on |x phi(x)| <= 0.25; the final sum u |G| <= 1.13 u:  eps_G = u (8 + |x| + x^2 |x| phi(x)).
# gelu_out = gelu(C) in fp32: |gelu'| <= 1.13 carries C's error; erff's 2 ulp and the argument's rounding on
# 0.5 |x| (1 + erf), the two products and (1 + erf)'s rounding add at most 4 u (|x| + 1).
# An empty trailing split (kbeg >= K) writes a zero partial, so it adds nothing and the bound holds as is.
FLOOR = 1e-30


def _gelu_grad64(x):
    import torch
    return 0.5 * (1 + torch.erf(x / 2 ** 0.5)) + x * torch.exp(-0.5 * x * x) / (2 * torch.pi) ** 0.5


def _eps_gelu_grad(x):
    import torch
    phi = torch.exp(-0.5 * x * x) / (2 * torch.pi) ** 0.5
    return U32 * (8 + x.abs() + x * x * x.abs() * phi)


def _view(buf, off, strides, size):
    import torch
    return torch.as_strided(buf, size, strides, off)


@dataclasses.dataclass
class Site:
    """One hl_gemm call: orientation, shape, operand strides (batch, row, col) and offsets into flat buffers, epilogue,
    and the split count the planner must choose."""
    name: str
    orient: str
    M: int
    N: int
    K: int
    batch: int
    sA: tuple           # (sAz, sAm, sAk)
    sB: tuple           # (sBz, sBk, sBn)
    sC: tuple           # (sCz, ldc, 1)
    splits: int
    a_off: int = 0
    b_off: int = 0
    c_off: int = 0
    c_extent: int = 0   # size of the output buffer (0: just what the view covers)
    alpha: float = 1.0
    bias: bool = False
    accumulate: bool = False
    dgelu: bool = False
    gelu_out: bool = False
    partial: bool = True

    @property
    def kper(self) -> int:
        return (self.K + self.splits - 1) // self.splits

    @property
    def empty_splits(self) -> int:
        """Trailing splits whose k range starts at or past K."""
        return sum(1 for s in range(self.splits) if s * self.kper >= self.K)

    @property
    def tiles(self) -> int:
        return ((self.N + 63) // 64) * ((self.M + 63) // 64) * self.batch


def _extent(off, strides, size):
    return off + sum((n - 1) * s for n, s in zip(size, strides)) + 1


def _linear(name, B, N, K, splits, ldx=None, ldy=None, y_off=0, y_extent=0, **kw):
    """hl_linear: y (B x N, ld ldy) [+]= x (B x K, ld ldx) W^T + bias."""
    ldx, ldy = ldx or K, ldy or N
    return Site(name, "xwt", B, N, K, 1, (0, ldx, 1), (0, 1, K), (0, ldy, 1), splits, c_off=y_off,
                c_extent=y_extent, **kw)


def _linear_dx(name, B, N, K, splits, ldy=None, y_off=0, **kw):
    """hl_linear_dx: dx (B x K) [+]= dy (B x N, ld ldy) W, W: N x K."""
    ldy = ldy or N
    return Site(name, "dyw", B, K, N, 1, (0, ldy, 1), (0, K, 1), (0, K, 1), splits, a_off=y_off, **kw)


def _linear_dw(name, B, N, K, ldy=None, y_off=0, ldx=None, splits=1):
    """dW (N x K) = dy^T (B x N, ld ldy) x (B x K, ld ldx): hl_linear_dw without a split buffer (splits 1), or
    token_head_train.cuh's tk_linear_dw with one (splits > 1)."""
    ldy, ldx = ldy or N, ldx or K
    return Site(name, "dytx", N, K, B, 1, (0, 1, ldy), (0, ldx, 1), (0, K, 1), splits, a_off=y_off,
                partial=splits > 1)


def _operands(site, integer: bool, g):
    """Flat fp32 buffers of A, B, bias, dgelu and C0 (C0: the accumulate input, NaN outside the view)."""
    import torch
    Asz, Bsz, Csz = (site.batch, site.M, site.K), (site.batch, site.K, site.N), (site.batch, site.M, site.N)
    draw = ((lambda n: torch.randint(-4, 5, (n,), device="cuda", generator=g).float()) if integer else
            (lambda n: torch.randn(n, device="cuda", generator=g)))
    A = draw(_extent(site.a_off, site.sA, Asz))
    Bm = draw(_extent(site.b_off, site.sB, Bsz))
    c_ext = max(site.c_extent, _extent(site.c_off, site.sC, Csz))
    C0 = torch.full((c_ext,), float("nan"), device="cuda")
    if site.accumulate:
        _view(C0, site.c_off, site.sC, Csz).copy_(draw(site.batch * site.M * site.N).view(Csz))
    bias = (draw(site.N) * (2 if integer else 1)) if site.bias else None
    dg = None
    if site.dgelu and not integer:
        dg = torch.zeros(c_ext, device="cuda")
        _view(dg, site.c_off, site.sC, Csz).copy_(2 * torch.randn(Csz, device="cuda", generator=g))
    return A, Bm, bias, dg, C0


def _run_site(site, A, Bm, bias, dg, C0, split):
    import torch
    out, gout = C0.clone(), (torch.full_like(C0, float("nan")) if site.gelu_out else None)
    d = HlGemm(A=A.data_ptr() + 4 * site.a_off, sAz=site.sA[0], sAm=site.sA[1], sAk=site.sA[2],
               Bm=Bm.data_ptr() + 4 * site.b_off, sBz=site.sB[0], sBk=site.sB[1], sBn=site.sB[2],
               C=out.data_ptr() + 4 * site.c_off, sCz=site.sC[0], ldc=site.sC[1],
               M=site.M, N=site.N, K=site.K, batch=site.batch, alpha=site.alpha,
               bias=probe.ptr(bias), dgelu=None if dg is None else dg.data_ptr() + 4 * site.c_off,
               gelu_out=None if gout is None else gout.data_ptr() + 4 * site.c_off,
               accumulate=int(site.accumulate), partial=probe.ptr(split) if site.partial else None, splits=-7)
    n = hl_gemm(d, site.orient)
    torch.cuda.synchronize()
    assert n == site.splits, f"{site.name}: {n} splits, the table says {site.splits}"
    return (out, gout) if gout is not None else (out,)


def _reference(site, A, Bm, bias, dg, C0, kmask=None):
    """fp64 epilogue(alpha * A B) over the k set kmask (all k by default), and the bound's ingredients."""
    Asz, Bsz, Csz = (site.batch, site.M, site.K), (site.batch, site.K, site.N), (site.batch, site.M, site.N)
    a = _view(A.double(), site.a_off, site.sA, Asz)
    b = _view(Bm.double(), site.b_off, site.sB, Bsz)
    am = a if kmask is None else a * kmask.view(1, 1, -1)
    S = site.alpha * (am @ b)
    Tab = abs(site.alpha) * (a.abs() @ b.abs())
    v = S + (bias.double() if bias is not None else 0)
    mag = Tab + (bias.double().abs() if bias is not None else 0)
    G, epsG = 1.0, 0.0
    if dg is not None:
        x = _view(dg.double(), site.c_off, site.sC, Csz)
        G, epsG = _gelu_grad64(x), _eps_gelu_grad(x)
        v = v * G
    c0 = _view(C0.double(), site.c_off, site.sC, Csz) if site.accumulate else 0
    v = v + c0
    return v, mag, G, epsG, c0


def _covered(site, n):
    import torch
    m = torch.zeros(n, dtype=torch.bool, device="cuda")
    _view(m, site.c_off, site.sC, (site.batch, site.M, site.N)).fill_(True)
    return m


def check_site_integer_exact(site, split_buf):
    """Integer operands in [-4, 4], an integer bias and C0, alpha a power of two: every partial sum is an integer below
    2^24 (|sum| <= 16 K), so the result equals fp64 exactly; a dropped, doubled or misindexed term fails.  dgelu rows
    run without dgelu here."""
    import torch
    g = torch.Generator(device="cuda").manual_seed(zlib.crc32(site.name.encode()))
    A, Bm, bias, dg, C0 = _operands(site, True, g)
    outs = _twice(lambda: _run_site(site, A, Bm, bias, None, C0, split_buf))
    Csz = (site.batch, site.M, site.N)
    ref, *_ = _reference(site, A, Bm, bias, None, C0)
    got = _view(outs[0], site.c_off, site.sC, Csz)
    assert torch.equal(got.double(), ref), f"{site.name}: {int((got.double() != ref).sum())} elements differ"
    cov = _covered(site, outs[0].numel())
    assert outs[0][~cov].isnan().all(), "wrote outside the output view"
    if site.gelu_out:       # gelu of an exact value: only gelu's own error (the bound below with C's error 0)
        x = ref
        assert_within(f"hl_gemm gelu_out (integer) {site.name}", _view(outs[1], site.c_off, site.sC, Csz),
                      probe.gelu64(x), 4 * U32 * (x.abs() + 1) + FLOOR)
        assert outs[1][~cov].isnan().all()


def check_site_within_bound(site, split_buf):
    """Random operands against fp64 within the bound above; returns the worst err/bound of (C, gelu_out)."""
    import torch
    g = torch.Generator(device="cuda").manual_seed(7 + zlib.crc32(site.name.encode()))
    A, Bm, bias, dg, C0 = _operands(site, False, g)
    outs = _twice(lambda: _run_site(site, A, Bm, bias, dg, C0, split_buf))
    Csz = (site.batch, site.M, site.N)
    kper = site.kper
    n = kper + (site.splits if site.splits > 1 else 0)
    ref, mag, G, epsG, c0 = _reference(site, A, Bm, bias, dg, C0)
    absG = G.abs() if torch.is_tensor(G) else G
    c0a = c0.abs() if torch.is_tensor(c0) else 0
    bound = gamma(n + 4) * absG * mag + epsG * mag + U32 * c0a + FLOOR
    got = _view(outs[0], site.c_off, site.sC, Csz)
    worst = assert_within(f"hl_gemm {site.name}", got, ref, bound)
    worst_g = 0.0
    cov = _covered(site, outs[0].numel())
    assert outs[0][~cov].isnan().all(), "wrote outside the output view"
    if site.gelu_out:
        worst_g = assert_within(f"hl_gemm gelu_out {site.name}", _view(outs[1], site.c_off, site.sC, Csz),
                                probe.gelu64(ref), 1.13 * bound + 4 * U32 * (ref.abs() + 1))
        assert outs[1][~cov].isnan().all()
    # teeth: the same bound rejects the reference without one k-term, and without one split's partial
    mask = torch.ones(site.K, dtype=torch.float64, device="cuda")
    mask[site.K // 2] = 0
    assert _rejects(got, _reference(site, A, Bm, bias, dg, C0, mask)[0], bound), "bound accepts a dropped k-term"
    if site.splits > 1:
        mask = torch.ones(site.K, dtype=torch.float64, device="cuda")
        mask[kper:min(site.K, 2 * kper)] = 0
        assert _rejects(got, _reference(site, A, Bm, bias, dg, C0, mask)[0], bound), "bound accepts a dropped split"
    return worst, worst_g

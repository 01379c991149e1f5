"""ctypes binding of the test-only probe library tests/libthmr_probe.so (tests/csrc/kernel_probe.cu), plus thin
torch-facing helpers.  Every wrapper returns a THMR status; `call` raises on a non-zero one."""
from __future__ import annotations

import ctypes
from ctypes import POINTER, Structure, c_char_p, c_double, c_float, c_int, c_long, c_longlong, c_void_p
from pathlib import Path

PROBE_PATH = Path(__file__).resolve().parent / "libthmr_probe.so"
_probe = None


class GemmDesc(Structure):
    """Mirror of probe_gemm_desc (kernel_probe.cu), i.e. of the engine's GemmDesc for a plain fp16 or FP8 GEMM."""
    _fields_ = [("A", c_void_p), ("lda", c_int), ("a_rows", c_longlong),
                ("B", c_void_p), ("ldb", c_int),
                ("M", c_int), ("N", c_int), ("K", c_int),
                ("bias", c_void_p),
                ("resid", c_void_p), ("ldr", c_int), ("resid_mod", c_int),
                ("act", c_int), ("act32", c_int),
                ("out32", c_void_p), ("ld32", c_int),
                ("out16", c_void_p), ("ld16", c_int),
                ("taps", c_int), ("cin", c_int), ("tap_row0", c_int), ("tap_stride", c_int),
                ("seq_pitch", c_int), ("seq_lo", c_int), ("seq_hi", c_int),
                ("alpha", c_float),
                ("force_bn", c_int),
                ("fp8", c_int),
                ("a_scale", c_void_p), ("ld_as", c_int),
                ("w_scale", c_void_p),
                ("out8", c_void_p), ("ld8", c_int), ("out8_scale", c_void_p), ("ld8s", c_int)]


P, I, L, LL, F, D = c_void_p, c_int, c_long, c_longlong, c_float, c_double
SIGNATURES = {
    "probe_last_error": (c_char_p, []),
    "probe_gemm_desc_size": (ctypes.c_size_t, []),
    "probe_check_device_flags": (c_int, []),
    "probe_gemm": (c_int, [POINTER(GemmDesc), P]),
    "probe_split_rows": (c_int, [P, L, P, L, I, I, I, I, I, P]),
    "probe_layernorm": (c_int, [P, P, P, P, I, P, I, I, F, I, I, P]),
    "probe_layernorm_e4m3": (c_int, [P, P, P, P, P, I, P, I, I, F, P]),
    "probe_softmax_rows": (c_int, [P, P, P, I, I, I, I, I, P]),
    "probe_vit_attention": (c_int, [P, I, I, P, P]),
    "probe_attention_f32": (c_int, [P, I, I, I, P, I, F, P]),
    "probe_dec_cross_attn": (c_int, [P, P, I, I, I, F, P, I, I, P]),
    "probe_dec_cross_attn_f32": (c_int, [P, P, I, I, I, F, P, I, I, P]),
    "probe_im2col_patch": (c_int, [P, P, I, I, I, I, I, I, I, I, P]),
    "probe_im2col_patch_f32": (c_int, [P, P, I, I, I, I, I, I, I, I, P]),
    "probe_relu_inplace": (c_int, [P, L, P]),
    "probe_upsample_rows": (c_int, [P, P, I, I, I, I, I, P]),
    "probe_mixer_add": (c_int, [P, P, P, P, I, I, I, P]),
    "probe_cast_f16": (c_int, [P, P, L, P]),
    "probe_head_assemble": (c_int, [P, I, P, I, I, I, P, P, P, P, P, P, P, I, I, P]),
    "probe_smpl_jreg": (c_int, [P, P, P, P, P, I, I, P]),
    "probe_smpl_pack_posedirs": (c_int, [P, P, P, I, P, I, P]),
    "probe_smpl_pose": (c_int, [P, I, P, P, P, I, P, P, P, P, I, P]),
    "probe_smpl_blend": (c_int, [P, P, I, I, I, P, P]),
    "probe_smpl_skin": (c_int, [I, I, P, P, I, P, P, L, P, L, I, I, P]),
    "probe_smpl_joints": (c_int, [P, P, L, P, P, P, P, P, I, P, P, F, F, P, P, P, I, P]),
    "probe_smplify_loss": (c_int, [P, P, P, P, P, I, I, P, P, P, P, P]),
    "probe_smplify_adam": (c_int, [P, P, P, P, L, I, D, P]),
    "probe_pose_draw": (c_int, [I, LL, LL, LL, LL, I, I, P]),
}

ACT = {"none": 0, "gelu": 1, "relu": 2}      # kActNone / kActGelu / kActRelu == kSplitAct*
FLAG_TIMEOUT, FLAG_OVERFLOW = 1, 2            # bits of probe_check_device_flags


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
        raise RuntimeError(f"{name} failed ({status}): {lib().probe_last_error().decode(errors='replace')}")


def ptr(t) -> int | None:
    return None if t is None else t.data_ptr()


def stream() -> int:
    import torch
    return torch.cuda.current_stream().cuda_stream


def flags() -> int:
    """Reads and clears the probe's device status words (FLAG_TIMEOUT | FLAG_OVERFLOW)."""
    f = lib().probe_check_device_flags()
    if f < 0:
        raise RuntimeError("probe_check_device_flags: CUDA error")
    return f


def gemm(A, B, M: int, N: int, K: int, *, lda: int | None = None, ldb: int | None = None, a_rows: int | None = None,
         bias=None, resid=None, ldr: int = 0, resid_mod: int = 0, act: str = "none", act32: int = 0,
         out32=None, ld32: int = 0, out16=None, ld16: int = 0, taps: int = 1, cin: int = 0, tap_row0: int = 0,
         tap_stride: int = 0, seq=(0, 0, 0), alpha: float = 1.0, force_bn: int = 0) -> None:
    d = GemmDesc(ptr(A), lda or A.stride(0), a_rows if a_rows is not None else M, ptr(B), ldb or B.stride(0), M, N, K,
                 ptr(bias), ptr(resid), ldr, resid_mod, ACT[act], act32, ptr(out32), ld32, ptr(out16), ld16,
                 taps, cin, tap_row0, tap_stride, seq[0], seq[1], seq[2], alpha, force_bn)
    call("probe_gemm", ctypes.byref(d), stream())


def gemm_fp8(A8, a_scale, B8, w_scale, M: int, N: int, K: int, *, a_rows: int | None = None, bias=None, resid=None,
             ldr: int = 0, act: str = "none", out32=None, ld32: int = 0, out16=None, ld16: int = 0, out8=None,
             out8_scale=None, alpha: float = 1.0, force_bn: int = 0) -> None:
    """FP8 GEMM: A8 [M, K] / B8 [N, K] e4m3 codes (float8_e4m3fn or uint8), a_scale [K/128, >= M padded to 128],
    w_scale [ceil(N/128), K/128]; out8 (e4m3 [M, N]) with out8_scale [N/128, >= M]."""
    # fields left out are zero; taps stays 1, the only value gemm_make_plan_fp8 accepts
    d = GemmDesc(A=ptr(A8), lda=A8.stride(0), a_rows=a_rows if a_rows is not None else M, B=ptr(B8), ldb=B8.stride(0),
                 M=M, N=N, K=K, bias=ptr(bias), resid=ptr(resid), ldr=ldr, act=ACT[act],
                 out32=ptr(out32), ld32=ld32, out16=ptr(out16), ld16=ld16, taps=1, alpha=alpha, force_bn=force_bn,
                 fp8=1, a_scale=ptr(a_scale), ld_as=a_scale.stride(0), w_scale=ptr(w_scale),
                 out8=ptr(out8), ld8=out8.stride(0) if out8 is not None else 0,
                 out8_scale=ptr(out8_scale), ld8s=out8_scale.stride(0) if out8_scale is not None else 0)
    call("probe_gemm", ctypes.byref(d), stream())


def split_rows(src, R: int, C: int, act: str = "none", T: int = 0, pitch: int = 0, lo: int = 0, dst=None,
               dst_rows: int | None = None):
    """fp32 [R, C] -> fp16 [rows, 3C] = [hi | lo | hi] of act(x) * 2^4 (strict.cuh split_rows_kernel)."""
    import torch
    if dst is None:
        dst = torch.zeros(dst_rows if dst_rows is not None else R, 3 * C, dtype=torch.float16, device=src.device)
    call("probe_split_rows", src.data_ptr(), src.stride(0), dst.data_ptr(), R, C, ACT[act], T, pitch, lo, stream())
    return dst


def layernorm_e4m3(x, gamma, beta, eps: float, y32=None, lds: int | None = None):
    """LayerNorm -> e4m3 codes [R, C] (uint8) + scales [C/128, lds] (elementwise.cuh layernorm_e4m3_kernel)."""
    import torch
    R, C = x.shape
    y8 = torch.zeros(R, C, dtype=torch.uint8, device=x.device)
    ys = torch.full((C // 128, lds or R), float("nan"), device=x.device)
    call("probe_layernorm_e4m3", x.data_ptr(), gamma.data_ptr(), beta.data_ptr(), y8.data_ptr(), ys.data_ptr(),
         ys.stride(0), ptr(y32), R, C, eps, stream())
    return y8, ys


# ------------------------------------------------------------------------------------------------ fp64 references
# Bounds are per element and scale-free: |y - y64| <= bound, where y64 is torch fp64 on the same rounded inputs the
# kernel sees and the bound is built from the magnitudes of the terms of the operation (never from the largest output).
U32 = 2.0 ** -24      # fp32 unit roundoff
U16 = 2.0 ** -11      # fp16 unit roundoff


def assert_within(name: str, got, ref, bound, report: dict | None = None) -> float:
    """|got - ref| <= bound element-wise (NaN fails); returns the worst |got - ref| / bound."""
    import torch
    got = got.detach().double()
    ref, bound = ref.to(got.device).double(), torch.as_tensor(bound, device=got.device).double()
    err = (got - ref).abs()
    ratio = err / bound
    bad = ~(err <= bound)
    worst = float(ratio[torch.isfinite(ratio)].max()) if bool(torch.isfinite(ratio).any()) else float("inf")
    if bool(bad.any()):
        idx = [int(i) for i in torch.nonzero(bad)[0]]
        raise AssertionError(f"{name}: {int(bad.sum())} of {bad.numel()} elements out of bound, first at {idx}: "
                             f"got {float(got[tuple(idx)]):.9g} want {float(ref[tuple(idx)]):.9g} "
                             f"bound {float(bound.expand_as(err)[tuple(idx)]):.3g}; worst err/bound {worst:.3g}")
    print(f"[bound] {name}: worst err/bound {worst:.3g}")
    if report is not None:
        report[name] = worst
    return worst


def gelu64(x):
    import torch
    return 0.5 * x * (1.0 + torch.erf(x / 2.0 ** 0.5))


def act64(x, act: str):
    import torch
    return {"none": lambda v: v, "gelu": gelu64, "relu": torch.relu}[act](x)


def attention64(q, k, v, scale: float):
    """softmax(q k^T * scale) v in fp64 with the probabilities: q [.., Tq, d], k / v [.., T, d]."""
    import torch
    s = (q.double() @ k.double().transpose(-1, -2)) * scale
    p = torch.softmax(s, -1)
    return p @ v.double(), p


def attention_bound(q, k, v, p64, o64, scale: float, c_s: float, c_pv: float, r_out: float):
    """Error bound of softmax(q k^T * scale) v for fp32 scores with a relative summation error c_s (of sum |q||k|), a
    relative error c_pv of every probability as used in P V (exp, probability rounding, row-sum), and an output rounding
    r_out:  r_out |o| + (c_pv + 2 c_s scale max_j sum_d |q_d||k_jd|) sum_j p_j |v_j| + 2^-30 (underflow floor)."""
    qk = (q.double().abs() @ k.double().abs().transpose(-1, -2)).amax(-1, keepdim=True)
    pv = p64 @ v.double().abs()
    return r_out * o64.abs() + (c_pv + 2 * c_s * scale * qk) * pv + 2.0 ** -30


SCALE_VIT = 80 ** -0.5


def vit_qkv(kind: str, B: int, H: int, g):
    """fp16 [B*192, 3*H*80] ViT qkv rows (q heads | k heads | v heads) and the q, k, v [B, H, 192, 80] views."""
    import torch
    q = torch.randn(B, H, 192, 80, device="cuda", generator=g)
    k = torch.randn(B, H, 192, 80, device="cuda", generator=g)
    v = torch.randn(B, H, 192, 80, device="cuda", generator=g)
    if kind == "uniform":            # q = 0: every row is the mean of V
        q.zero_()
    elif kind == "dominant":         # row i is dominated by key (37 i) mod 192: every key position, so every one of the
        j = (37 * torch.arange(192, device="cuda")) % 192       # 24 n-tiles and 4 lanes, holds some row's maximum
        q = 1.5 * k[:, :, j]
    elif kind == "large":            # logits of +-300: nearly every exponential underflows
        q, k = 6 * q, 6 * k
    elif kind == "random":
        q, k = 1.5 * q, 1.5 * k
    q, k, v = q.half(), k.half(), v.half()
    qkv = torch.stack([q, k, v], 2).permute(0, 3, 2, 1, 4).reshape(B * 192, 3 * H * 80).contiguous()
    return qkv, q, k, v


def heads_to_rows(o, B, H):
    """[B, H, 192, 80] -> the [B*192, H*80] row layout of the attention output."""
    return o.permute(0, 2, 1, 3).reshape(B * 192, H * 80)


def dec_cross_attn_check(name, q, kv, koff, voff, out, B, heads, scale, r_out):
    """Decoder one-query cross-attention (8 heads x 64) of layer offsets koff / voff into the stacked K/V rows."""
    # scores: 64 fp32 products summed serially (2^-18 of sum |q||k|); probabilities: expf, the 192-term row sum and the
    # divide, then 64 + 3 serial PV additions: 2^-17 of sum p|v|.  Both rigorous (n u bounds).
    kk = kv[:, koff:koff + heads * 64].view(B, 192, heads, 64).permute(0, 2, 1, 3)
    vv = kv[:, voff:voff + heads * 64].view(B, 192, heads, 64).permute(0, 2, 1, 3)
    qq = q.view(B, heads, 1, 64)
    o64, p64 = attention64(qq, kk, vv, scale)
    bound = attention_bound(qq, kk, vv, p64, o64, scale, 2.0 ** -17, 2.0 ** -17, r_out)
    assert_within(f"{name} B={B} koff={koff}", out.view(B, heads, 1, 64), o64, bound)


def im2col_ref(img):
    """Patch rows of the centre crop (columns 32..223, padding 2), k = c*256 + dy*16 + dx: F.pad + F.unfold."""
    import torch.nn.functional as F
    B = img.shape[0]
    crop = F.pad(img[:, :, :, 32:224], (2, 2, 2, 2))
    return F.unfold(crop, 16, stride=16).transpose(1, 2).reshape(B * 192, 768)

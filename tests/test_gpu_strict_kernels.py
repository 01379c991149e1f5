"""Strict-mode stages (csrc/strict.cuh, csrc/engine_strict.cuh) one at a time, through the test-only kernel probe, against
torch fp64 on the same fp32 inputs: the split-fp16 operand builder, the split-precision GEMM (2^-19 of sum|a||w| plus the
tensor cores' truncating accumulation, and a check that this bound rejects the plain fp16 GEMM), the overflow status
word, and the fp32 kernels."""
import pytest
import torch
import torch.nn.functional as F

import probe
from probe import U32, assert_within
from tokenhmr_b200.weights import split_weight

pytestmark = pytest.mark.gpu

ALPHA = 1.0 / (16.0 * 256.0)     # kStrictAlpha: activations are split at 2^4, weights at 2^8
# Split-precision GEMM, per product a.w: hi + lo keeps 22 significand bits of each operand (|a - a'| <= 2^-22 |a|, same
# for w) and the dropped lo.lo term is <= 2^-22 |a||w|: at most 3 * 2^-22 of sum|a||w|.  Inside one 16-product tensor-core
# step the products are aligned and truncated at 2^-23 of the largest one: 3 * 2^-23 of sum|a||w| over the 3K columns.
# Together 1.125 * 2^-20 < 2^-19.  Below |a| = 2^-6 (|w| = 2^-10) the lo part is an fp16 subnormal: absolute floor
# 2^-29 |w| (2^-33 |a|) per product.
C_SPLIT = 2.0 ** -19
# split_rows' GELU is fp32 erff (<= 2 ulp): |GELU error| <= 2^-22 |a| per activation, i.e. 2^-22 sum|a||w| more.
C_GELU = 2.0 ** -22
# The tensor cores' fp32 accumulator is not rounded to nearest: each 16-column step truncates the running sum P_s by up
# to one ulp, 2^-23 |P_s|, and these errors share a sign.  The step count (3K / 16 = 240 at K = 1280) therefore
# multiplies the accumulator's magnitude: 2^-23 sum_s |P_s|, with P_s taken in the kernel's column order (per tap the
# hi.hi products, whose prefix sums grow towards the result, then 2K / 16 correction steps that leave P_s ~ unchanged).
C_TRUNC = 2.0 ** -23


def _trunc_accum(taps):
    """C_TRUNC * sum_s |P_s|: `taps` yields, per tap, the list of fp64 contributions of its 16-column chunks."""
    P = tot = None
    for chunks in taps:
        for c in chunks:
            P = c if P is None else P + c
            tot = P.abs() if tot is None else tot + P.abs()
        tot = tot + 2 * len(chunks) * P.abs()
    return C_TRUNC * tot


def _gemm_chunks(a64, w64):
    return [a64[:, i:i + 16] @ w64[:, i:i + 16].t() for i in range(0, a64.shape[1], 16)]


@pytest.fixture(autouse=True)
def _flags(cuda_dev, built_lib):
    yield
    assert probe.flags() == 0, "probe device flags set"
    assert built_lib.thmr_check_device_flags() == 0, built_lib.thmr_last_error()


def _nan(*shape, dtype=torch.float32):
    return torch.full(shape, float("nan"), dtype=dtype, device="cuda")


def _wide(shape, lo_exp: float, hi_exp: float, g):
    """Random signs, magnitudes log-uniform in [2^lo_exp, 2^hi_exp)."""
    e = lo_exp + (hi_exp - lo_exp) * torch.rand(shape, device="cuda", generator=g)
    s = torch.where(torch.rand(shape, device="cuda", generator=g) < 0.5, -1.0, 1.0)
    return s * torch.exp2(e)


def _split_gemm_bound(a64, w64, act: str, extra):
    mag = a64.abs() @ w64.abs().t()
    floor = 2.0 ** -29 * w64.abs().sum(1)[None, :] + 2.0 ** -33 * a64.abs().sum(1)[:, None]
    return ((C_SPLIT + (C_GELU if act == "gelu" else 0.0)) * mag + _trunc_accum([_gemm_chunks(a64, w64)]) + floor
            + 3 * U32 * extra)


# ------------------------------------------------------------------------------------------------ operand builder
@pytest.mark.parametrize("act", ["none", "gelu", "relu"])
def test_split_rows_hi_lo_and_remap(cuda_dev, act):
    """[hi | lo | hi] of act(x) * 2^4 with hi = fp16(f), lo = fp16(f - hi), and the row remap of the soft-codebook split
    (row b*T + t -> b*pitch + lo + t) leaving the pad rows of the destination untouched."""
    g = torch.Generator(device="cuda").manual_seed(8)
    B, T, PAD, C = 64, 160, 3, 2048
    pitch = T + 2 * PAD
    x = _wide((B * T, C), -8, 11.9, g)
    dst = torch.full((B * pitch, 3 * C), -5.0, dtype=torch.float16, device=cuda_dev)
    probe.split_rows(x, B * T, C, act, T, pitch, PAD, dst=dst)
    torch.cuda.synchronize()
    rows = dst.view(B, pitch, 3 * C)
    assert (rows[:, :PAD] == -5).all() and (rows[:, PAD + T:] == -5).all()
    d = rows[:, PAD:PAD + T].reshape(B * T, 3 * C)
    hi, lo = d[:, :C], d[:, C:2 * C]
    assert torch.equal(d[:, 2 * C:], hi)
    if act != "gelu":
        f = (x.relu() if act == "relu" else x) * 16.0          # exact: power-of-two scale
        assert torch.equal(hi, f.half()) and torch.equal(lo, (f - f.half().float()).half())
    else:
        f = hi.float() + lo.float()                               # exact in fp32
        assert (lo.float().abs() <= 2.0 ** -11 * hi.float().abs()).all()    # lo is at most half an ulp of hi
        a64 = probe.gelu64(x.double())
        assert_within("split_rows gelu", f.double() / 16, a64,
                      2.0 ** -22 * a64.abs() + C_GELU * x.double().abs() + 2.0 ** -29)


def test_split_rows_overflow_flag(cuda_dev):
    """|a| < 4094 fits the split range; 4100 or NaN sets the probe's overflow status word, and reading it clears it."""
    x = torch.zeros(8, 64, device=cuda_dev)
    x[3, 5] = 4090.0
    probe.split_rows(x, 8, 64)
    assert probe.flags() == 0
    for bad in (4100.0, -4100.0, float("nan")):
        y = x.clone()
        y[7, 63] = bad
        probe.split_rows(y, 8, 64)
        assert probe.flags() == probe.FLAG_OVERFLOW, bad
        assert probe.flags() == 0, "reading the flag clears it"


# ------------------------------------------------------------------------------------------------ split GEMM
SPLIT_CASES = {   # name: (M, N, K, act, resid)
    "none": (4096, 256, 1280, "none", None),
    "gelu": (4096, 256, 1280, "gelu", None),
    "relu": (4096, 200, 1280, "relu", None),
    "resid_alias": (4096, 256, 1280, "none", "alias"),
    "resid_mod": (3 * 192, 1280, 768, "none", "table"),   # patch embed: + position table row % 192
    "k160": (64 * 64, 64, 160, "gelu", None),             # mixer tok1: K = 160 is not a multiple of 64
}


def _split_gemm(A32, W32, act, **kw):
    M, K = A32.shape
    N = W32.shape[0]
    Ws = split_weight(W32)
    As = probe.split_rows(A32, M, K, act)
    out = kw.pop("out32", None)
    if out is None:
        out = _nan(M, N)
    probe.gemm(As, Ws, M, N, 3 * K, out32=out, ld32=N, alpha=ALPHA, **kw)
    return out


@pytest.mark.parametrize("case", list(SPLIT_CASES))
def test_split_gemm_vs_fp64(cuda_dev, case):
    """Activations spanning 2^-8 .. 4000 and weights up to 200, packed by weights.split_weight and split by split_rows
    (activation fused), through the GEMM with alpha = 2^-12, against fp64 (bound: C_SPLIT, C_TRUNC)."""
    M, N, K, act, resid = SPLIT_CASES[case]
    g = torch.Generator(device="cuda").manual_seed(list(SPLIT_CASES).index(case))
    A = _wide((M, K), -8, 11.9, g)
    W = _wide((N, K), -10, 7.6, g)
    bias = 1000 * torch.randn(N, device=cuda_dev, generator=g)
    kw, rrows = {}, torch.zeros(M, N, device=cuda_dev)
    if resid == "alias":
        out = 1e4 * torch.randn(M, N, device=cuda_dev, generator=g)
        rrows = out.clone()
        kw = dict(resid=out, ldr=N, out32=out)
    elif resid == "table":
        table = 1e4 * torch.randn(192, N, device=cuda_dev, generator=g)
        rrows = table[torch.arange(M, device=cuda_dev) % 192]
        kw = dict(resid=table, ldr=N, resid_mod=192)
    out = _split_gemm(A, W, act, bias=bias, **kw)
    torch.cuda.synchronize()
    a64 = probe.act64(A.double(), act)
    y64 = a64 @ W.double().t() + bias.double() + rrows.double()
    bound = _split_gemm_bound(a64, W.double(), act, y64.abs() + bias.double().abs() + rrows.double().abs())
    assert_within(f"split_gemm[{case}]", out, y64, bound)


@pytest.mark.parametrize("dil", [1, 3])
def test_split_conv_taps_padded_sequences(cuda_dev, dil):
    """Strict Conv1d(k=3, dilation): split operands of all padded rows, weights packed per tap [hi | hi | lo]
    (split_weight taps = 3), the implicit GEMM over cin = 3 C with tap_row0 = -dil across the batch boundaries."""
    g = torch.Generator(device="cuda").manual_seed(30 + dil)
    B, L, PAD, C, cout = 7, 55, 3, 256, 192
    Lp = L + 2 * PAD
    x = torch.zeros(B, Lp, C, device=cuda_dev)
    x[:, PAD:PAD + L] = _wide((B, L, C), -8, 11.9, g)
    w = _wide((cout, C, 3), -10, 7.6, g)
    wt = w.permute(0, 2, 1).reshape(cout, 3 * C)                 # tap-major [Cout, 3*Cin] (weights.py conv())
    bias = torch.randn(cout, device=cuda_dev, generator=g)
    As = probe.split_rows(x.view(B * Lp, C), B * Lp, C, "relu")
    Ws = split_weight(wt, taps=3)
    out = _nan(B * Lp, cout)
    probe.gemm(As, Ws, B * Lp, cout, 9 * C, lda=3 * C, ldb=9 * C, bias=bias, out32=out, ld32=cout, taps=3, cin=3 * C,
               tap_row0=-dil, tap_stride=dil, seq=(Lp, PAD, PAD + L), alpha=ALPHA)
    torch.cuda.synchronize()
    xs = x[:, PAD:PAD + L].double().relu().permute(0, 2, 1)
    y64 = F.conv1d(xs, w.double(), bias.double(), padding=dil, dilation=dil).permute(0, 2, 1)
    mag = F.conv1d(xs.abs(), w.double().abs(), padding=dil, dilation=dil).permute(0, 2, 1)
    floor = 2.0 ** -29 * w.double().abs().sum((1, 2)) + 2.0 ** -33 * 3 * float(xs.abs().sum(1).max())
    xt = F.pad(xs, (dil, dil)).permute(0, 2, 1)                 # tap t of output l reads input l + (t - 1) dil
    taps = ([xt[:, t * dil:t * dil + L, i:i + 16] @ w.double()[:, i:i + 16, t].t() for i in range(0, C, 16)]
            for t in range(3))
    o = out.view(B, Lp, cout)
    bound = C_SPLIT * mag + _trunc_accum(taps) + floor + 3 * U32 * (y64.abs() + bias.double().abs())
    assert_within(f"split_conv dil={dil}", o[:, PAD:PAD + L], y64, bound)
    assert torch.equal(o[:, :PAD], torch.zeros_like(o[:, :PAD])) and torch.equal(o[:, PAD + L:], torch.zeros_like(o[:, PAD + L:]))


def test_split_bound_rejects_plain_fp16_gemm(cuda_dev):
    """Self-check of the bound: on the same data the default mode's fp16-operand GEMM (thmr_gemm_f16) is far outside
    the split-precision bound, so the strict tests can tell the two modes apart."""
    from tokenhmr_b200._lib import check, lib
    g = torch.Generator(device="cuda").manual_seed(99)
    M, N, K = 1024, 256, 1280
    A = _wide((M, K), -8, 11.9, g)
    W = _wide((N, K), -10, 7.6, g)
    split = _split_gemm(A, W, "none")
    plain = _nan(M, N)
    A16, W16 = A.half(), W.half()
    check(lib().thmr_gemm_f16(A16.data_ptr(), K, W16.data_ptr(), K, M, N, K, None, None, 0, 0, plain.data_ptr(), N,
                              None, 0, 0, probe.stream()))
    torch.cuda.synchronize()
    y64 = A.double() @ W.double().t()
    bound = _split_gemm_bound(A.double(), W.double(), "none", y64.abs())
    assert_within("split_gemm (self-check data)", split, y64, bound)
    ratio = ((plain.double() - y64).abs() / bound)
    print(f"[bound] plain fp16 GEMM against the split bound: median err/bound {float(ratio.median()):.3g}, "
          f"max {float(ratio.max()):.3g}")
    assert float((ratio > 1).double().mean()) > 0.5, "the split bound does not separate fp16 operands from split ones"


# ------------------------------------------------------------------------------------------------ fp32 kernels
def test_attention_f32_vs_fp64(cuda_dev):
    """The strict fp32 CUDA-core attention on the fast kernel's data (random, uniform, one dominant key per row covering
    every key position, +-300 logits) at B = 64, H = 16."""
    B, H = 64, 16
    for kind in ("random", "uniform", "dominant", "large"):
        qkv, q, k, v = probe.vit_qkv(kind, B, H, torch.Generator(device="cuda").manual_seed(5))
        q32 = qkv.float()
        out = _nan(B * 192, H * 80)
        probe.call("probe_attention_f32", q32.data_ptr(), 3 * H * 80, B, H, out.data_ptr(), H * 80, probe.SCALE_VIT,
                   probe.stream())
        torch.cuda.synchronize()
        o64, p64 = probe.attention64(q, k, v, probe.SCALE_VIT)
        # scores: four fp32 FMA chains of 20 products + 2 adds (2^-19 of sum |q||k|, rigorous); probabilities: expf of
        # the rounded s - max, a 192-term serial row sum and a 192-term serial PV FMA chain whose rounding errors are
        # independent (sqrt(192) 2^-24 = 2^-20.2): 2^-18 (~4e-6) with a 4-sigma margin; fp32 output.
        bound = probe.attention_bound(q, k, v, p64, o64, probe.SCALE_VIT, 2.0 ** -19, 2.0 ** -18, 2 * U32)
        assert_within(f"attention_f32[{kind}]", out, probe.heads_to_rows(o64, B, H), probe.heads_to_rows(bound, B, H))


@pytest.mark.parametrize("B", [1, 64, 65])
@pytest.mark.parametrize("layer", [0, 5])
def test_dec_cross_attn_f32(cuda_dev, B, layer):
    heads, ld, scale = 8, 6144, 64 ** -0.5
    g = torch.Generator(device="cuda").manual_seed(B * 10 + layer)
    q = 3 * torch.randn(B, heads * 64, device=cuda_dev, generator=g)
    kv = 2 * torch.randn(B * 192, ld, device=cuda_dev, generator=g)
    koff, voff = 1024 * layer, 1024 * layer + 512
    out = _nan(B, heads * 64)
    probe.call("probe_dec_cross_attn_f32", q.data_ptr(), kv.data_ptr(), ld, koff, voff, scale, out.data_ptr(), B, heads,
               probe.stream())
    torch.cuda.synchronize()
    probe.dec_cross_attn_check("dec_cross_attn f32", q, kv, koff, voff, out, B, heads, scale, 2 * U32)


def test_im2col_patch_f32_and_relu_inplace(cuda_dev):
    B = 3
    img = torch.randn(B, 3, 256, 256, device=cuda_dev, generator=torch.Generator(device="cuda").manual_seed(2))
    out = _nan(B * 192, 768)
    probe.call("probe_im2col_patch_f32", img.data_ptr(), out.data_ptr(), B, 256, 32, 192, 16, 2, 16, 12, probe.stream())
    torch.cuda.synchronize()
    assert torch.equal(out, probe.im2col_ref(img))
    x = torch.randn(64, 27, 512, device=cuda_dev)
    want = x.relu()
    probe.call("probe_relu_inplace", x.data_ptr(), x.numel() // 4, probe.stream())
    torch.cuda.synchronize()
    assert torch.equal(x, want)

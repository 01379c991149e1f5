"""Default-mode kernels the engine dispatches, one stage at a time, through the test-only kernel probe
(tests/csrc/kernel_probe.cu) against torch fp64 on the same rounded inputs the kernel sees.

Bounds are per element and scale-free (probe.assert_within); gathers and scatters must match exactly."""
import pytest
import torch
import torch.nn.functional as F

import probe
from probe import U16, U32, assert_within

pytestmark = pytest.mark.gpu

# fp32 accumulation of fp16 products on the tensor cores: the products are exact, and each of the K/16 accumulator
# updates rounds (or truncates) at 2^-24 .. 2^-23 of a partial sum.  For the zero-mean products used here a partial sum
# stays near sum|a||w| / sqrt(K), so the accumulated error stays below ~2^-22 sum|a||w| for every K up to 5120;
# 2^-20 leaves a 4x margin and is still 2^9 below the fp16 operand rounding (2^-11) that the default mode accepts.
C_ACC = 2.0 ** -20
# The epilogue's exact-erf GELU (gemm_wgmma.cuh gelu_erf, Abramowitz-Stegun 7.1.28): |erf error| < 2e-6 -> |x| 2^-20 / 2.
GELU_ERR = 2.0 ** -21
GELU_LIP = 1.13     # max |GELU'(x)|


@pytest.fixture(autouse=True)
def _flags(cuda_dev, built_lib):
    yield
    assert probe.flags() == 0, "probe device flags set"
    assert built_lib.thmr_check_device_flags() == 0, built_lib.thmr_last_error()


def _nan(*shape, dtype=torch.float32):
    return torch.full(shape, float("nan"), dtype=dtype, device="cuda")


# ------------------------------------------------------------------------------------------------ GEMM epilogues
M_G, K_G = 576, 320        # 3 x 192 rows (three images of the patch-embed position table), 5 k-blocks
SEQ = (192, 5, 170)        # padded sequences: rows with row % 192 outside [5, 170) are stored as zero
EPILOGUES = {
    "alpha": dict(alpha=0.3),
    "resid_mod": dict(resid="table"),
    "seq_relu": dict(seq=True, act="relu"),
    "act32_relu": dict(act="relu", act32=1),
    "act32_gelu": dict(act="gelu", act32=1),
    "ld16_ld32": dict(ld16=8, ld32=4, act="gelu"),
    "resid_alias": dict(resid="alias"),
    "all": dict(alpha=0.3, seq=True, act="gelu", ld16=8, resid="rows", ldr=12),
    "all_act32_alias": dict(alpha=0.3, seq=True, act="relu", act32=1, resid="alias", ld32=2),
    "table_seq_gelu": dict(alpha=0.5, seq=True, act="gelu", resid="table", ld16=16),
}


@pytest.mark.parametrize("N", [198, 197])
@pytest.mark.parametrize("bn", [32, 64, 128, 256])
@pytest.mark.parametrize("case", list(EPILOGUES))
def test_gemm_epilogue_options(cuda_dev, case, bn, N):
    """alpha, the position-table residual (resid_mod), padded-sequence masking, act32, ld16 != N and a residual aliasing
    the fp32 output, alone and combined, at every tile width.  The epilogue order is alpha*acc + bias + resid -> mask ->
    act: masked rows are exactly zero in both outputs, and pitch padding is never written."""
    o = EPILOGUES[case]
    g = torch.Generator(device="cuda").manual_seed(1000 * list(EPILOGUES).index(case) + bn + N)
    M, K = M_G, K_G
    A = torch.randn(M, K, device=cuda_dev, generator=g).half()
    W = (0.1 * torch.randn(N, K, device=cuda_dev, generator=g)).half()
    bias = torch.randn(N, device=cuda_dev, generator=g)
    alpha, act, act32 = o.get("alpha", 1.0), o.get("act", "none"), o.get("act32", 0)
    ld32, ld16 = N + o.get("ld32", 0), N + o.get("ld16", 0)
    out32, out16 = _nan(M, ld32), _nan(M, ld16, dtype=torch.float16)
    resid, ldr, resid_mod, rrows = None, 0, 0, torch.zeros(M, N, device=cuda_dev)
    if o.get("resid") == "table":
        resid, ldr, resid_mod = torch.randn(192, N, device=cuda_dev, generator=g), N, 192
        rrows = resid[torch.arange(M, device=cuda_dev) % 192]
    elif o.get("resid") == "rows":
        ldr = N + o.get("ldr", 0)
        resid = torch.randn(M, ldr, device=cuda_dev, generator=g)
        rrows = resid[:, :N]
    elif o.get("resid") == "alias":      # in-place residual add: out32 = out32 + ...
        out32[:, :N] = torch.randn(M, N, device=cuda_dev, generator=g)
        resid, ldr, rrows = out32, ld32, out32[:, :N].clone()
    seq = SEQ if o.get("seq") else (0, 0, 0)
    probe.gemm(A, W, M, N, K, bias=bias, resid=resid, ldr=ldr, resid_mod=resid_mod, act=act, act32=act32,
               out32=out32, ld32=ld32, out16=out16, ld16=ld16, seq=seq, alpha=alpha, force_bn=bn)
    torch.cuda.synchronize()

    A64, W64 = A.double(), W.double()
    y64 = alpha * (A64 @ W64.t()) + bias.double() + rrows.double()
    b32 = C_ACC * abs(alpha) * (A64.abs() @ W64.abs().t()) + 3 * U32 * (y64.abs() + bias.double().abs()
                                                                        + rrows.double().abs())
    keep = torch.ones(M, dtype=torch.bool, device=cuda_dev)
    if seq[0]:
        r = torch.arange(M, device=cuda_dev) % seq[0]
        keep = (r >= seq[1]) & (r < seq[2])
    ya = probe.act64(y64, act)
    ref32, bnd32 = (ya, GELU_LIP * b32 + GELU_ERR * y64.abs()) if act32 else (y64, b32)
    bnd16 = U16 * ya.abs() + GELU_LIP * b32 + GELU_ERR * y64.abs() + 2.0 ** -25
    got32, got16 = out32[:, :N], out16[:, :N]
    assert_within(f"gemm[{case}] out32", got32[keep], ref32[keep], bnd32[keep])
    assert_within(f"gemm[{case}] out16", got16[keep], ya[keep], bnd16[keep])
    if not bool(keep.all()):
        z = ~keep
        assert torch.equal(got32[z], torch.zeros_like(got32[z])) and torch.equal(got16[z], torch.zeros_like(got16[z]))
        assert not torch.signbit(got32[z]).any()
    assert torch.isnan(out32[:, N:]).all() and torch.isnan(out16[:, N:]).all()


@pytest.mark.parametrize("dil", [1, 3])
@pytest.mark.parametrize("bn", [0, 64])
def test_gemm_implicit_conv_padded_sequences(cuda_dev, dil, bn):
    """The tokenizer's Conv1d(k=3, dilation) as the implicit GEMM over zero-padded sequences (taps = 3, tap_row0 =
    -dil): taps read across the sequence (and batch) boundaries into the pad rows, which are stored as zero again."""
    g = torch.Generator(device="cuda").manual_seed(17 + dil + bn)
    B, L, PAD, cin, cout = 5, 55, 3, 128, 192
    Lp = L + 2 * PAD
    x = torch.zeros(B, Lp, cin, device=cuda_dev)
    x[:, PAD:PAD + L] = torch.randn(B, L, cin, device=cuda_dev, generator=g)
    x16 = x.half()
    w = (0.05 * torch.randn(cout, cin, 3, device=cuda_dev, generator=g)).half()
    wt = w.permute(0, 2, 1).reshape(cout, 3 * cin).contiguous()      # tap-major, as weights.py packs it
    bias = torch.randn(cout, device=cuda_dev, generator=g)
    out32, out16 = _nan(B * Lp, cout), _nan(B * Lp, cout, dtype=torch.float16)
    probe.gemm(x16.view(B * Lp, cin), wt, B * Lp, cout, 3 * cin, lda=cin, ldb=3 * cin, bias=bias, act="relu",
               out32=out32, ld32=cout, out16=out16, ld16=cout, taps=3, cin=cin, tap_row0=-dil, tap_stride=dil,
               seq=(Lp, PAD, PAD + L), force_bn=bn)
    torch.cuda.synchronize()
    xs = x16[:, PAD:PAD + L].double().permute(0, 2, 1)
    y64 = F.conv1d(xs, w.double(), bias.double(), padding=dil, dilation=dil).permute(0, 2, 1)
    mag = F.conv1d(xs.abs(), w.double().abs(), padding=dil, dilation=dil).permute(0, 2, 1)
    b32 = C_ACC * mag + 3 * U32 * (y64.abs() + bias.double().abs())
    o32, o16 = out32.view(B, Lp, cout), out16.view(B, Lp, cout)
    assert_within(f"conv dil={dil} out32", o32[:, PAD:PAD + L], y64, b32)
    assert_within(f"conv dil={dil} out16", o16[:, PAD:PAD + L], y64.relu(), U16 * y64.relu() + b32 + 2.0 ** -25)
    for sl in (slice(0, PAD), slice(PAD + L, Lp)):
        assert torch.equal(o32[:, sl], torch.zeros_like(o32[:, sl])) and torch.equal(o16[:, sl], torch.zeros_like(o16[:, sl]))


# ------------------------------------------------------------------------------------------------ ViT attention
# mma.sync scores: 80 exact products, 5 fp32 accumulator updates -> 2^-22 of sum |q||k|.  Probabilities as used in PV:
# fp16 rounding of exp2 (2^-11) + ex2.approx (2^-22) + the fp32 row sum of 192 terms and the PV accumulation (both
# below 2^-18) -> 2^-11 + 2^-17.  Output rounded to fp16 (2^-11).
C_S_FAST, C_PV_FAST = 2.0 ** -22, U16 + 2.0 ** -17


@pytest.mark.parametrize("kind", ["random", "uniform", "dominant", "large"])
def test_vit_attention_fast_vs_fp64(cuda_dev, kind):
    """The fused mma.sync attention at the ViT shape (B = 64, H = 16) against fp64 softmax(q k^T / sqrt(80)) v."""
    B, H = 64, 16
    qkv, q, k, v = probe.vit_qkv(kind, B, H, torch.Generator(device="cuda").manual_seed(5))
    out = torch.empty(B * 192, H * 80, dtype=torch.float16, device=cuda_dev)
    probe.call("probe_vit_attention", qkv.data_ptr(), B, H, out.data_ptr(), probe.stream())
    torch.cuda.synchronize()
    o64, p64 = probe.attention64(q, k, v, probe.SCALE_VIT)
    bound = probe.attention_bound(q, k, v, p64, o64, probe.SCALE_VIT, C_S_FAST, C_PV_FAST, U16)
    bound = bound + 2.0 ** -25 * v.double().abs().sum(-2, keepdim=True)   # exp2 values below 2^-14 are fp16 subnormals
    assert_within(f"vit_attention[{kind}]", out, probe.heads_to_rows(o64, B, H), probe.heads_to_rows(bound, B, H))


# ------------------------------------------------------------------------------------------------ decoder cross-attention
@pytest.mark.parametrize("B", [1, 64, 65])
@pytest.mark.parametrize("layer", [0, 5])
def test_dec_cross_attn_f16(cuda_dev, B, layer):
    """One-query cross-attention over the 192 ViT tokens of the stacked K/V of six layers (ld = 6144): layer l reads
    K at columns 1024 l and V at 1024 l + 512 of the fp16 to_kv output."""
    heads, ld, scale = 8, 6144, 64 ** -0.5
    g = torch.Generator(device="cuda").manual_seed(B * 10 + layer)
    q = 3 * torch.randn(B, heads * 64, device=cuda_dev, generator=g)
    kv = (2 * torch.randn(B * 192, ld, device=cuda_dev, generator=g)).half()
    koff, voff = 1024 * layer, 1024 * layer + 512
    out = torch.empty(B, heads * 64, dtype=torch.float16, device=cuda_dev)
    probe.call("probe_dec_cross_attn", q.data_ptr(), kv.data_ptr(), ld, koff, voff, scale, out.data_ptr(), B, heads,
               probe.stream())
    torch.cuda.synchronize()
    probe.dec_cross_attn_check("dec_cross_attn f16", q, kv, koff, voff, out, B, heads, scale, U16)


# ------------------------------------------------------------------------------------------------ LayerNorm
def _ln_vec4(C: int) -> int:
    v = (C // 4 + 31) // 32
    return 1 if v <= 1 else 8 if v <= 8 else 10 if v <= 10 else 16


def ln_check(name, x, g, b, eps, relu, y, fp16: bool):
    """Two-pass LayerNorm bound: the mean and the variance are recursive sums with n = 2 VEC4 + 6 roundings per term
    (register kernels: two lane chains of 2 VEC4 terms, a 5-level shuffle tree) or C / 256 + 14 (wide kernel), so
    |d mean| <= n u mean|x| and |d rstd| / rstd <= (n / 2 + 2) u; the output adds 3 roundings and fp16 2^-11."""
    C = x.shape[-1]
    n = (2 * _ln_vec4(C) + 6) if C <= 2048 else (C // 256 + 14)
    x64 = x.double()
    mu = x64.mean(-1, keepdim=True)
    rstd = 1 / torch.sqrt(x64.var(-1, unbiased=False, keepdim=True) + eps)
    y64 = F.layer_norm(x64, (C,), g.double(), b.double(), eps)
    d_mu = n * U32 * x64.abs().mean(-1, keepdim=True)
    bnd = g.double().abs() * rstd * (d_mu + (x64 - mu).abs() * (n / 2 + 2) * U32) + 3 * U32 * (y64.abs() + b.double().abs())
    if relu:
        y64 = y64.relu()
    if fp16:
        bnd = bnd + U16 * y64.abs() + 2.0 ** -25
    assert_within(name, y, y64, bnd)


LN_CASES = [   # (R, C, outputs, relu): every dispatch variant of layernorm_launch
    (1, 64, "both", 0), (10240, 64, "both", 0),           # V1
    (1, 128, "16", 0), (777, 128, "16", 0),               # V1 PLAIN16
    (300, 520, "both", 1), (300, 1024, "32", 0),          # V8
    (300, 1024, "16", 0),                                 # V8 PLAIN16
    (300, 1152, "32", 1), (1, 1280, "16", 0),             # V10, V10 PLAIN16 (the ViT's LayerNorm) ...
    (12288, 1280, "16", 0),                               # ... at bs = 64: every warp walks ~3 rows
    (12288, 1536, "both", 0), (100, 2048, "32", 1),       # V16
    (4500, 2048, "16", 0),                                # V16 PLAIN16
    (3, 10240, "32", 1), (2, 4100, "both", 0),            # wide kernel
]


@pytest.mark.parametrize("R,C,outs,relu", LN_CASES)
@pytest.mark.parametrize("mean", [0.0, 1000.0])
def test_layernorm_dispatch_variants(cuda_dev, R, C, outs, relu, mean):
    """Rows of mean 1000 and std 1 separate two-pass statistics (which pass) from a one-pass E[x^2] - E[x]^2."""
    gen = torch.Generator(device="cuda").manual_seed(R + C)
    x = mean + (1.0 if mean else 3.0) * torch.randn(R, C, device=cuda_dev, generator=gen)
    g, b = torch.randn(C, device=cuda_dev, generator=gen), torch.randn(C, device=cuda_dev, generator=gen)
    eps = 1e-6 if C == 1280 else 1e-5
    y16 = _nan(R, C, dtype=torch.float16) if outs in ("16", "both") else None
    y32 = _nan(R, C) if outs in ("32", "both") else None
    probe.call("probe_layernorm", x.data_ptr(), g.data_ptr(), b.data_ptr(), probe.ptr(y16), 0, probe.ptr(y32), R, C,
               eps, relu, 0, probe.stream())
    torch.cuda.synchronize()
    if y32 is not None:
        ln_check(f"layernorm R={R} C={C} fp32", x, g, b, eps, relu, y32, False)
    if y16 is not None:
        ln_check(f"layernorm R={R} C={C} fp16", x, g, b, eps, relu, y16, True)


@pytest.mark.parametrize("outs", ["16", "32", "both"])
def test_layernorm_transposed_output(cuda_dev, outs):
    """Mixer token mixing: C = 64, outputs transposed inside groups of out_t = 160 rows (bs = 64: 10240 rows)."""
    B, T, C = 64, 160, 64
    gen = torch.Generator(device="cuda").manual_seed(3)
    x = 2 * torch.randn(B * T, C, device=cuda_dev, generator=gen) + 0.5
    g, b = torch.randn(C, device=cuda_dev, generator=gen), torch.randn(C, device=cuda_dev, generator=gen)
    y16 = _nan(B * C * T, dtype=torch.float16) if outs in ("16", "both") else None
    y32 = _nan(B * C * T) if outs in ("32", "both") else None
    probe.call("probe_layernorm", x.data_ptr(), g.data_ptr(), b.data_ptr(), probe.ptr(y16), 0, probe.ptr(y32), B * T,
               C, 1e-5, 0, T, probe.stream())
    torch.cuda.synchronize()
    for y, fp16 in ((y16, True), (y32, False)):
        if y is not None:     # (B, C, T) -> rows (b, t)
            ln_check(f"layernorm out_t=160 fp{16 if fp16 else 32}", x, g, b, 1e-5, 0,
                     y.view(B, C, T).permute(0, 2, 1).reshape(B * T, C), fp16)


# ------------------------------------------------------------------------------------------------ softmax rows
@pytest.mark.parametrize("C", [2048, 520])
def test_softmax_rows_and_padded_scatter(cuda_dev, C):
    """Classifier softmax over x20-scaled logits (bs = 64: 10240 rows), including rows shifted by +-200 that overflow /
    underflow every exponential unless the row maximum is subtracted; the fp16 copy lands at row b*pitch + lo + t and
    the pad rows of the padded layout are never written."""
    B, T, PAD = 64, 160, 3
    pitch, R = T + 2 * PAD, B * T
    gen = torch.Generator(device="cuda").manual_seed(C)
    x = 20 * torch.randn(R, C, device=cuda_dev, generator=gen)
    x[::7] += 200.0
    x[3::7] -= 200.0
    p32 = _nan(R, C)
    p16 = torch.full((B * pitch, C), -7.0, dtype=torch.float16, device=cuda_dev)
    probe.call("probe_softmax_rows", x.data_ptr(), p32.data_ptr(), p16.data_ptr(), R, C, T, pitch, PAD, probe.stream())
    torch.cuda.synchronize()
    x64 = x.double()
    p64 = torch.softmax(x64, -1)
    # expf (2 ulp) of x - max (rounded: u |x - m|), a 70-term row sum (lane chains of 64 + 5-level tree), 1/sum, product
    bound = p64 * U32 * ((x64 - x64.amax(-1, keepdim=True)).abs() + 80) + 2.0 ** -120
    assert_within(f"softmax C={C}", p32, p64, bound)
    assert ((p32.double().sum(-1) - 1).abs() <= bound.sum(-1)).all()
    rows = p16.view(B, pitch, C)
    assert torch.equal(rows[:, PAD:PAD + T], p32.half().view(B, T, C))
    assert (rows[:, :PAD] == -7).all() and (rows[:, PAD + T:] == -7).all()


# ------------------------------------------------------------------------------------------------ gathers
UPSAMPLE_CHAINS = {"decoder": [160, 125, 90, 55, 21], "encoder": [21, 40, 80, 160, 320]}


@pytest.mark.parametrize("chain", list(UPSAMPLE_CHAINS))
@pytest.mark.parametrize("dtype", [torch.float16, torch.float32])
def test_upsample_rows_equals_interpolate_nearest(cuda_dev, chain, dtype):
    """nn.Upsample(size) nearest on zero-padded channels-last sequences: the release sizes of the pose decoder
    (fp16 rows, C / 8 units; fp32 rows in strict mode, C / 4 units) and of the tokenizer encoder (fp32)."""
    B, W, PAD = 5, 512, 3
    gen = torch.Generator(device="cuda").manual_seed(1)
    units = W * torch.finfo(dtype).bits // 128
    sizes = UPSAMPLE_CHAINS[chain]
    for Lin, Lout in zip(sizes[:-1], sizes[1:]):
        src = torch.zeros(B, Lin + 2 * PAD, W, dtype=dtype, device=cuda_dev)
        src[:, PAD:PAD + Lin] = torch.randn(B, Lin, W, device=cuda_dev, generator=gen).to(dtype)
        dst = torch.full((B, Lout + 2 * PAD, W), 7.0, dtype=dtype, device=cuda_dev)
        probe.call("probe_upsample_rows", src.data_ptr(), dst.data_ptr(), B, Lin, Lout, PAD, units, probe.stream())
        torch.cuda.synchronize()
        want = F.interpolate(src[:, PAD:PAD + Lin].permute(0, 2, 1), size=Lout, mode="nearest").permute(0, 2, 1)
        assert torch.equal(dst[:, PAD:PAD + Lout], want), (Lin, Lout)
        assert (dst[:, :PAD] == 0).all() and (dst[:, PAD + Lout:] == 0).all()


def test_im2col_patch_f16(cuda_dev):
    """Patch im2col of the centre crop (columns 32..223, padding 2) in the PatchEmbed weight order (c, dy, dx)."""
    B = 3
    img = torch.randn(B, 3, 256, 256, device=cuda_dev, generator=torch.Generator(device="cuda").manual_seed(2))
    out = _nan(B * 192, 768, dtype=torch.float16)
    probe.call("probe_im2col_patch", img.data_ptr(), out.data_ptr(), B, 256, 32, 192, 16, 2, 16, 12, probe.stream())
    torch.cuda.synchronize()
    assert torch.equal(out, probe.im2col_ref(img).half())


def test_mixer_add(cuda_dev):
    """out = x + y^T (+ z): the token-mix output (B, H, T) added back in the (B*T, H) layout."""
    B, T, H = 64, 160, 64
    gen = torch.Generator(device="cuda").manual_seed(4)
    x, yT, z = (torch.randn(*s, device=cuda_dev, generator=gen) for s in ((B * T, H), (B, H, T), (B * T, H)))
    for zz in (None, z):
        out = _nan(B * T, H)
        probe.call("probe_mixer_add", x.data_ptr(), yT.data_ptr(), probe.ptr(zz), out.data_ptr(), B, T, H, probe.stream())
        torch.cuda.synchronize()
        want = x + yT.permute(0, 2, 1).reshape(B * T, H)
        assert torch.equal(out, want if zz is None else want + zz)


def test_cast_f16(cuda_dev):
    x = 100 * torch.randn(64, 1024, device=cuda_dev)
    out = _nan(64, 1024, dtype=torch.float16)
    probe.call("probe_cast_f16", x.data_ptr(), out.data_ptr(), x.numel() // 4, probe.stream())
    torch.cuda.synchronize()
    assert torch.equal(out, x.half())


def test_head_assemble_vs_oracle(cuda_dev):
    """Read-out assembly: pose6d = cat[grot, body pose rows of the padded tokenizer output, hands] + init_pose, betas,
    cam, and rot6d -> rotation matrices against oracle.tokenhmr_oracle.rot6d_to_rotmat in fp64."""
    from oracle import tokenhmr_oracle as O
    B, PAD, Lj, nb = 65, 3, 21, 10
    Lp = Lj + 2 * PAD
    gen = torch.Generator(device="cuda").manual_seed(6)
    readout = torch.randn(B, 32, device=cuda_dev, generator=gen)
    bpose = torch.randn(B * Lp, 8, device=cuda_dev, generator=gen)
    init_pose = torch.randn(144, device=cuda_dev, generator=gen)
    init_betas, init_cam = torch.randn(nb, device=cuda_dev, generator=gen), torch.randn(3, device=cuda_dev, generator=gen)
    rot, betas, cam, pose6d = _nan(B, 24, 9), _nan(B, nb), _nan(B, 3), _nan(B, 144)
    probe.call("probe_head_assemble", readout.data_ptr(), 32, bpose.data_ptr(), 8, Lp, PAD, init_pose.data_ptr(),
               init_betas.data_ptr(), init_cam.data_ptr(), rot.data_ptr(), betas.data_ptr(), cam.data_ptr(),
               pose6d.data_ptr(), B, nb, probe.stream())
    torch.cuda.synchronize()
    body = bpose.view(B, Lp, 8)[:, PAD:PAD + Lj, :6].reshape(B, 126)
    want6d = torch.cat([readout[:, :6], body, readout[:, 6:18]], -1) + init_pose         # token_head.py:103
    assert torch.equal(pose6d, want6d)
    assert torch.equal(betas, readout[:, 18:28] + init_betas) and torch.equal(cam, readout[:, 28:31] + init_cam)
    x = want6d.double().cpu().view(B * 24, 6)
    R64 = O.rot6d_to_rotmat(x).view(B, 24, 9)
    # ~16 roundings; the Gram-Schmidt subtraction amplifies them by |a2| / |a2 - (b1.a2) b1|
    a1, a2 = x[:, :3], x[:, 3:]
    u = a2 - (F.normalize(a1, dim=-1) * a2).sum(-1, keepdim=True) * F.normalize(a1, dim=-1)
    amp = (1 + a2.norm(dim=-1) / u.norm(dim=-1)).view(B, 24, 1)
    assert_within("head_assemble rotmats", rot.cpu(), R64, 2.0 ** -19 * amp.expand(B, 24, 9))

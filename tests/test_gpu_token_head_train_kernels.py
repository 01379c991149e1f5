"""The token head's training kernels (csrc/token_head_train.cuh) one at a time, through the head-training probe
(tests/csrc/head_train_probe.cu), against torch fp64 on the fp32 values each kernel reads: im2col and its gather
backward through the tokenizer's resize maps; the conv composites at every tokenizer call shape; LayerNorm at widths
10240 and 64 with the fused ReLU masks; the softmax at peaky logits; the two-stage column sums over one, two, three and
130 partials; the batched transpose and the ReLU copy; hl_gemm on a table of the token head's call sites whose split
counts the test asserts.  Then the whole head (heads.TokenHead) at the first batch sizes with several wide column-sum
partials and empty split-K splits, and at decoder shapes that move every tail parameter's offset.

As tests/test_gpu_head_train_kernels.py: bounds are per element and derived in comments from each kernel's order of
operations (probe.assert_within); integer inputs make the copies, gathers, GEMMs and column sums exact, and those are
compared bit for bit; every output starts as NaN and pitch padding must still be NaN afterwards; every launch runs
twice with bit-identical results; each bound family rejects an fp64 reference with one term taken out."""
import dataclasses
import zlib

import pytest
import torch
import torch.nn.functional as F

import head_train_probe as hp
import probe
from head_train_probe import _linear, _linear_dw, _linear_dx, _nan, _rejects, _twice, Site, gamma
from probe import U32, assert_within

pytestmark = pytest.mark.gpu

T, HID, MIX, CLS, CODE, WIDTH, JOINTS = 160, 64, 10240, 2048, 256, 512, 21
UPS = (125, 90, 55, 21)                      # kTkUpLen
COL_ROWS = 160                               # kTkColRows
READ_LD = 160                                # kRhReadLd
EPS = 9.99999974737875e-06                   # kRhLnEps: the fp32 value of 1e-5
TINY = 2.0 ** -126                           # absolute floor where a result may be subnormal


@pytest.fixture(autouse=True)
def _flags(cuda_dev, built_lib):
    yield
    assert hp.flags() == 0, "head-train probe device flags set"
    assert built_lib.thmr_check_device_flags() == 0, built_lib.thmr_last_error()


def _gen(*key):
    return torch.Generator(device="cuda").manual_seed(zlib.crc32(repr(key).encode()))


def _ints(shape, g, lo=-4, hi=5):
    return torch.randint(lo, hi, shape, device="cuda", generator=g).float()


# ------------------------------------------------------------------------------------------------ im2col / col2im
# fp64 restatement: nn.Upsample(size) 'nearest' through ATen's fp32 map (F.interpolate on fp32 input: the map the
# kernels use, tests/test_token_head_probe_host.py), ReLU, zero padding of dil * (taps // 2) at both ends, and the
# taps as columns c * taps + j.
def _src(lin, lout):
    """ATen's nearest map on fp32 input, for use as an index gather.  The references never differentiate through
    F.interpolate itself: on the GPU its backward at 125 -> 90 credits input 74 with the output its forward reads
    from input 75 (test_seq_map_matches_aten_on_the_gpu records it; on the host the two agree)."""
    return F.interpolate(torch.arange(lin, dtype=torch.float32, device="cuda").view(1, 1, lin), size=lout,
                         mode="nearest").view(lout).long()


def _im2col64(X, lin, lout, taps, dil, relu):
    """X (B, lin, Cin) -> col (B * lout, Cin * taps), in X's dtype."""
    B, _, Cin = X.shape
    xr = X[:, _src(lin, lout), :]
    if relu:
        xr = torch.relu(xr)
    pad = dil * (taps // 2)
    xp = F.pad(xr.transpose(1, 2), (pad, pad))                            # (B, Cin, lout + 2 pad)
    win = xp.unfold(2, (taps - 1) * dil + 1, 1)[..., ::dil]               # (B, Cin, lout, taps)
    return win.permute(0, 2, 1, 3).reshape(B * lout, Cin * taps)


def _col2im64(dcol, B, Cin, lin, lout, taps, dil):
    """The adjoint of _im2col64 (no ReLU): fp64 autograd."""
    X = torch.zeros(B, lin, Cin, dtype=torch.float64, device=dcol.device, requires_grad=True)
    (g,) = torch.autograd.grad((_im2col64(X, lin, lout, taps, dil, False) * dcol.double()).sum(), X)
    return g.reshape(B * lin, Cin)


def _im2col(X, Cin, lin, lout, taps, dil, relu, B, pad=7):
    col = _nan(B * lout * Cin * taps + pad)
    hp.call("head_probe_tk_im2col", X.data_ptr(), Cin, lin, lout, taps, dil, relu, col.data_ptr(), B, probe.stream())
    torch.cuda.synchronize()
    return (col,)


def _col2im(dcol, Cin, lin, lout, taps, dil, mask, resid, mask_out, B, pad=7):
    dX = _nan(B * lin * Cin + pad)
    hp.call("head_probe_tk_col2im", dcol.data_ptr(), Cin, lin, lout, taps, dil, probe.ptr(mask), probe.ptr(resid),
            probe.ptr(mask_out), dX.data_ptr(), B, probe.stream())
    torch.cuda.synchronize()
    return (dX,)


# (Cin, lin, lout, taps, dil): conv_in, the four resize convs, the ResNet1D's conv1 at dilations 3 and 1 (padding
# reaches past both ends of the 21 positions), its taps-1 conv2; post and out share conv1's dilation-1 shape.
SHAPES = [(CODE, T, T, 3, 1), (WIDTH, T, 125, 3, 1), (WIDTH, 125, 90, 3, 1), (WIDTH, 90, 55, 3, 1),
          (WIDTH, 55, 21, 3, 1), (WIDTH, 21, 21, 3, 3), (WIDTH, 21, 21, 3, 1), (WIDTH, 21, 21, 1, 1)]
SHAPE_IDS = [f"C{c}-{a}to{b}-k{k}d{d}" for c, a, b, k, d in SHAPES]
# Not a product shape: an upsampling map, where one input position is read by several output positions, so the
# gather's multi-position sum runs.  The tokenizer only downsizes; this tests the kernel's contract.
UPSAMPLE = (64, 21, 55, 3, 1)


@pytest.mark.parametrize("shape", SHAPES + [UPSAMPLE], ids=SHAPE_IDS + ["contract-upsample-C64-21to55"])
@pytest.mark.parametrize("relu", [0, 1])
def test_im2col_exact(shape, relu):
    Cin, lin, lout, taps, dil = shape
    B = 2
    g = _gen("im2col", shape, relu)
    X = torch.randn(B * lin, Cin, device="cuda", generator=g)
    (col,) = _twice(lambda: _im2col(X, Cin, lin, lout, taps, dil, relu, B))
    n = B * lout * Cin * taps
    want = _im2col64(X.double().view(B, lin, Cin), lin, lout, taps, dil, relu)
    assert torch.equal(col[:n].view_as(want).double(), want)
    assert col[n:].isnan().all()
    # the column order and the cross-correlation direction: on integer data col @ W^T is F.conv1d exactly
    Xi = _ints((B * lin, Cin), g)
    Cout = 8
    W = _ints((Cout, Cin, taps), g)
    (col,) = _im2col(Xi, Cin, lin, lout, taps, dil, relu, B)
    got = col[:n].view(B * lout, Cin * taps).double() @ W.double().view(Cout, Cin * taps).t()
    xr = Xi.view(B, lin, Cin).transpose(1, 2)[:, :, _src(lin, lout)].double()
    want = F.conv1d(torch.relu(xr) if relu else xr, W.double(), padding=dil * (taps // 2), dilation=dil)
    assert torch.equal(got.view(B, lout, Cout), want.transpose(1, 2))


@pytest.mark.parametrize("lin,lout", [(T, T)] + list(zip((T,) + UPS[:-1], UPS)) + [(JOINTS, 55)])
def test_seq_map_matches_aten_on_the_gpu(lin, lout):
    """The map the kernels use is ATen's on fp32 input on the device as well (tests/test_token_head_probe_host.py
    checks every size on the host).  What ATen's fp64 map and its backward's per-input counts do is only printed:
    on an H100 with torch 2.11 the forward maps agree at every pair here, and the backward's counts differ at
    125 -> 90 (inputs 74 and 75) in both dtypes."""
    src, lo = hp.tk_seq_map(lin, lout)
    assert src == _src(lin, lout).tolist()
    for dt in (torch.float32, torch.float64):
        x = torch.arange(lin, dtype=dt, device="cuda").view(1, 1, lin).requires_grad_(True)
        y = F.interpolate(x, size=lout, mode="nearest")
        (gx,) = torch.autograd.grad(y.sum(), x)
        fwd = [(p, int(v)) for p, v in enumerate(y.view(lout).tolist()) if int(v) != src[p]]
        bwd = [(s, int(c)) for s, c in enumerate(gx.view(lin).tolist()) if int(c) != lo[s + 1] - lo[s]]
        print(f"[resize] {lin} -> {lout} {dt}: ATen's forward map differs at {fwd[:4]}, its backward's counts at "
              f"{bwd[:4]}")


# The combinations tk_backward passes: none (conv_in, post, out); mask (the resize convs: Y_u; ResNet conv2: hh);
# mask + resid (ResNet block 1's conv1: x1, the block's skip gradient); resid + mask_out (block 0's conv1: the skip
# gradient, then Y4's ReLU).
COMBOS = {"none": (False, False, False), "mask": (True, False, False), "mask+resid": (True, True, False),
          "resid+mask_out": (False, True, True)}


def _masks(B, lin, Cin, combo, g):
    use_m, use_r, use_mo = COMBOS[combo]
    mk = lambda: torch.randn(B * lin, Cin, device="cuda", generator=g)
    mask, resid, mask_out = (mk() if use_m else None), (_ints((B * lin, Cin), g) if use_r else None), \
        (mk() if use_mo else None)
    for m in (mask, mask_out):          # NaN counts as "not > 0", and so does -0
        if m is not None:
            m.view(-1)[::97] = float("nan")
            m.view(-1)[5::101] = -0.0
    return mask, resid, mask_out


def _apply_masks64(v, mask, resid, mask_out):
    if mask is not None:
        v = torch.where(mask.double() > 0, v, torch.zeros_like(v))
    if resid is not None:
        v = v + resid.double()
    if mask_out is not None:
        v = torch.where(mask_out.double() > 0, v, torch.zeros_like(v))
    return v


@pytest.mark.parametrize("shape", SHAPES + [UPSAMPLE], ids=SHAPE_IDS + ["contract-upsample-C64-21to55"])
@pytest.mark.parametrize("combo", list(COMBOS))
def test_col2im(shape, combo):
    """Exact on integer dcol (every partial sum an integer); exact zeros at the positions no output reads, before resid;
    within a chain bound on random dcol."""
    Cin, lin, lout, taps, dil = shape
    B = 2
    g = _gen("col2im", shape, combo)
    mask, resid, mask_out = _masks(B, lin, Cin, combo, g)
    dcol = _ints((B * lout, Cin * taps), g)
    (dX,) = _twice(lambda: _col2im(dcol, Cin, lin, lout, taps, dil, mask, resid, mask_out, B))
    n = B * lin * Cin
    raw = _col2im64(dcol, B, Cin, lin, lout, taps, dil)
    want = _apply_masks64(raw, mask, resid, mask_out)
    assert torch.equal(dX[:n].view_as(want).double(), want)
    assert dX[n:].isnan().all()
    src, lo = hp.tk_seq_map(lin, lout)
    unread = [s for s in range(lin) if lo[s] == lo[s + 1]]
    assert (len(unread) == lin - lout) if lout < lin else not unread
    if unread:                          # the gather reads nothing there: an exact 0 before the masks and resid
        rows = torch.tensor([b * lin + s for b in range(B) for s in unread], device="cuda")
        assert torch.equal(raw[rows], torch.zeros_like(raw[rows]))
        got = dX[:n].view(B * lin, Cin)[rows]
        if resid is None:
            assert torch.equal(got, torch.zeros_like(got)) and not got.signbit().any()
        else:
            assert torch.equal(got.double(), _apply_masks64(torch.zeros_like(raw[rows]), None if mask is None else
                                                            mask[rows], resid[rows],
                                                            None if mask_out is None else mask_out[rows]))
    if lout > lin:
        assert max(lo[s + 1] - lo[s] for s in range(lin)) >= 3      # several positions per input: the sum runs

    # random dcol: each input element sums at most P * taps terms (P positions read it) in a fixed order:
    # gamma_(P taps) of the sum of |terms|, then + resid: u of the result
    dcolr = torch.randn(B * lout, Cin * taps, device="cuda", generator=g)
    (dX,) = _twice(lambda: _col2im(dcolr, Cin, lin, lout, taps, dil, mask, resid, mask_out, B))
    per = max(lo[s + 1] - lo[s] for s in range(lin))
    ref = _apply_masks64(_col2im64(dcolr, B, Cin, lin, lout, taps, dil), mask, resid, mask_out)
    mag = _apply_masks64(_col2im64(dcolr.abs(), B, Cin, lin, lout, taps, dil), mask, None, mask_out)
    bound = gamma(max(per * taps, 1)) * mag + U32 * ref.abs() + 2.0 ** -60
    assert_within(f"col2im {SHAPE_IDS[SHAPES.index(shape)] if shape in SHAPES else 'upsample'} {combo}",
                  dX[:n].view_as(ref), ref, bound)
    if taps > 1:                        # teeth: the reference without tap 0
        cut = dcolr.view(B * lout, Cin, taps).clone()
        cut[..., 0] = 0
        assert _rejects(dX[:n].view_as(ref), _apply_masks64(_col2im64(cut.view_as(dcolr), B, Cin, lin, lout, taps,
                                                                      dil), mask, resid, mask_out), bound)


# ------------------------------------------------------------------------------------------------ conv composites
def _planner(M, N, K, batch=1, partial=True):
    """hl_split_count restated (head_train.cuh): 1 without a split buffer or at >= 132 tiles, else
    min(264 / tiles, K / 64), at least 1."""
    tiles = ((N + 63) // 64) * ((M + 63) // 64) * batch
    if not partial or tiles >= 132:
        return 1
    return max(1, min(264 // tiles, K // 64))


def _gemm_rounds(M, N, K):
    """Roundings per product of one hl_gemm output: kper + splits (the reduce), as in head_train_probe.py."""
    s = _planner(M, N, K)
    return (K + s - 1) // s + (s if s > 1 else 0)


# (name, Cin, Cout, lin, lout, taps, dil, relu, accumulate, backward mask combo or None): the tokenizer's conv calls
CONVS = [("conv_in", CODE, WIDTH, T, T, 3, 1, 0, False, "none")] + \
    [(f"up{u}", WIDTH, WIDTH, ([T] + list(UPS))[u], UPS[u], 3, 1, 1, False, "mask") for u in range(4)] + \
    [("res0.conv1", WIDTH, WIDTH, JOINTS, JOINTS, 3, 3, 1, False, "resid+mask_out"),
     ("res0.conv2", WIDTH, WIDTH, JOINTS, JOINTS, 1, 1, 1, True, "mask"),
     ("res1.conv1", WIDTH, WIDTH, JOINTS, JOINTS, 3, 1, 1, False, "mask+resid"),
     ("res1.conv2", WIDTH, WIDTH, JOINTS, JOINTS, 1, 1, 1, True, "mask"),
     ("post", WIDTH, WIDTH, JOINTS, JOINTS, 3, 1, 0, False, "none"),
     ("out", WIDTH, 6, JOINTS, JOINTS, 3, 1, 0, False, None)]      # its backward is the batched kDyW site below


@pytest.mark.parametrize("B", [1, 5])
@pytest.mark.parametrize("conv", CONVS, ids=[c[0] for c in CONVS])
def test_conv_forward_and_backward(conv, B, split_buf):
    name, Cin, Cout, lin, lout, taps, dil, relu, acc, combo = conv
    g = _gen("conv", name, B)
    K, rows = Cin * taps, B * lout
    X = torch.randn(B * lin, Cin, device="cuda", generator=g)
    W = torch.randn(Cout, Cin, taps, device="cuda", generator=g) / K ** 0.5
    bias = torch.randn(Cout, device="cuda", generator=g)
    Y0 = torch.randn(rows, Cout, device="cuda", generator=g) if acc else None
    col = torch.empty(rows * K, device="cuda")

    def fwd():
        Y = Y0.clone() if acc else _nan(rows, Cout)
        hp.call("head_probe_tk_conv", X.data_ptr(), Cin, lin, lout, taps, dil, relu, W.data_ptr(), bias.data_ptr(),
                Cout, Y.data_ptr(), int(acc), B, col.data_ptr(), split_buf.data_ptr(), probe.stream())
        torch.cuda.synchronize()
        return (Y,)

    (Y,) = _twice(fwd)
    xr = X.view(B, lin, Cin).transpose(1, 2)[:, :, _src(lin, lout)].double()
    xr = torch.relu(xr) if relu else xr
    ref = F.conv1d(xr, W.double(), bias.double(), padding=dil * (taps // 2), dilation=dil).transpose(1, 2)
    mag = F.conv1d(xr.abs(), W.double().abs(), bias.double().abs(), padding=dil * (taps // 2),
                   dilation=dil).transpose(1, 2)
    ref, mag = ref.reshape(rows, Cout), mag.reshape(rows, Cout)
    if acc:
        ref = ref + Y0.double()
    # the GEMM's chain (kper + splits), + bias, + C0: see head_train_probe.py
    bound = gamma(_gemm_rounds(rows, Cout, K) + 4) * mag + (U32 * Y0.double().abs() if acc else 0) + 2.0 ** -60
    assert_within(f"tk_conv {name} B={B}", Y, ref, bound)
    assert _rejects(Y, ref - bias.double(), bound), "bound accepts a dropped bias"
    if combo is None:
        return

    dY = torch.randn(rows, Cout, device="cuda", generator=g)
    mask, resid, mask_out = _masks(B, lin, Cin, combo, g)
    if resid is not None:
        resid = torch.randn(B * lin, Cin, device="cuda", generator=g)
    dcol = torch.empty(rows * K, device="cuda")

    def bwd():
        dX = _nan(B * lin * Cin + 3)
        hp.call("head_probe_tk_conv_bwd", dY.data_ptr(), Cout, W.data_ptr(), Cin, lin, lout, taps, dil,
                probe.ptr(mask), probe.ptr(resid), probe.ptr(mask_out), dX.data_ptr(), B, dcol.data_ptr(),
                split_buf.data_ptr(), probe.stream())
        torch.cuda.synchronize()
        return (dX,)

    (dX,) = _twice(bwd)
    n = B * lin * Cin
    assert dX[n:].isnan().all()
    # fp64 autograd of conv1d(resize(x)) (no ReLU: the engine's masks carry it), then the masks and resid
    x64 = torch.zeros(B, Cin, lin, dtype=torch.float64, device="cuda", requires_grad=True)
    y64 = F.conv1d(x64[:, :, _src(lin, lout)], W.double(), padding=dil * (taps // 2), dilation=dil)
    (gx,) = torch.autograd.grad((y64 * dY.double().view(B, lout, Cout).transpose(1, 2)).sum(), x64, retain_graph=True)
    ref = _apply_masks64(gx.transpose(1, 2).reshape(n // Cin, Cin), mask, resid, mask_out)
    # dcol = dY W: one hl_gemm output per (row, c, j), then the gather's P taps terms: every product passes through
    # at most gemm_rounds + P taps roundings; + resid: u of the result
    src, lo = hp.tk_seq_map(lin, lout)
    per = max(lo[s + 1] - lo[s] for s in range(lin))
    mag_col = dY.double().abs() @ W.double().abs().view(Cout, K)
    mag = _apply_masks64(_col2im64(mag_col, B, Cin, lin, lout, taps, dil), mask, None, mask_out)
    bound = gamma(_gemm_rounds(rows, K, Cout) + per * taps) * mag + U32 * ref.abs() + 2.0 ** -60
    got = dX[:n].view_as(ref)
    assert_within(f"tk_conv_bwd {name} B={B}", got, ref, bound)
    cut = dY.clone()                    # teeth: one output position's gradient left out
    cut[rows // 2] = 0
    (gx,) = torch.autograd.grad((y64 * cut.double().view(B, lout, Cout).transpose(1, 2)).sum(), x64)
    assert _rejects(got, _apply_masks64(gx.transpose(1, 2).reshape(n // Cin, Cin), mask, resid, mask_out), bound)


# ------------------------------------------------------------------------------------------------ LayerNorm
def _ln_rows(rows, N, g):
    """Row r is kind r % 3: mean 0 / std 1, mean 1000 / std 1, or the constant 0.7 (variance 0: rstd = eps^-1/2)."""
    x = torch.randn(rows, N, device="cuda", generator=g)
    x[1::3] += 1000
    x[2::3] = 0.7
    return x


def _ln_fwd_bounds(x, gw, bw, n):
    """fp64 mean, rstd, pre-ReLU y and their bounds.  The sums: n chained roundings (n below per width), then the
    fp32 1/N (exact for 64; for 10240 its own rounding and the product's: 2 u more, inside gamma_(n+2)).  As in
    tests/test_gpu_head_train_kernels.py: dmu = gamma_(n+2) mean |x|; var: a product per term and the chain,
    d = x - mean's rounding twice: gamma_(n+6) var plus dmu^2; rstd = rsqrtf(var + eps): 2 ulp (4 u), the sum's u and
    half var's relative error; y = d rs g + b: three roundings (ReLU does not increase an error).  Second-order
    terms are folded into 1.01."""
    xd, gd, bd = x.double(), gw.double(), bw.double()
    mu = xd.mean(1, keepdim=True)
    var = ((xd - mu) ** 2).mean(1, keepdim=True)
    rs = (var + EPS).rsqrt()
    y64 = (xd - mu) * rs * gd + bd
    dmu = gamma(n + 2) * xd.abs().mean(1, keepdim=True)
    drs = rs * (5 * U32 + 0.5 * (gamma(n + 6) * var + dmu ** 2) / (var + EPS))
    d = (xd - mu).abs()
    bound_y = 1.01 * (gd.abs() * (rs * (dmu + U32 * d) + d * drs) + 3 * U32 * (d * rs * gd.abs() + bd.abs())) + 2.0 ** -60
    return mu, rs, y64, dmu, drs, bound_y


def _ln_bwd_ref(x, gw, mean, rstd, dy, n):
    """fp64 dx from the kernel's own mean and rstd, and its bound: h 2 u; g dy u; m1 the n-chain and 1/N, gamma_(n+2)
    of mean |g dy|; m2 a product and h's 2 u more, gamma_(n+5) of mean |g dy h|; t = g dy - m1 - h m2: 3 u of the
    terms and h's 2 u on h m2; times rstd: u.  Returns (rstd t, bound without the accumulate term, pieces)."""
    xd, gd = x.double(), gw.double()
    m_, r_ = mean.double().unsqueeze(1), rstd.double().unsqueeze(1)
    h = (xd - m_) * r_
    gdy = dy.double() * gd
    m1, m2 = gdy.mean(1, keepdim=True), (gdy * h).mean(1, keepdim=True)
    t = gdy - m1 - h * m2
    S1, S2 = gdy.abs().mean(1, keepdim=True), (gdy * h).abs().mean(1, keepdim=True)
    inner = 2 * U32 * gdy.abs() + gamma(n + 2) * S1 + h.abs() * gamma(n + 5) * S2 + \
        4 * U32 * (gdy.abs() + m1.abs() + 2 * (h * m2).abs())
    return r_ * t, 1.01 * r_ * inner, (gdy, h, m2, r_)


N_WIDE = 10 * 4 + 5 + 8     # per thread 10 float4s of 4 additions each, a warp's 5 shuffles, 8 warp partials
N_64 = 1 + 5                # per lane two columns, 5 shuffles


@pytest.mark.parametrize("B", [1, 7, 161])
def test_layernorm_wide(B):
    g = _gen("lnwide", B)
    gw = 1 + 0.1 * torch.randn(MIX, device="cuda", generator=g)
    bw = 0.3 * torch.randn(MIX, device="cuda", generator=g)
    x = _ln_rows(B, MIX, g)

    def fwd():
        y, mean, rstd = _nan(B + 1, MIX), _nan(B + 1), _nan(B + 1)
        hp.call("head_probe_tk_ln_wide_fwd", x.data_ptr(), gw.data_ptr(), bw.data_ptr(), y.data_ptr(),
                mean.data_ptr(), rstd.data_ptr(), B, probe.stream())
        torch.cuda.synchronize()
        return y, mean, rstd

    y, mean, rstd = _twice(fwd)
    assert y[B].isnan().all() and mean[B].isnan() and rstd[B].isnan()
    y, mean, rstd = y[:B], mean[:B], rstd[:B]
    mu, rs, y64, dmu, drs, bound_y = _ln_fwd_bounds(x, gw, bw, N_WIDE)
    assert_within(f"ln10240 y B={B}", y, torch.relu(y64), bound_y)
    assert_within(f"ln10240 mean B={B}", mean, mu.squeeze(1), dmu.squeeze(1) + 2.0 ** -60)
    assert_within(f"ln10240 rstd B={B}", rstd, rs.squeeze(1), 1.01 * drs.squeeze(1))
    if B > 1:
        assert torch.allclose(rstd[2::3].double(), torch.full_like(rstd[2::3].double(), EPS ** -0.5), rtol=1e-6, atol=0)
    keep = torch.ones(MIX, dtype=torch.bool, device="cuda")
    keep[0] = False                     # teeth: the mean over all but one column, on the mean-0 rows
    mu_d = x.double()[:, keep].mean(1, keepdim=True)
    assert _rejects(y[0::3], torch.relu((x.double() - mu_d) * rs * gw.double() + bw.double())[0::3], bound_y[0::3])

    # backward: dy masked in place by [y > 0], dx overwritten
    dy0 = torch.randn(B, MIX, device="cuda", generator=g)

    def bwd():
        dy, dx = dy0.clone(), _nan(B + 1, MIX)
        hp.call("head_probe_tk_ln_wide_bwd", x.data_ptr(), gw.data_ptr(), mean.data_ptr(), rstd.data_ptr(),
                y.data_ptr(), dy.data_ptr(), dx.data_ptr(), B, probe.stream())
        torch.cuda.synchronize()
        return dy, dx

    dy, dx = _twice(bwd)
    assert dx[B].isnan().all()
    masked = torch.where(y > 0, dy0, torch.zeros_like(dy0))
    assert torch.equal(dy, masked) and torch.equal(dy.signbit(), masked.signbit())
    assert (y > 0).any() and (y <= 0).any()
    ref, bound, (gdy, h, m2, r_) = _ln_bwd_ref(x, gw, mean, rstd, masked, N_WIDE)
    bound = bound + U32 * ref.abs() + 2.0 ** -60
    assert_within(f"ln10240 dx B={B}", dx[:B], ref, bound)
    # teeth: without the xhat mean(g dy xhat) term
    assert _rejects(dx[:B], r_ * (gdy - gdy.mean(1, keepdim=True)), bound)


@pytest.mark.parametrize("rows", [1, 7, 9, 160 * 5])
@pytest.mark.parametrize("relu", [0, 1])
def test_layernorm_64(rows, relu):
    g = _gen("ln64", rows, relu)
    gw = 1 + 0.1 * torch.randn(HID, device="cuda", generator=g)
    bw = 0.3 * torch.randn(HID, device="cuda", generator=g)
    x = _ln_rows(rows, HID, g)

    def fwd():
        y, mean, rstd = _nan(rows + 1, HID), _nan(rows + 1), _nan(rows + 1)
        hp.call("head_probe_tk_ln64_fwd", x.data_ptr(), gw.data_ptr(), bw.data_ptr(), y.data_ptr(), mean.data_ptr(),
                rstd.data_ptr(), rows, relu, probe.stream())
        torch.cuda.synchronize()
        return y, mean, rstd

    y, mean, rstd = _twice(fwd)
    assert y[rows].isnan().all() and mean[rows].isnan() and rstd[rows].isnan()
    y, mean, rstd = y[:rows], mean[:rows], rstd[:rows]
    mu, rs, y64, dmu, drs, bound_y = _ln_fwd_bounds(x, gw, bw, N_64)
    act = torch.relu if relu else (lambda v: v)
    assert_within(f"ln64 y rows={rows} relu={relu}", y, act(y64), bound_y)
    assert_within(f"ln64 mean rows={rows}", mean, mu.squeeze(1), dmu.squeeze(1) + 2.0 ** -60)
    assert_within(f"ln64 rstd rows={rows}", rstd, rs.squeeze(1), 1.01 * drs.squeeze(1))
    if rows > 2:
        assert torch.allclose(rstd[2::3].double(), torch.full_like(rstd[2::3].double(), EPS ** -0.5), rtol=1e-6, atol=0)
    keep = torch.ones(HID, dtype=torch.bool, device="cuda")
    keep[0] = False
    mu_d = x.double()[:, keep].mean(1, keepdim=True)
    assert _rejects(y[0::3], act((x.double() - mu_d) * rs * gw.double() + bw.double())[0::3], bound_y[0::3])

    dy0 = torch.randn(rows, HID, device="cuda", generator=g)
    dx0 = torch.randn(rows, HID, device="cuda", generator=g)
    # the engine's two uses: mixer_norm_layer (y = its ReLU output, dx overwritten) and the mixer layers' LayerNorms
    # (no ReLU: y null, dx accumulated); and the other two combinations of the flags
    for with_y, acc in ((True, 0), (False, 1), (True, 1), (False, 0)):
        yy = y if with_y else None

        def bwd():
            dy, dx = dy0.clone(), (torch.cat([dx0, _nan(1, HID)]) if acc else _nan(rows + 1, HID))
            hp.call("head_probe_tk_ln64_bwd", x.data_ptr(), gw.data_ptr(), mean.data_ptr(), rstd.data_ptr(),
                    probe.ptr(yy), dy.data_ptr(), dx.data_ptr(), rows, acc, probe.stream())
            torch.cuda.synchronize()
            return dy, dx

        dy, dx = _twice(bwd)
        assert dx[rows].isnan().all()
        masked = torch.where(y > 0, dy0, torch.zeros_like(dy0)) if with_y else dy0
        assert torch.equal(dy, masked) and torch.equal(dy.signbit(), masked.signbit())
        ref, bound, (gdy, h, m2, r_) = _ln_bwd_ref(x, gw, mean, rstd, masked, N_64)
        if acc:                         # + dx0: one more rounding
            ref = ref + dx0.double()
            bound = bound + U32 * (dx0.double().abs() + (ref - dx0.double()).abs())
        bound = bound + U32 * ref.abs() + 2.0 ** -60
        tag = f"ln64 dx rows={rows} y={with_y} acc={acc}"
        assert_within(tag, dx[:rows], ref, bound)
        base = dx0.double() if acc else 0
        assert _rejects(dx[:rows], base + r_ * (gdy - gdy.mean(1, keepdim=True)), bound), tag + " teeth"


# ------------------------------------------------------------------------------------------------ softmax
def _softmax_rows(scale, g, rows=24):
    """rows x 2048 logits at `scale`: random rows; a row whose maximum is the last element of the last lane's last
    float4 (element 2047); a row of ties (all equal: P = 1/2048 exactly); a row with four tied maxima."""
    x = scale * torch.randn(rows, CLS, device="cuda", generator=g)
    x[1, 2047] = x[1].max() + scale
    x[2] = 0.375 * scale
    x[3, [0, 511, 1024, 2047]] = x[3].max() + 1
    return x


@pytest.mark.parametrize("scale", [1.0, 20.0, 80.0])
def test_softmax_forward_and_backward(scale):
    g = _gen("softmax", scale)
    rows = 24
    x = _softmax_rows(scale, g, rows)

    def fwd():
        p = torch.cat([x, _nan(1, CLS)])
        hp.call("head_probe_tk_softmax_fwd", p.data_ptr(), rows, probe.stream())
        torch.cuda.synchronize()
        return (p,)

    (P,) = _twice(fwd)
    assert P[rows].isnan().all()
    P = P[:rows]
    xd = x.double()
    m = xd.amax(1, keepdim=True)
    P64 = torch.softmax(xd, 1)
    # P_i = expf(x_i - m) / sum: x_i - m rounds (relative u |x_i - m| on the exponential), expf 2 ulp (4 u); the sum
    # is 64 additions per lane and 5 shuffles of positive terms, gamma_69, plus its terms' own errors (their
    # P-weighted mean); 1 / sum and the product: 2 u.  Where expf underflows the result is subnormal or zero: an
    # absolute floor (P <= 1 and 1 / sum <= 1, as the maximum's term is exactly 1).
    rel_i = 4 * U32 + U32 * (xd - m).abs()
    rel = rel_i + (P64 * rel_i).sum(1, keepdim=True) + gamma(69) + 2 * U32
    bound = 1.01 * rel * P64 + TINY
    assert_within(f"softmax P scale={scale}", P, P64, bound)
    assert torch.equal(P[2], torch.full_like(P[2], 1 / 2048))
    assert int(P[1].argmax()) == 2047
    if scale == 80.0:
        assert (P == 0).any() or (P < TINY).any(), "expf did not underflow"
    cut = torch.exp(xd - m)             # teeth: one term out of the normaliser
    cut_sum = cut.sum(1, keepdim=True) - cut[:, 1000:1001]
    assert _rejects(P, cut / cut_sum, bound)

    # backward from the kernel's own P: d_i <- P_i (d_i - s), s = sum P d: a 64-term fmaf chain per lane and 5
    # shuffles, gamma_70 of sum |P d|; d_i - s and the product: 2 u of |d_i - s|.  Where one P is ~1, d_i - s cancels
    # for it; the bound is absolute in sum |P d| there, so it holds.
    d0 = torch.randn(rows, CLS, device="cuda", generator=g)

    def bwd():
        d = torch.cat([d0, _nan(1, CLS)])
        hp.call("head_probe_tk_softmax_bwd", P.data_ptr(), d.data_ptr(), rows, probe.stream())
        torch.cuda.synchronize()
        return (d,)

    (dP,) = _twice(bwd)
    assert dP[rows].isnan().all()
    Pd, dd = P.double(), d0.double()
    s = (Pd * dd).sum(1, keepdim=True)
    ref = Pd * (dd - s)
    bound = Pd * (gamma(70) * (Pd * dd).abs().sum(1, keepdim=True) + 2 * U32 * (dd - s).abs()) + TINY
    assert_within(f"softmax dP scale={scale}", dP[:rows], ref, bound)
    if scale >= 20:
        assert (Pd.amax(1) > 0.999).any(), "no row with one P ~ 1"
    j = (Pd * dd).abs().argmax(1, keepdim=True)     # teeth: s without its largest term
    s_cut = s - (Pd * dd).gather(1, j)
    assert _rejects(dP[:rows], Pd * (dd - s_cut), bound)


# ------------------------------------------------------------------------------------------------ column sums
COLSUM_ROWS = [1, 159, 160, 161, 330, 160 * 130]
COLSUM_N = [64, 160, 256, 2048, 10240]


def test_colsum_chunk_counts():
    """The row counts below run over 1, 1, 1, 2, 3 and 130 partials."""
    chunks = [hp.lib().head_probe_tk_colsum_chunks(r) for r in COLSUM_ROWS]
    assert chunks == [1, 1, 1, 2, 3, 130]


def _colsum(dy, rows, N, x=None, mean=None, rstd=None, pad=5):
    chunks = (rows + COL_ROWS - 1) // COL_ROWS
    out = _nan(N + pad)
    og = _nan(N + pad) if x is not None else None
    part, part_g = _nan(chunks * N + pad), _nan(chunks * N + pad)
    hp.call("head_probe_tk_colsum", dy.data_ptr(), N, rows, N, out.data_ptr(), probe.ptr(x), probe.ptr(mean),
            probe.ptr(rstd), probe.ptr(og), part.data_ptr(), part_g.data_ptr(), probe.stream())
    torch.cuda.synchronize()
    return (out, part) + ((og, part_g) if x is not None else ())


@pytest.mark.parametrize("N", COLSUM_N)
@pytest.mark.parametrize("rows", COLSUM_ROWS)
def test_colsum(rows, N):
    g = _gen("colsum", rows, N)
    chunks = (rows + COL_ROWS - 1) // COL_ROWS
    # integer dy: every partial and the total is an integer below 2^24, so both stages are exact
    dy = _ints((rows, N), g, -50, 51)
    out, part = _twice(lambda: _colsum(dy, rows, N))
    pad_rows = chunks * COL_ROWS - rows
    per_chunk = F.pad(dy.double(), (0, 0, 0, pad_rows)).view(chunks, COL_ROWS, N).sum(1)
    assert torch.equal(part[:chunks * N].view(chunks, N).double(), per_chunk)
    assert torch.equal(out[:N].double(), dy.double().sum(0))
    assert out[N:].isnan().all() and part[chunks * N:].isnan().all()
    del dy

    # random: each partial a chain of at most 160 terms, then the chunk sum: gamma_(160 + chunks) of sum |dy|.  The
    # LayerNorm-weight sums add a subtraction and two products per term (one may fuse): gamma_(163 + chunks).
    dyr = torch.randn(rows, N, device="cuda", generator=g)
    x = 3 + 2 * torch.randn(rows, N, device="cuda", generator=g)
    mean = 3 + 0.1 * torch.randn(rows, device="cuda", generator=g)
    rstd = 0.5 + torch.rand(rows, device="cuda", generator=g)
    out, part, og, part_g = _twice(lambda: _colsum(dyr, rows, N, x, mean, rstd))
    assert og[N:].isnan().all() and part_g[chunks * N:].isnan().all()
    d = dyr.double()
    dxh = d * ((x.double() - mean.double()[:, None]) * rstd.double()[:, None])
    del x
    n = min(rows, COL_ROWS) + (chunks if chunks > 1 else 0)
    bound = gamma(n) * d.abs().sum(0) + 2.0 ** -60
    bound_g = gamma(n + 3) * dxh.abs().sum(0) + 2.0 ** -60
    assert_within(f"tk colsum rows={rows} N={N}", out[:N], d.sum(0), bound)
    assert_within(f"tk colsum xhat rows={rows} N={N}", og[:N], dxh.sum(0), bound_g)
    # teeth: without the last partial's rows (one chunk: without the first row)
    cut = slice(0, (chunks - 1) * COL_ROWS) if chunks > 1 else slice(1, rows)
    if rows > 1:
        assert _rejects(og[:N], dxh[cut].sum(0), bound_g)
        assert _rejects(out[:N], d[cut].sum(0), bound)


# ------------------------------------------------------------------------------------------------ transpose, ReLU copy
@pytest.mark.parametrize("R,C", [(160, 64), (64, 160), (33, 65)])
@pytest.mark.parametrize("add", [False, True])
def test_transpose_exact(R, C, add):
    """Copies, and with add one fp32 addition: equal to torch fp32 bit for bit."""
    B = 3
    g = _gen("transpose", R, C, add)
    x = torch.randn(B, R, C, device="cuda", generator=g)
    a = torch.randn(B, C, R, device="cuda", generator=g) if add else None

    def run():
        out = _nan(B * C * R + 11)
        hp.call("head_probe_tk_transpose", x.data_ptr(), R, C, probe.ptr(a), out.data_ptr(), B, probe.stream())
        torch.cuda.synchronize()
        return (out,)

    (out,) = _twice(run)
    want = x.transpose(1, 2) + (a if add else 0)
    assert torch.equal(out[:B * C * R].view(B, C, R), want)
    assert out[B * C * R:].isnan().all()


@pytest.mark.parametrize("n", [1, 255, 256, 21 * 512 * 5 + 3])
def test_relu_copy_exact(n):
    g = _gen("relu", n)
    x = torch.randn(n, device="cuda", generator=g)
    x[::7] = -0.0

    def run():
        out = _nan(n + 9)
        hp.call("head_probe_tk_relu_copy", x.data_ptr(), out.data_ptr(), n, probe.stream())
        torch.cuda.synchronize()
        return (out,)

    (out,) = _twice(run)
    assert torch.equal(out[:n], torch.where(x > 0, x, torch.zeros_like(x)))
    assert out[n:].isnan().all()


# ------------------------------------------------------------------------------------------------ hl_gemm call sites
def _tk_dw(name, rows, N, K, splits, **kw):
    """tk_linear_dw: dW (N x K) = dy^T (rows x N) x (rows x K), with the split buffer."""
    return _linear_dw(name, rows, N, K, splits=splits, **kw)


def _out_conv_dcol(B):
    """tk_backward's batched output-conv backward: dcol[b] (21 x 1536) = dY[b] (21 x 6) W (6 x 1536), with dY the body
    columns of dread: A at dread + 6, rows 6 apart, images 160 apart."""
    return Site(f"out conv dcol B={B}", "dyw", JOINTS, 3 * WIDTH, 6, B, (READ_LD, 6, 1), (0, 3 * WIDTH, 1),
                (JOINTS * 3 * WIDTH, 3 * WIDTH, 1), 1, a_off=6)


# Split counts from hl_split_count (restated in _planner: min(264 / tiles, K / 64) with a split buffer below 132
# tiles), written out so the table provably covers (tests/test_token_head_probe_host.py checks these claims):
#   empty trailing splits: mixer_norm dW at B = 106 (264 splits, kper 65: 3 start past K) and 161 (1), the token MLP
#   dW at B = 106; 264 splits on one 64 x 64 tile, exactly kSplitFloats of partials;
#   unaligned kper: soft lookup B = 1 (22 / 94), class_pred dW B = 5 (8 / 100), conv dcol B = 5 (5 / 103), conv_in
#   B = 1 (11 / 70), class_pred dx B = 5 (20 / 103);
#   gelu_out / dgelu after the reduce (token MLP, B = 5: 2 splits) and direct (B = 161: 161 tiles);
#   accumulate after the reduce (dP with grad_cls_probs at B = 1, channel MLP 2 at B = 5, ResNet conv2 at B = 1) and
#   direct (dP at B = 5);
#   the batched output-conv backward; mixer_trans forward (>= 132 tiles, direct) and its input gradient with
#   accumulate (16 splits at B = 5, 2 at B = 330).
SITES = [
    _linear_dx("soft lookup Z B=1", T, CLS, CODE, 22),                                    # kper 94
    _linear_dx("soft lookup Z B=5", 5 * T, CLS, CODE, 5),
    _linear("dP += dZ cb^T B=1", T, CLS, CODE, 2, accumulate=True),                      # accumulate, reduced
    _linear("dP += dZ cb^T B=5", 5 * T, CLS, CODE, 1, accumulate=True),                  # accumulate, direct
    _linear("dP = dZ cb^T B=5", 5 * T, CLS, CODE, 1),
    _linear("class_pred B=5", 5 * T, CLS, HID, 1, bias=True),                             # K = 64
    _tk_dw("class_pred dW B=5", 5 * T, CLS, HID, 8),                                      # kper 100
    _tk_dw("class_pred dW B=1", T, CLS, HID, 2),
    _linear_dx("class_pred dx B=5", 5 * T, CLS, HID, 20),                                 # kper 103
    _linear("mixer_norm B=5", 5 * T, HID, HID, 1, bias=True),
    _tk_dw("mixer_norm dW B=5", 5 * T, HID, HID, 12),
    _tk_dw("mixer_norm dW B=106", 106 * T, HID, HID, 264),                                # 3 empty, one tile
    _tk_dw("mixer_norm dW B=161", 161 * T, HID, HID, 264),                                # 1 empty
    _linear("token MLP1 B=5", 5 * HID, HID, T, 2, bias=True, gelu_out=True),              # gelu_out, reduced
    _linear("token MLP1 B=161", 161 * HID, HID, T, 1, bias=True, gelu_out=True),          # gelu_out, direct
    _linear("token MLP2 B=5", 5 * HID, T, HID, 1, bias=True),
    _linear_dx("token MLP2 dx B=5", 5 * HID, T, HID, 2, dgelu=True),                      # dgelu, reduced
    _linear_dx("token MLP2 dx B=161", 161 * HID, T, HID, 1, dgelu=True),                  # dgelu, direct
    _linear_dx("token MLP1 dx B=5", 5 * HID, HID, T, 1),
    _tk_dw("token MLP2 dW B=5", 5 * HID, T, HID, 5),
    _tk_dw("token MLP2 dW B=106", 106 * HID, T, HID, 88),                                 # 1 empty
    _tk_dw("token MLP1 dW B=106", 106 * HID, HID, T, 88),                                 # 1 empty
    _linear("channel MLP1 B=5", 5 * T, CODE, HID, 1, bias=True, gelu_out=True),
    _linear("channel MLP2 B=5", 5 * T, HID, CODE, 4, bias=True, accumulate=True),         # accumulate, reduced
    _linear("channel MLP2 B=161", 161 * T, HID, CODE, 1, bias=True, accumulate=True),     # accumulate, direct
    _linear_dx("channel MLP2 dx B=5", 5 * T, HID, CODE, 1, dgelu=True),
    _tk_dw("channel MLP2 dW B=5", 5 * T, HID, CODE, 12),
    _tk_dw("channel MLP1 dW B=5", 5 * T, CODE, HID, 12),
    _linear_dx("channel MLP1 dx B=5", 5 * T, CODE, HID, 4),
    _linear("mixer_trans B=5", 5, MIX, 1024, 1, bias=True),                               # 160 tiles: direct
    _linear_dx("mixer_trans dx B=5", 5, MIX, 1024, 16, accumulate=True),
    _linear_dx("mixer_trans dx B=330", 330, MIX, 1024, 2, accumulate=True),
    _linear_dw("mixer_trans dW B=5", 5, MIX, 1024),                                       # no split buffer
    _linear("decpose_grot B=5", 5, 6, 1024, 16, ldy=READ_LD, bias=True, y_extent=5 * READ_LD),
    _linear("conv_in B=1", T, WIDTH, 3 * CODE, 11, bias=True),                            # kper 70
    _linear("up0 conv B=5", 5 * 125, WIDTH, 3 * WIDTH, 3, bias=True),
    _linear("up3 conv B=1", JOINTS, WIDTH, 3 * WIDTH, 24, bias=True),
    _linear("res conv2 B=1", JOINTS, WIDTH, WIDTH, 8, bias=True, accumulate=True),        # accumulate, reduced
    _linear("out conv B=5", 5 * JOINTS, 6, 3 * WIDTH, 24, bias=True),
    _linear_dx("conv dcol 21 B=5", 5 * JOINTS, WIDTH, 3 * WIDTH, 5),                      # kper 103
    _linear_dx("conv dcol 21 B=1", JOINTS, WIDTH, 3 * WIDTH, 8),
    _linear_dx("conv_in dcol B=1", T, WIDTH, 3 * CODE, 7),
    _linear_dx("up0 dcol B=5", 5 * 125, WIDTH, 3 * WIDTH, 1),
    _out_conv_dcol(1),
    _out_conv_dcol(5),
]


@pytest.fixture(scope="module")
def split_buf(cuda_dev):
    n = hp.lib().head_probe_hl_split_floats()
    assert n == 264 * 64 * 64
    return torch.empty(n, device=cuda_dev)


@pytest.mark.parametrize("site", SITES, ids=[s.name for s in SITES])
def test_hl_gemm_integer_exact(site, split_buf):
    hp.check_site_integer_exact(site, split_buf)


@pytest.mark.parametrize("site", SITES, ids=[s.name for s in SITES])
def test_hl_gemm_random_within_bound(site, split_buf):
    hp.check_site_within_bound(site, split_buf)


def test_empty_splits_write_zero_partials(split_buf):
    """mixer_norm dW at B = 106: the last three of 264 splits start past K.  Their partials are zeros, not stale
    buffer contents: the split buffer is filled with NaN first, and the integer result must still be exact."""
    site = next(s for s in SITES if s.name == "mixer_norm dW B=106")
    assert site.empty_splits == 3
    split_buf.fill_(float("nan"))
    hp.check_site_integer_exact(site, split_buf)
    part = split_buf.view(264, 64, 64)
    assert torch.equal(part[261:], torch.zeros_like(part[261:]))
    assert part.isfinite().all()        # 264 splits x one tile fill the buffer exactly


# ------------------------------------------------------------------------------------------------ the whole head
# Helpers and bound as in tests/test_gpu_token_head_train.py: per output and per parameter gradient,
# max |x - x64| <= max(4 x the fp32 torch restatement's own error, 1e-5 max |x64|), on the _clear_of_kinks weights,
# after the fp64 check that no ReLU input lies within 1e-6 (relative) of its kink.
def _cfg(depth=6, heads=8, mlp=1024):
    from tokenhmr_b200.config import tiny_config
    return dataclasses.replace(tiny_config(vit_depth=2), dec_depth=depth, dec_heads=heads, dec_mlp_dim=mlp)


def _check_head(cfg, sd, B, seed, dev):
    import test_gpu_token_head_train as TH
    from tokenhmr_b200.heads import TokenHead
    sd = TH._clear_of_kinks(sd)
    head = TokenHead(cfg, sd, dev)
    feats = TH._feats(cfg, B, seed, dev)
    assert TH._kink_margin(sd, feats, cfg) > 1e-6
    up = TH._upstream(cfg, B, seed + 1, dev)
    got, outs = TH._run(head, feats, up)
    l64, r64 = TH._restated(sd, feats, cfg, torch.float64)
    g64 = TH._ref_grads(l64, r64, up)
    r64 = {k: v.detach() for k, v in r64.items()}
    del l64
    l32, r32 = TH._restated(sd, feats, cfg, torch.float32)
    g32 = TH._ref_grads(l32, r32, up)
    r32 = {k: v.detach() for k, v in r32.items()}
    del l32
    worst_out = max(TH._within(outs[k], r64[k], r32[k], k) for k in outs)
    assert set(got) == set(g64)
    ratios = {k: TH._ratio(got[k], g64[k], g32[k]) for k in g64}
    over = {k: r for k, r in ratios.items() if r[0] > 1.0}
    worst = max(ratios.items(), key=lambda kv: kv[1][0])
    print(f"[head] depth={cfg.dec_depth} heads={cfg.dec_heads} mlp={cfg.dec_mlp_dim} B={B}: worst output error / "
          f"bound {worst_out:.2f}; worst gradient error / bound {worst[1][0]:.2f} ({worst[0]})")
    assert not over, over
    for l in range(cfg.dec_depth):
        assert not got[f"transformer.transformer.layers.{l}.0.fn.to_qkv.weight"][:2 * cfg.dec_inner].any()
    assert not got["transformer.to_token_embedding.weight"].any()


@pytest.fixture(scope="module")
def release_sd():
    from tokenhmr_b200 import synth
    return synth.make_state_dict(_cfg())


@pytest.mark.parametrize("scale", [1.0, 0.05])
@pytest.mark.parametrize("B", [161, 330])
def test_head_at_multi_partial_batches(release_sd, cuda_dev, B, scale):
    """B = 161 and 330: the 10240-wide column sums over 2 and 3 partials, mixer_norm dW with an empty trailing split
    (161), mixer_trans's input gradient at 2 splits (330), and the token MLP's gelu_out / dgelu epilogues direct."""
    import test_gpu_token_head_train as TH
    _check_head(_cfg(), TH._scaled(release_sd, scale), B, 100 + B, cuda_dev)
    torch.cuda.empty_cache()


@pytest.mark.parametrize("depth,heads,mlp", [(1, 1, 1), (2, 3, 200)])
def test_head_non_release_decoders(cuda_dev, depth, heads, mlp):
    """Other decoder shapes move every tail parameter's offset in tk_layout."""
    from tokenhmr_b200 import synth
    cfg = _cfg(depth, heads, mlp)
    _check_head(cfg, synth.make_state_dict(cfg), 5, 10 * depth + heads, cuda_dev)

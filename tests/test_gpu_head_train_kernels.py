"""The regression head's training kernels (csrc/head_train.cuh) one at a time, through their test-only probe
(tests/csrc/head_train_probe.cu), against torch fp64 on the fp32 values each kernel reads: the tiled fp32 GEMM in its
three orientations and every epilogue, on a table of call sites whose split counts the test asserts; the factorised
cross-attention forward and backward; LayerNorm forward and backward; the column sums; the token-0 kernel; and the
read-out backward with its degenerate Gram-Schmidt
inputs and null upstream gradients.  Then the whole head (heads.RegressionHead) at the batch sizes and decoder shapes
tests/test_gpu_head_train.py does not reach, and with each subset of upstream gradients.

Bounds are per element and derived in comments from each kernel's order of operations (probe.assert_within); integer
inputs make the GEMM, the column sums and the scores exact, and those are compared bit for bit.  Every output starts as
NaN, so an unwritten element fails, and pitch padding must still be NaN afterwards.  Every kernel runs twice and the
two results must be identical.  Each bound family also shows it has teeth: it rejects an fp64 reference with one term
taken out."""
import dataclasses
import zlib

import pytest
import torch
import torch.nn.functional as F

import head_train_probe as hp
import probe
from oracle import regression_oracle as R
from oracle import tokenhmr_oracle as O
from probe import U32, assert_within

pytestmark = pytest.mark.gpu

REG = "transformer_decoder"
E, C, T, D = 1024, 1280, 192, 64            # kRhDim, kRhCtx, kRhTokens, kRhDimHead
CHUNK, NCHUNK, READ_LD = 16, 12, 160        # kRhChunk, kRhChunks, kRhReadLd
EPS = 9.99999974737875e-06                  # kRhLnEps: the fp32 value of 1e-5
SCALE = 0.125                               # 1 / sqrt(64), exact


@pytest.fixture(autouse=True)
def _flags(cuda_dev, built_lib):
    yield
    assert hp.flags() == 0, "head-train probe device flags set"
    assert built_lib.thmr_check_device_flags() == 0, built_lib.thmr_last_error()


def _nan(*shape):
    return torch.full(shape, float("nan"), device="cuda")


def gamma(n: int) -> float:
    """gamma_n = n u / (1 - n u): the relative error bound of n chained fp32 roundings."""
    return n * U32 / (1 - n * U32)


def _rejects(got, ref, bound) -> bool:
    """True when some element of got lies outside bound of the (perturbed) reference."""
    err = (got.double() - ref.double()).abs()
    return bool((~(err <= torch.as_tensor(bound, device=err.device).double())).any())


def _twice(run):
    """Runs a launch twice; the two results must be bit-identical (no atomics, fixed reduction order)."""
    a = run()
    b = run()
    for x, y in zip(a, b):
        assert torch.equal(x.nan_to_num(1234.5), y.nan_to_num(1234.5)) and torch.equal(x.isnan(), y.isnan())
    return a


# ------------------------------------------------------------------------------------------------ hl_gemm
# C[z] = epilogue(alpha * sum_k A(m,k) B(k,n)).  Each output is a serial fmaf chain over its split's k range (at most
# kper = ceil(K / splits) terms), then, when split, the reduce kernel's `splits` additions in split order, so every
# product passes through at most kper + splits roundings: |acc - S| <= gamma_(kper+splits) sum_k |a||b| (= Tab).
# Then alpha (a power of two here: exact), + bias (1 rounding), * gelu'(dgelu) (1 rounding), + C0 (1 rounding): with
# G the fp64 gelu' (1 without dgelu) and eps_G the error of the fp32 gelu' itself,
#   |C - C64| <= gamma_(kper+splits+4) |G| (|alpha| Tab + |bias|) + eps_G (|alpha| Tab + |bias|) + u |C0|.
# gelu'(x) = 0.5 (1 + erff(x / sqrt 2)) + x phi(x) with expf: erff's 2 ulp and the argument's rounding (erf' <= 1.13)
# give u (2 + 0.8 |x|) on the first half; expf's 2 ulp, the rounding of -x^2/2 (relative u x^2 / 2 on the result) and
# three products on |x phi(x)| <= 0.25; the final sum u |G| <= 1.13 u:  eps_G = u (8 + |x| + x^2 |x| phi(x)).
# gelu_out = gelu(C) in fp32: |gelu'| <= 1.13 carries C's error; erff's 2 ulp and the argument's rounding on
# 0.5 |x| (1 + erf), the two products and (1 + erf)'s rounding add at most 4 u (|x| + 1).
FLOOR = 1e-30


def _gelu_grad64(x):
    return 0.5 * (1 + torch.erf(x / 2 ** 0.5)) + x * torch.exp(-0.5 * x * x) / (2 * torch.pi) ** 0.5


def _eps_gelu_grad(x):
    phi = torch.exp(-0.5 * x * x) / (2 * torch.pi) ** 0.5
    return U32 * (8 + x.abs() + x * x * x.abs() * phi)


def _view(buf, off, strides, size):
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


def _linear_dw(name, B, N, K, ldy=None, y_off=0, ldx=None):
    """hl_linear_dw: dW (N x K) = dy^T (B x N, ld ldy) x (B x K, ld ldx); no split buffer."""
    ldy, ldx = ldy or N, ldx or K
    return Site(name, "dytx", N, K, B, 1, (0, 1, ldy), (0, ldx, 1), (0, K, 1), 1, a_off=y_off, partial=False)


def _per_head(kind, H, B, splits):
    """The six batched per-head call sites of rh_forward / rh_backward, with their real strides: q, dO, o, dq are
    B x I (I = 64 H); kq, d~, c, u are B x H x 1280; W_k, W_v are the two halves of to_kv (2I x 1280)."""
    I = D * H
    if kind == "kq":          # kq[b,h,:] = q[b,h,:] W_k[h]
        return Site(f"kq H={H} B={B}", "dyw", B, C, D, H, (D, I, 1), (D * C, C, 1), (C, H * C, 1), splits)
    if kind == "dtil":        # d~[b,h,:] = dO[b,h,:] W_v[h]
        return Site(f"d~ H={H} B={B}", "dyw", B, C, D, H, (D, I, 1), (D * C, C, 1), (C, H * C, 1), splits,
                    b_off=I * C)
    if kind == "o":           # o[b,h,:] = W_v[h] c[b,h,:]
        return Site(f"o H={H} B={B}", "xwt", B, D, C, H, (C, H * C, 1), (D * C, 1, C), (D, I, 1), splits,
                    b_off=I * C)
    if kind == "dq":          # dq[b,h,:] = W_k[h] u[b,h,:] / 8
        return Site(f"dq H={H} B={B}", "xwt", B, D, C, H, (C, H * C, 1), (D * C, 1, C), (D, I, 1), splits,
                    alpha=SCALE)
    if kind == "dWv":         # dW_v[h] = sum_b dO[b,h,:] (x) c[b,h,:], into the V half of to_kv's gradient
        return Site(f"dW_v H={H} B={B}", "dytx", D, C, B, H, (D, 1, I), (C, H * C, 1), (D * C, C, 1), splits,
                    c_off=I * C, c_extent=2 * I * C, partial=False)
    if kind == "dWk":         # dW_k[h] = sum_b q[b,h,:] (x) u[b,h,:] / 8, into the K half
        return Site(f"dW_k H={H} B={B}", "dytx", D, C, B, H, (D, 1, I), (C, H * C, 1), (D * C, C, 1), splits,
                    alpha=SCALE, c_extent=2 * I * C, partial=False)
    raise ValueError(kind)


# The split counts are the planner's (splits = min(264 / tiles, K / 64) when a split buffer is given and tiles < 132),
# written out so that the table provably covers: several M tiles (M = 65, 130, 600); split boundaries inside a 16-wide
# k-block (kper 94, 103, 205, 342, 117, 72); splits = 1 for each of its reasons (tiles >= 132; K < 128; no split
# buffer); the direct (non-split) epilogue with bias + accumulate, gelu_out and dgelu, and the same epilogues after the
# reduce kernel; pitch padding (ldc > N); and the six per-head call sites at 1, 3 and 8 heads.
SITES = [
    _linear("to_q B=130", 130, 512, 1024, 11),                                              # kper 94
    _linear("to_out B=130", 130, 1024, 512, 5, ldx=512, bias=True, accumulate=True),       # kper 103
    _linear("fc2 B=130", 130, 1024, 1024, 5, bias=True, accumulate=True),                  # kper 205
    _linear("fc1 B=65", 65, 1024, 1024, 8, bias=True, gelu_out=True),
    _linear("fc1 mlp=1030 B=130", 130, 1030, 1024, 5, bias=True, gelu_out=True),
    _linear("to_q B=600", 600, 512, 1024, 3),                                               # kper 342
    _linear("fc1 B=600", 600, 1024, 1024, 1, bias=True, gelu_out=True),                    # tiles 160: direct
    _linear("to_out B=600", 600, 1024, 512, 1, ldx=512, bias=True, accumulate=True),       # direct
    _linear("decpose B=65", 65, 144, 1024, 16, ldy=READ_LD, bias=True, y_extent=65 * READ_LD),
    _linear("decshape B=7", 7, 10, 1024, 16, ldy=READ_LD, y_off=144, bias=True, y_extent=7 * READ_LD),
    _linear_dx("fc2 dx B=600", 600, 1024, 1024, 1, dgelu=True),                             # direct dgelu
    _linear_dx("fc2 dx B=130", 130, 1024, 1024, 5, dgelu=True),
    _linear_dx("to_out dx B=65", 65, 1024, 512, 16),
    _linear_dx("decpose dx B=65", 65, 144, 1024, 2, ldy=READ_LD),                           # kper 72
    _linear_dx("decshape dx B=65", 65, 10, 1024, 1, ldy=READ_LD, y_off=144, accumulate=True),   # K = 10
    _linear_dx("deccam dx B=130", 130, 3, 1024, 1, ldy=READ_LD, y_off=154, accumulate=True),    # K = 3
    _linear_dx("fc2 dx mlp=1 B=70", 70, 1024, 1, 16, dgelu=True),
    _linear_dw("fc2 dW B=600", 600, 1024, 1024),
    _linear_dw("decpose dW B=65", 65, 144, 1024, ldy=READ_LD),
    _linear_dw("fc1 dW mlp=200 B=70", 70, 200, 1024),
] + [_per_head(kind, H, B, s) for kind, B, split_by_heads in (
    ("kq", 7, {1: 1, 3: 1, 8: 1}),          # K = 64
    ("dtil", 7, {1: 1, 3: 1, 8: 1}),
    ("o", 130, {1: 20, 3: 20, 8: 11}),      # kper 64, 64, 117
    ("dq", 130, {1: 20, 3: 20, 8: 11}),
    ("dWv", 65, {1: 1, 3: 1, 8: 1}),        # no split buffer
    ("dWk", 65, {1: 1, 3: 1, 8: 1}),
) for H, s in split_by_heads.items()]


def test_site_table_covers_every_planner_branch():
    """What the table claims about itself (host-side; the GPU test asserts the kernel's split counts)."""
    kper = lambda s: (s.K + s.splits - 1) // s.splits
    assert {65, 130, 600} <= {s.M for s in SITES}
    assert any(s.splits > 1 and kper(s) % 16 for s in SITES)
    tiles = lambda s: ((s.N + 63) // 64) * ((s.M + 63) // 64) * s.batch
    assert any(s.splits == 1 and s.partial and tiles(s) >= 132 for s in SITES)
    assert any(s.splits == 1 and s.partial and s.K < 128 for s in SITES)
    assert any(s.splits == 1 and not s.partial for s in SITES)
    for flag in ("accumulate", "gelu_out", "dgelu"):
        assert any(getattr(s, flag) and s.splits == 1 for s in SITES), flag
        assert any(getattr(s, flag) and s.splits > 1 for s in SITES), flag
    assert any(s.sC[1] > s.N for s in SITES)
    assert {s.batch for s in SITES} >= {1, 3, 8}


def _operands(site, integer: bool, g):
    """Flat fp32 buffers of A, B, bias, dgelu and C0 (C0: the accumulate input, NaN outside the view)."""
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
    Csz = (site.batch, site.M, site.N)
    out, gout = C0.clone(), (torch.full_like(C0, float("nan")) if site.gelu_out else None)
    d = hp.HlGemm(A=A.data_ptr() + 4 * site.a_off, sAz=site.sA[0], sAm=site.sA[1], sAk=site.sA[2],
                     Bm=Bm.data_ptr() + 4 * site.b_off, sBz=site.sB[0], sBk=site.sB[1], sBn=site.sB[2],
                     C=out.data_ptr() + 4 * site.c_off, sCz=site.sC[0], ldc=site.sC[1],
                     M=site.M, N=site.N, K=site.K, batch=site.batch, alpha=site.alpha,
                     bias=probe.ptr(bias), dgelu=None if dg is None else dg.data_ptr() + 4 * site.c_off,
                     gelu_out=None if gout is None else gout.data_ptr() + 4 * site.c_off,
                     accumulate=int(site.accumulate), partial=probe.ptr(split) if site.partial else None, splits=-7)
    n = hp.hl_gemm(d, site.orient)
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
    m = torch.zeros(n, dtype=torch.bool, device="cuda")
    _view(m, site.c_off, site.sC, (site.batch, site.M, site.N)).fill_(True)
    return m


@pytest.fixture(scope="module")
def split_buf(cuda_dev):
    n = hp.lib().head_probe_hl_split_floats()
    assert n == 264 * 64 * 64
    return torch.empty(n, device=cuda_dev)


@pytest.mark.parametrize("site", SITES, ids=[s.name for s in SITES])
def test_hl_gemm_integer_exact(site, split_buf):
    """Integer operands in [-4, 4], an integer bias and C0, alpha a power of two: every partial sum is an integer below
    2^24 (|sum| <= 16 K), so the result equals fp64 exactly; a dropped, doubled or misindexed term fails.  dgelu rows
    run without dgelu here."""
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


@pytest.mark.parametrize("site", SITES, ids=[s.name for s in SITES])
def test_hl_gemm_random_within_bound(site, split_buf):
    g = torch.Generator(device="cuda").manual_seed(7 + zlib.crc32(site.name.encode()))
    A, Bm, bias, dg, C0 = _operands(site, False, g)
    outs = _twice(lambda: _run_site(site, A, Bm, bias, dg, C0, split_buf))
    Csz = (site.batch, site.M, site.N)
    kper = (site.K + site.splits - 1) // site.splits
    n = kper + (site.splits if site.splits > 1 else 0)
    ref, mag, G, epsG, c0 = _reference(site, A, Bm, bias, dg, C0)
    absG = G.abs() if torch.is_tensor(G) else G
    c0a = c0.abs() if torch.is_tensor(c0) else 0
    bound = gamma(n + 4) * absG * mag + epsG * mag + U32 * c0a + FLOOR
    got = _view(outs[0], site.c_off, site.sC, Csz)
    assert_within(f"hl_gemm {site.name}", got, ref, bound)
    cov = _covered(site, outs[0].numel())
    assert outs[0][~cov].isnan().all(), "wrote outside the output view"
    if site.gelu_out:
        assert_within(f"hl_gemm gelu_out {site.name}", _view(outs[1], site.c_off, site.sC, Csz), probe.gelu64(ref),
                      1.13 * bound + 4 * U32 * (ref.abs() + 1))
        assert outs[1][~cov].isnan().all()
    # teeth: the same bound rejects the reference without one k-term, and without one split's partial
    mask = torch.ones(site.K, dtype=torch.float64, device="cuda")
    mask[site.K // 2] = 0
    assert _rejects(got, _reference(site, A, Bm, bias, dg, C0, mask)[0], bound), "bound accepts a dropped k-term"
    if site.splits > 1:
        mask = torch.ones(site.K, dtype=torch.float64, device="cuda")
        mask[kper:min(site.K, 2 * kper)] = 0
        assert _rejects(got, _reference(site, A, Bm, bias, dg, C0, mask)[0], bound), "bound accepts a dropped split"


# ------------------------------------------------------------------------------------------------ cross-attention
def _attn_inputs(regime: str, B: int, H: int, g, integer=False):
    """X (B, 1280, 192) channel-first features and the per-head query vector kq (B, H, 1280)."""
    if integer:
        X = torch.randint(-4, 5, (B, C, T), device="cuda", generator=g).float()
        v = torch.randint(-4, 5, (B, H, C), device="cuda", generator=g).float()
        return X, v
    X = torch.randn(B, C, T, device="cuda", generator=g)
    v = torch.randn(B, H, C, device="cuda", generator=g)
    if regime == "zero":                # uniform P: c is the mean of X over the positions
        v.zero_()
    elif regime == "dominant":          # head h peaks at a position of chunk (h + b) mod 12
        for b in range(B):
            for h in range(H):
                t = 16 * ((h + b) % NCHUNK) + (5 * h + 3) % CHUNK
                v[b, h] = 0.05 * X[b, :, t] + 0.01 * v[b, h]
    elif regime == "large":             # scores of +- several hundred: whole chunks underflow in the combine
        v *= 60
    return X, v


def _attn_fwd(X, v, B, H):
    s, stat, part = _nan(B, H, T), _nan(B, NCHUNK, H, 2), _nan(B, NCHUNK, H, C)
    c, lse = _nan(B, H, C), _nan(B, H)
    hp.call("head_probe_rh_attn_fwd", X.data_ptr(), v.data_ptr(), H, SCALE, B, s.data_ptr(), stat.data_ptr(),
            part.data_ptr(), c.data_ptr(), lse.data_ptr(), probe.stream())
    torch.cuda.synchronize()
    return s, stat, part, c, lse


# Scores: each lane takes 40 of the 1280 channels in a serial fmaf chain, then a 5-level shuffle tree: 45 roundings,
# times 1/8 (exact): |s - s64| <= gamma_45 / 8 sum_c |v_c| |X_cj|.  A score error moves p_j by that much relatively and
# L by at most the largest one: 2 gamma_45 / 8 max_j sum |v||X| (as probe.attention_bound).  Probabilities:
# expf(s - m_loc) and expf(m_loc - m) round their arguments (u |s - m| together, since s <= m_loc <= m) and each
# carry 2 ulp (4 u); L is a 5-level shuffle sum, 12 products and 12 additions, then 1 / L: 19 u more.  The output is a
# 16-term fmaf chain per chunk and a 12-term one over the chunks: 28 u of sum p |x|.  Together 56 u + u |s_j - m|.
def _attn_fwd_ref(X, v):
    Xd, vd = X.double(), v.double()
    s64 = SCALE * torch.einsum("bct,bhc->bht", Xd, vd)
    sabs = SCALE * torch.einsum("bct,bhc->bht", Xd.abs(), vd.abs())
    p = torch.softmax(s64, -1)
    c64 = torch.einsum("bht,bct->bhc", p, Xd)
    lse64 = torch.logsumexp(s64, -1)
    m = s64.amax(-1, keepdim=True)
    e_s = 2 * gamma(45) * sabs.amax(-1, keepdim=True)
    rel = 56 * U32 + U32 * (s64 - m).abs() + e_s                         # per position
    bound_c = U32 * c64.abs() + torch.einsum("bht,bct->bhc", p * rel, Xd.abs()) + 2.0 ** -30
    # lse = m + logf(L): the sum's and logf's roundings, and L's relative error (the p-weighted rel above, less the
    # output chains' 28 u)
    bound_lse = 2 * U32 * (lse64.abs() + m.squeeze(-1).abs() + (lse64 - m.squeeze(-1)).abs()) + \
        (p * (rel - 28 * U32)).sum(-1) + 2.0 ** -30
    bound_s = gamma(45) * sabs + 2.0 ** -60
    return s64, c64, lse64, p, bound_s, bound_c, bound_lse


@pytest.mark.parametrize("B", [1, 7])
@pytest.mark.parametrize("H", [1, 3, 8])
def test_attn_forward_integer_scores_exact(H, B):
    g = torch.Generator(device="cuda").manual_seed(100 * H + B)
    X, v = _attn_inputs("random", B, H, g, integer=True)
    s, *_ = _twice(lambda: _attn_fwd(X, v, B, H))
    want = SCALE * torch.einsum("bct,bhc->bht", X.double(), v.double())
    assert torch.equal(s.double(), want)


@pytest.mark.parametrize("regime", ["random", "zero", "dominant", "large"])
@pytest.mark.parametrize("B", [1, 7])
@pytest.mark.parametrize("H", [1, 3, 8])
def test_attn_forward_and_backward(H, B, regime):
    g = torch.Generator(device="cuda").manual_seed(1000 * H + 10 * B + len(regime))
    X, v = _attn_inputs(regime, B, H, g)
    s, stat, part, c, lse = _twice(lambda: _attn_fwd(X, v, B, H))
    assert stat.isfinite().all() and part.isfinite().all()
    s64, c64, lse64, p, bound_s, bound_c, bound_lse = _attn_fwd_ref(X, v)
    assert_within(f"attn s {regime} H={H} B={B}", s, s64, bound_s)
    assert_within(f"attn c {regime} H={H} B={B}", c, c64, bound_c)
    assert_within(f"attn lse {regime} H={H} B={B}", lse, lse64, bound_lse)
    if regime == "large":               # some chunk's weight e^(m_k - m) is 0 in fp32
        mk = stat[..., 0].double()
        assert (torch.exp(mk - mk.amax(1, keepdim=True)) < 2.0 ** -150).any()
    # teeth: without its most probable position the reference leaves the bound
    j = p.argmax(-1, keepdim=True)
    p_drop = p.scatter(-1, j, 0.0)
    assert _rejects(c, torch.einsum("bht,bct->bhc", p_drop, X.double()), bound_c)

    # Backward, from the kernel's own fp32 s and lse as the engine feeds them.  fp64: P = exp(s - lse),
    # dP = X^T d~, delta = dO . o, dS = P (dP - delta), u = X dS.
    I = D * H
    dtil = torch.randn(B, H, C, device="cuda", generator=g)
    dO, o = torch.randn(B, I, device="cuda", generator=g), torch.randn(B, I, device="cuda", generator=g)

    def bwd():
        part_b, u = _nan(B, NCHUNK, H, C), _nan(B, H, C)
        hp.call("head_probe_rh_attn_bwd", X.data_ptr(), dtil.data_ptr(), H, SCALE, B, s.data_ptr(), lse.data_ptr(),
                dO.data_ptr(), o.data_ptr(), part_b.data_ptr(), u.data_ptr(), probe.stream())
        torch.cuda.synchronize()
        return (u,)

    (u,) = _twice(bwd)
    Xd = X.double()
    P = torch.exp(s.double() - lse.double().unsqueeze(-1))
    dP = torch.einsum("bct,bhc->bht", Xd, dtil.double())
    dPabs = torch.einsum("bct,bhc->bht", Xd.abs(), dtil.double().abs())
    dOh, oh = dO.double().view(B, H, D), o.double().view(B, H, D)
    delta = (dOh * oh).sum(-1, keepdim=True)
    dabs = (dOh * oh).abs().sum(-1, keepdim=True)
    dS = P * (dP - delta)
    u64 = torch.einsum("bht,bct->bhc", dS, Xd)
    # dP: 40 lane terms + 5 shuffles (gamma_45 of sum |d~||X|); delta: a product, an fma and 5 shuffles (gamma_7);
    # P = expf(s - lse): the argument's rounding u |s - lse| and 2 ulp (4 u); dP - delta and the product with P: 2 u;
    # u: a 16-term fmaf chain per chunk and 12 chunk additions: gamma_28 of sum |dS| |x|.
    rel_p = U32 * (s.double() - lse.double().unsqueeze(-1)).abs()
    w = P * (gamma(45) * dPabs + gamma(7) * dabs) + dS.abs() * (gamma(28) + 6 * U32 + rel_p)
    bound_u = torch.einsum("bht,bct->bhc", w, Xd.abs()) + 2.0 ** -30
    assert_within(f"attn u {regime} H={H} B={B}", u, u64, bound_u)
    j = dS.abs().argmax(-1, keepdim=True)
    assert _rejects(u, torch.einsum("bht,bct->bhc", dS.scatter(-1, j, 0.0), Xd), bound_u)


# ------------------------------------------------------------------------------------------------ LayerNorm
def _ln_rows(B: int, first: int, g):
    """Row r is kind (r + first) % 3: mean 0 / std 1, mean 1000 / std 1, or the constant 0.7 (variance 0, so
    rstd = eps^-1/2)."""
    x = torch.randn(B, E, device="cuda", generator=g)
    for r in range(B):
        k = (r + first) % 3
        if k == 1:
            x[r] += 1000
        elif k == 2:
            x[r] = 0.7
    return x


def _ln_fwd(x, gw, bw, B):
    y, mean, rstd = _nan(B, E), _nan(B), _nan(B)
    hp.call("head_probe_rh_ln_fwd", x.data_ptr(), gw.data_ptr(), bw.data_ptr(), y.data_ptr(), mean.data_ptr(),
            rstd.data_ptr(), B, probe.stream())
    torch.cuda.synchronize()
    return y, mean, rstd


@pytest.mark.parametrize("B", [1, 5, 130])
def test_layernorm_forward_and_backward(B):
    g = torch.Generator(device="cuda").manual_seed(B)
    gw = 1 + 0.1 * torch.randn(E, device="cuda", generator=g)
    bw = 0.05 * torch.randn(E, device="cuda", generator=g)
    for first in range(3 if B == 1 else 1):
        x = _ln_rows(B, first, g)
        y, mean, rstd = _twice(lambda: _ln_fwd(x, gw, bw, B))
        xd, gd_, bd = x.double(), gw.double(), bw.double()
        mu = xd.mean(1, keepdim=True)
        var = ((xd - mu) ** 2).mean(1, keepdim=True)
        rs = (var + EPS).rsqrt()
        y64 = (xd - mu) * rs * gd_ + bd
        # mean: 3 additions per thread, 5 shuffles, 8 warp partials: gamma_16 of mean |x| (1/1024 is exact).
        # d = x - mean carries that plus u |d|.  var: a product per term and the same 16-chain: gamma_18 of var, plus
        # dmu^2 (sum_i (d_i - dmu)^2 = sum_i d_i^2 + N dmu^2, as sum_i d_i = 0), with d's own rounding twice:
        # gamma_20 of var.  rstd = rsqrtf(var + eps): 2 ulp (4 u), the sum's u, and half var's relative error.
        # y = d rs g + b: three roundings.  Second-order terms are folded into the factor 1.01.
        dmu = gamma(16) * xd.abs().mean(1, keepdim=True)
        drs = rs * (5 * U32 + 0.5 * (gamma(20) * var + dmu ** 2) / (var + EPS))
        d = (xd - mu).abs()
        bound_y = 1.01 * (gd_.abs() * (rs * (dmu + U32 * d) + d * drs) + 3 * U32 * (d * rs * gd_.abs() + bd.abs())) \
            + 2.0 ** -60
        tag = f"B={B} first={first}"
        assert_within(f"ln y {tag}", y, y64, bound_y)
        assert_within(f"ln mean {tag}", mean, mu.squeeze(1), dmu.squeeze(1) + 2.0 ** -60)
        assert_within(f"ln rstd {tag}", rstd, rs.squeeze(1), 1.01 * drs.squeeze(1))
        const = [r for r in range(B) if (r + first) % 3 == 2]
        if const:
            assert torch.allclose(rstd[const].double(), torch.full((len(const),), EPS ** -0.5, device="cuda",
                                                                    dtype=torch.float64), rtol=1e-6, atol=0)
        keep = torch.ones(E, dtype=torch.bool, device="cuda")
        keep[0] = False                   # teeth: the mean over 1023 of the 1024 columns, on the mean-0 rows
        mu_d = xd[:, keep].mean(1, keepdim=True)
        zero_mean = [r for r in range(B) if (r + first) % 3 == 0]
        if zero_mean:
            assert _rejects(y[zero_mean], ((xd - mu_d) * rs * gd_ + bd)[zero_mean], bound_y[zero_mean])

        # backward from the kernel's own mean and rstd, added into a pre-filled dx
        dy = torch.randn(B, E, device="cuda", generator=g)
        dx0 = torch.randn(B, E, device="cuda", generator=g)

        def bwd():
            dx = dx0.clone()
            hp.call("head_probe_rh_ln_bwd", x.data_ptr(), gw.data_ptr(), mean.data_ptr(), rstd.data_ptr(),
                    dy.data_ptr(), dx.data_ptr(), B, probe.stream())
            torch.cuda.synchronize()
            return (dx,)

        (dx,) = _twice(bwd)
        m_, r_ = mean.double().unsqueeze(1), rstd.double().unsqueeze(1)
        h = (xd - m_) * r_
        gdy = dy.double() * gd_
        m1, m2 = gdy.mean(1, keepdim=True), (gdy * h).mean(1, keepdim=True)
        t = gdy - m1 - h * m2
        dx64 = dx0.double() + r_ * t
        # h: 2 u; g dy: u; m1: the 16-chain, gamma_16 of mean |g dy|; m2: a product and h's 2 u more, gamma_19 of
        # mean |g dy h|; t: h m2's rounding and two subtractions, 3 u of (|g dy| + |m1| + |h m2|) and 2 u |h m2|
        # from h; times rstd: u; + dx0: u.
        S1, S2 = gdy.abs().mean(1, keepdim=True), (gdy * h).abs().mean(1, keepdim=True)
        inner = 2 * U32 * gdy.abs() + gamma(16) * S1 + h.abs() * gamma(19) * S2 + \
            4 * U32 * (gdy.abs() + m1.abs() + 2 * (h * m2).abs())
        bound_dx = 1.01 * (r_ * inner + U32 * (dx0.double().abs() + (r_ * t).abs())) + 2.0 ** -60
        assert_within(f"ln dx {tag}", dx, dx64, bound_dx)
        m1_d = gdy[:, keep].sum(1, keepdim=True) / E       # teeth: one term out of mean(g dy)
        assert _rejects(dx, dx0.double() + r_ * (gdy - m1_d - h * m2), bound_dx)


# ------------------------------------------------------------------------------------------------ column sums
@pytest.mark.parametrize("B", [1, 5, 130])
@pytest.mark.parametrize("threads,N,ld,col", [(256, 144, READ_LD, 0), (256, 10, READ_LD, 144), (256, 3, READ_LD, 154),
                                              (128, 1024, 1024, 0), (128, 1030, 1030, 0), (128, 1, 1, 0)])
def test_colsum(B, threads, N, ld, col):
    """The plain sums (integer inputs: exact, and out2 == out bit for bit), and the LayerNorm-weight sum out_g."""
    g = torch.Generator(device="cuda").manual_seed(B * 7 + N)
    PAD = 5

    def run(dy, with_g, x=None, mean=None, rstd=None):
        out, out2 = _nan(N + PAD), _nan(N + PAD)
        og = _nan(N + PAD) if with_g else None
        hp.call("head_probe_rh_colsum", threads, dy.data_ptr() + 4 * col, ld, B, N, out.data_ptr(), out2.data_ptr(),
                probe.ptr(x), probe.ptr(mean), probe.ptr(rstd), probe.ptr(og), probe.stream())
        torch.cuda.synchronize()
        return (out, out2) + ((og,) if with_g else ())

    dy = torch.randint(-50, 51, (B, ld), device="cuda", generator=g).float()
    out, out2 = _twice(lambda: run(dy, False))
    assert torch.equal(out[:N].double(), dy[:, col:col + N].double().sum(0))
    assert torch.equal(out2[:N], out[:N]) and out[N:].isnan().all() and out2[N:].isnan().all()
    # out_g = sum_b dy (x - mean) rstd in row order: per term a subtraction, two products (one may fuse with the
    # addition) and the B-term chain: gamma_(B+3) of sum_b |dy| |xhat|.  x is read at the same pitch and column.
    dyr = torch.randn(B, ld, device="cuda", generator=g)
    x = 3 + 2 * torch.randn(B, ld, device="cuda", generator=g)
    mean = 3 + 0.1 * torch.randn(B, device="cuda", generator=g)
    rstd = 0.5 + torch.rand(B, device="cuda", generator=g)
    out, out2, og = _twice(lambda: run(dyr, True, x[:, col:], mean, rstd))
    d = dyr[:, col:col + N].double()
    xhat = (x[:, col:col + N].double() - mean.double()[:, None]) * rstd.double()[:, None]
    bound = gamma(B + 3) * (d * xhat).abs().sum(0) + 2.0 ** -60
    assert_within(f"colsum out_g B={B} N={N}", og[:N], (d * xhat).sum(0), bound)
    assert og[N:].isnan().all()
    assert torch.equal(out2[:N], out[:N])
    assert_within(f"colsum out B={B} N={N}", out[:N], d.sum(0), gamma(B) * d.abs().sum(0) + 2.0 ** -60)
    if B > 1:                           # teeth: the first row left out
        assert _rejects(og[:N], (d * xhat)[1:].sum(0), bound)


# ------------------------------------------------------------------------------------------------ token 0
@pytest.mark.parametrize("B", [1, 5, 130])
def test_token0_exact(B):
    g = torch.Generator(device="cuda").manual_seed(B)
    tok_b, pos = torch.randn(E, device="cuda", generator=g), torch.randn(E, device="cuda", generator=g)

    def run():
        x = _nan(B * E + 300)
        hp.call("head_probe_rh_token0", tok_b.data_ptr(), pos.data_ptr(), x.data_ptr(), B, probe.stream())
        torch.cuda.synchronize()
        return (x,)

    (x,) = _twice(run)
    assert torch.equal(x[:B * E].view(B, E), (tok_b + pos).expand(B, E))
    assert x[B * E:].isnan().all()


# ------------------------------------------------------------------------------------------------ read-out backward
def _readout_bwd(pose6d, g_rot, g_p6, g_betas, g_cam, B):
    dread = _nan(B + 1, READ_LD)          # one spare row: must stay NaN
    hp.call("head_probe_rh_readout_bwd", pose6d.data_ptr(), probe.ptr(g_rot), probe.ptr(g_p6), probe.ptr(g_betas),
            probe.ptr(g_cam), dread.data_ptr(), B, probe.stream())
    torch.cuda.synchronize()
    return (dread,)


def _rot6d_grad64(pose6d, g_rot):
    """fp64 autograd of sum(rot6d_to_rotmat(x) * g) on the fp32 x: (B, 144)."""
    x = pose6d.double().detach().reshape(-1, 6).requires_grad_(True)
    Rm = O.rot6d_to_rotmat(x)
    (gx,) = torch.autograd.grad((Rm * g_rot.double().reshape(-1, 3, 3)).sum(), x)
    return gx.reshape(pose6d.shape[0], 144)


def _gs_scales(pose6d):
    """Per joint: |a1|, |u| (Gram-Schmidt residual), |a2|, each clamped at F.normalize's 1e-12 as in the kernel."""
    x = pose6d.double().reshape(-1, 6)
    a1, a2 = x[:, :3], x[:, 3:]
    b1 = F.normalize(a1, dim=-1)
    u = a2 - (b1 * a2).sum(-1, keepdim=True) * b1
    return a1.norm(dim=-1).clamp_min(1e-12), u.norm(dim=-1).clamp_min(1e-12), a2.norm(dim=-1)


def _gx_bound(pose6d, g_rot):
    # The forward's b1, b2 are within 2^-19 amp of fp64 (tests/test_gpu_kernels.py::test_head_assemble_vs_oracle), with
    # amp = 1 + |a2| / |u| the Gram-Schmidt amplification.  The backward divides by |u| (d b2 / d a2 ~ 1 / |u|) and by
    # |a1|, where the a1 path also carries dp gu ~ |a2| |g| / |u|: |gx| ~ |g| (amp / |a1| + 1 / |u|).  Each of its ~30
    # roundings, and the errors of b1, b2, u and |u| it starts from, is relative ~ amp u on that, so the error needs amp
    # to the second power (the first fails by orders of magnitude at amp ~ 1e3):
    #   |gx - gx64| <= 2^-18 |g| amp (amp / |a1| + 1 / |u|).
    n1, nu, n2 = _gs_scales(pose6d)
    amp = 1 + n2 / nu
    gn = g_rot.double().reshape(-1, 9).norm(dim=-1)
    per_joint = 2.0 ** -18 * gn * amp * (amp / n1 + 1 / nu)
    return per_joint.view(-1, 24, 1).expand(-1, 24, 6).reshape(-1, 144)


def _readout_inputs(B, g):
    """6D poses near the identity (odd images), random (even images), and in every image joints 20..23 with a2 nearly
    parallel to a1 (amp 1e2 .. 1e4), where the Gram-Schmidt backward is ill-conditioned."""
    pose6d = 0.3 * torch.randn(B, 144, device="cuda", generator=g)
    pose6d += torch.tensor([1.0, 0, 0, 0, 1.0, 0], device="cuda").repeat(24)
    pose6d[::2] = torch.randn(pose6d[::2].shape, device="cuda", generator=g)
    j = pose6d.view(B, 24, 6)[:, 20:]
    tilt = torch.tensor([1e-2, 1e-3, 3e-4, 1e-4], device="cuda").view(1, 4, 1)
    j[..., 3:] = -2.5 * j[..., :3] + tilt * torch.randn(B, 4, 3, device="cuda", generator=g)
    return (pose6d, torch.randn(B, 24, 3, 3, device="cuda", generator=g),
            torch.randn(B, 144, device="cuda", generator=g),
            torch.randn(B, 10, device="cuda", generator=g), torch.randn(B, 3, device="cuda", generator=g))


@pytest.mark.parametrize("B", [1, 5, 130])
def test_readout_backward_every_upstream_subset(B):
    g = torch.Generator(device="cuda").manual_seed(50 + B)
    pose6d, g_rot, g_p6, g_betas, g_cam = _readout_inputs(B, g)
    gx64 = _rot6d_grad64(pose6d, g_rot)
    gxb = _gx_bound(pose6d, g_rot)
    for mask in range(16):
        use = [bool(mask >> i & 1) for i in range(4)]
        args = [t if on else None for t, on in zip((g_rot, g_p6, g_betas, g_cam), use)]
        (dread,) = _twice(lambda: _readout_bwd(pose6d, *args, B))
        assert dread[B].isnan().all()
        d = dread[:B]
        assert torch.equal(d[:, 157:], torch.zeros(B, 3, device="cuda")), "pad columns"
        assert torch.equal(d[:, 144:154], g_betas if use[2] else torch.zeros(B, 10, device="cuda"))
        assert torch.equal(d[:, 154:157], g_cam if use[3] else torch.zeros(B, 3, device="cuda"))
        if not use[0]:
            assert torch.equal(d[:, :144], g_p6 if use[1] else torch.zeros(B, 144, device="cuda"))
            continue
        want = gx64 + (g_p6.double() if use[1] else 0)
        bound = gxb + (U32 * want.abs() if use[1] else 0) + 2.0 ** -60   # the fp32 addition of g_pose6d
        assert_within(f"readout gx B={B} mask={mask}", d[:, :144], want, bound)
        if mask == 1:                 # teeth: one joint's b3 gradient left out
            g_cut = g_rot.clone()
            g_cut[0, 3, 2] = 0
            assert _rejects(d[:, :144], _rot6d_grad64(pose6d, g_cut), bound)


def test_readout_backward_at_the_normalize_clamp():
    """Exactly representable degenerate inputs: a1 = 0 (|a1| clamped at 1e-12) and a2 = 2 a1 on an axis (u = 0
    exactly).  The gradient follows F.normalize's clamp: g / 1e-12 through the clamp, with no projection term."""
    B = 1
    g = torch.Generator(device="cuda").manual_seed(3)
    pose6d = torch.tensor([1.0, 0, 0, 0, 1.0, 0], device="cuda").repeat(24).view(B, 144)
    x = pose6d.view(24, 6)
    x[0] = torch.tensor([0.0, 0.0, 0.0, 0.3, -0.5, 0.25])       # a1 = 0
    x[1] = torch.tensor([0.0, 0.5, 0.0, 0.0, 1.0, 0.0])         # a2 = 2 a1 along y: u = 0
    x[2] = torch.tensor([0.0, 0.0, -2.0, 0.0, 0.0, -4.0])       # along z
    x[3] = torch.tensor([0.0, 0.0, 0.0, 0.0, 0.0, 0.0])         # both zero
    g_rot = torch.randn(B, 24, 3, 3, device="cuda", generator=g)
    (dread,) = _twice(lambda: _readout_bwd(pose6d, g_rot, None, None, None, B))
    gx64 = _rot6d_grad64(pose6d, g_rot)
    assert gx64[0, :4 * 6].abs().max() > 1e11                    # the clamp's 1 / 1e-12 is in play
    n1, nu, n2 = _gs_scales(pose6d)
    gn = g_rot.double().reshape(-1, 9).norm(dim=-1)
    # relative: ~30 roundings on terms of size |g| (1 + |a2|) (1 / |a1| + 1 / |u|), the clamped norms included
    per_joint = 2.0 ** -18 * gn * (1 + n2) * (1 / n1 + 1 / nu)
    bound = per_joint.view(-1, 24, 1).expand(-1, 24, 6).reshape(-1, 144)
    assert_within("readout gx at the clamp", dread[:B, :144], gx64, bound)
    assert torch.equal(dread[:B, 144:], torch.zeros(B, 16, device="cuda"))
    # the a2 = 2 a1 joints: no gradient along a1's axis, exactly
    assert dread[0, 6 + 1] == 0 and dread[0, 6 + 4] == 0 and dread[0, 12 + 2] == 0 and dread[0, 12 + 5] == 0


# ------------------------------------------------------------------------------------------------ the whole head
# Helpers as in tests/test_gpu_head_train.py.  Gradient bound per parameter tensor, unchanged from there:
# max |g - g64| <= max(4 x the fp32 torch restatement's own error, 1e-5 max |g64|).  Forward outputs are also held row
# by row: max_row |y - y64| <= 1e-5 max_row |y64|.
def _feats(cfg, B, seed, dev):
    gen = torch.Generator().manual_seed(seed)
    return torch.randn(B, cfg.vit_dim, cfg.grid_h, cfg.grid_w, generator=gen).to(dev)


def _head_sd(sd, dtype, dev):
    return {k: v.to(dev, dtype).clone().requires_grad_(k.split(".")[-1] not in ("init_body_pose", "init_betas",
                                                                                  "init_cam"))
            for k, v in sd.items() if k.startswith("smpl_head.")}


def _restated(sd, feats, cfg, dtype):
    leaves = _head_sd(sd, dtype, feats.device)
    params, cam, aux = R.regression_head_forward(leaves, feats.to(dtype).flatten(2).transpose(1, 2), cfg,
                                                 O.Numerics(False))
    rot = torch.cat([params["global_orient"], params["body_pose"]], 1)
    return leaves, aux["pred_body_pose_6d"], params["betas"], cam, rot


def _upstream(B, seed, dev):
    gen = torch.Generator().manual_seed(seed)
    return (torch.randn(B, 24, 3, 3, generator=gen).to(dev), torch.randn(B, 10, generator=gen).to(dev),
            torch.randn(B, 3, generator=gen).to(dev), torch.randn(B, 144, generator=gen).to(dev))


def _loss(outs, up, use):
    """sum over the used outputs of output * upstream; outs = (rotmats, betas, cam, pose6d)."""
    return sum((o * u.to(o.dtype)).sum() for o, u, on in zip(outs, up, use) if on)


def _ref_grads(leaves, outs, up, use=(True, True, True, False)):
    loss = _loss(outs, up, use)
    names = [k for k, v in leaves.items() if v.requires_grad]
    gs = torch.autograd.grad(loss, [leaves[k] for k in names], allow_unused=True)
    return {k[len("smpl_head."):]: (torch.zeros_like(leaves[k]) if g is None else g) for k, g in zip(names, gs)}


def _cuda_grads(head, feats, up, use=(True, True, True, False)):
    from tokenhmr_b200.heads import _RegHeadFn
    head.zero_grad(set_to_none=True)
    pose6d, betas, cam, rot = _RegHeadFn.apply(head, True, feats, *head._params())
    _loss((rot, betas, cam, pose6d), up, use).backward()
    return {k: p.grad.clone() for k, p in head.named_parameters()}, (rot.detach(), betas.detach(), cam.detach(),
                                                                     pose6d.detach())


def _check_head(cfg, sd, B, seed, dev, use=(True, True, True, False)):
    """Forward row by row and every parameter gradient against the fp64 restatement; returns the CUDA gradients."""
    from tokenhmr_b200.heads import RegressionHead
    head = RegressionHead(cfg, sd, dev)
    feats = _feats(cfg, B, seed, dev)
    up = _upstream(B, seed + 1, dev)
    got, outs = _cuda_grads(head, feats, up, use)
    l64, p6, be, ca, rot = _restated(sd, feats, cfg, torch.float64)
    for name, a, b in zip(("rotmats", "betas", "cam", "pose6d"), outs, (rot, be, ca, p6)):
        a, b = a.double().reshape(B, -1), b.detach().reshape(B, -1)
        err, scale = (a - b).abs().amax(1), b.abs().amax(1)
        assert (err <= 1e-5 * scale).all(), (name, float((err / scale).max()))
        print(f"[row] {name} B={B}: worst row error / row scale {float((err / scale).max()):.2e}")
    g64 = _ref_grads(l64, (rot, be, ca, p6), up, use)
    del l64, rot, be, ca, p6
    l32, p6, be, ca, rot = _restated(sd, feats, cfg, torch.float32)
    g32 = _ref_grads(l32, (rot, be, ca, p6), up, use)
    del l32, rot, be, ca, p6
    assert set(got) == set(g64)
    worst = 0.0
    for k, ref in g64.items():
        scale = ref.abs().max().item()
        err = (got[k].double() - ref).abs().max().item()
        own = (g32[k].double() - ref).abs().max().item()
        bound = max(4 * own, 1e-5 * scale)
        worst = max(worst, err / max(bound, 1e-300))
        assert err <= bound, (k, err, own, scale)
    print(f"[grad] depth={cfg.dec_depth} heads={cfg.dec_heads} mlp={cfg.dec_mlp_dim} B={B} use={use}: "
          f"worst gradient error / bound {worst:.3f}")
    inner = cfg.dec_inner
    for l in range(cfg.dec_depth):
        assert not got[f"transformer.transformer.layers.{l}.0.fn.to_qkv.weight"][:2 * inner].any()
    assert not got["transformer.to_token_embedding.weight"].any()
    return got


def _cfg(depth=6, heads=8, mlp=1024):
    from tokenhmr_b200.config import tiny_config
    return dataclasses.replace(tiny_config(vit_depth=1, head=REG), dec_depth=depth, dec_heads=heads, dec_mlp_dim=mlp)


@pytest.fixture(scope="module")
def release_sd():
    from tokenhmr_b200 import synth
    return synth.make_state_dict(_cfg())


@pytest.mark.parametrize("B", [65, 130])
def test_head_release_dims_at_multi_tile_batches(release_sd, cuda_dev, B):
    _check_head(_cfg(), release_sd, B, 300 + B, cuda_dev)


def test_head_depth1_at_the_direct_epilogue_batch(cuda_dev):
    """B = 600: every 1024-wide linear has >= 132 tiles, so the bias + accumulate, gelu_out and dgelu epilogues run
    without split-K, end to end."""
    from tokenhmr_b200 import synth
    cfg = _cfg(depth=1)
    _check_head(cfg, synth.make_state_dict(cfg), 600, 600, cuda_dev)
    torch.cuda.empty_cache()


@pytest.mark.parametrize("B", [1, 70])
@pytest.mark.parametrize("depth,heads,mlp", [(1, 1, 1), (2, 3, 200), (3, 7, 1030)])
def test_head_non_release_dims(cuda_dev, depth, heads, mlp, B):
    from tokenhmr_b200 import synth
    cfg = _cfg(depth, heads, mlp)
    _check_head(cfg, synth.make_state_dict(cfg), B, 10 * depth + B, cuda_dev)


@pytest.mark.parametrize("use", [(False, False, True, False), (False, True, False, False), (True, False, False, False),
                                 (False, False, False, True), (True, True, True, True)],
                         ids=["cam", "betas", "rotmats", "pose6d", "all"])
def test_head_upstream_subsets(release_sd, cuda_dev, use):
    """Through _RegHeadFn, an output the loss leaves unused arrives as a null upstream gradient."""
    got = _check_head(_cfg(), release_sd, 5, 77, cuda_dev, use)
    if use == (False, False, True, False):
        for k in ("decpose.weight", "decpose.bias", "decshape.weight", "decshape.bias"):
            assert torch.equal(got[k], torch.zeros_like(got[k])), k

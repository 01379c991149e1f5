"""The GEMM's specialised epilogue kinds (gemm_epilogue_kind: kEpiF16, kEpiBiasF16, kEpiBiasGeluF16, kEpiBiasResidF32)
against the general epilogue (gemm_epilogue_rows), bit for bit, through the GEMM plan probe: at the ViT's five M = 12288
shapes and at M = 576 with partial row and column tiles, at block_n 128 and 256.  Also: the plan falls back to the
general kind where a base or pitch forbids 16-byte row vectors, and the per-tile timeline records each CTA's tiles."""
import pytest
import torch

import gemm_probe

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _flags(cuda_dev, built_lib):
    yield
    assert gemm_probe.flags() == 0, "GEMM probe pipeline timeout"
    assert built_lib.thmr_check_device_flags() == 0, built_lib.thmr_last_error()


KINDS = ["f16", "bias_f16", "bias_gelu_f16", "bias_resid_f32"]


def operands(M, N, K, kind, g, alpha=1.0):
    A = torch.randn(M, K, device="cuda", generator=g).half()
    W = (K ** -0.5 * torch.randn(N, K, device="cuda", generator=g)).half()
    kw = {"alpha": alpha}
    if kind != "f16":
        kw["bias"] = torch.randn(N, device="cuda", generator=g)
    if kind == "bias_gelu_f16":
        kw["act"] = "gelu"
    x0 = torch.randn(M, N, device="cuda", generator=g) if kind == "bias_resid_f32" else None
    return A, W, kw, x0


def run(A, W, M, N, K, kind, kw, x0, bn, epi):
    """One launch; returns the output (fp32 in-place residual, or fp16)."""
    if kind == "bias_resid_f32":
        x = x0.clone()
        gemm_probe.gemm(A, W, M, N, K, resid=x, ldr=N, out32=x, ld32=N, force_bn=bn, epi=epi, **kw)
        return x
    y = torch.full((M, N), float("nan"), dtype=torch.float16, device="cuda")
    gemm_probe.gemm(A, W, M, N, K, out16=y, ld16=N, force_bn=bn, epi=epi, **kw)
    return y


# name: (N, K, epilogue kind) of the ViT's GEMMs at bs = 64 (M = 12288)
VIT = {"qkv": (3840, 1280, "bias_f16"), "proj": (1280, 1280, "bias_resid_f32"), "fc1": (5120, 1280, "bias_gelu_f16"),
       "fc2": (1280, 5120, "bias_resid_f32"), "to_kv": (6144, 1280, "f16")}


@pytest.mark.parametrize("bn", [128, 256])
@pytest.mark.parametrize("gemm", list(VIT))
def test_vit_kinds_equal_general(cuda_dev, gemm, bn):
    M = 12288
    N, K, kind = VIT[gemm]
    g = torch.Generator(device="cuda").manual_seed(11)
    A, W, kw, x0 = operands(M, N, K, kind, g)
    assert gemm_probe.plan(A, W, M, N, K, force_bn=bn, **kw, **({"out16": A, "ld16": N} if x0 is None else
                                                              {"resid": x0, "ldr": N, "out32": x0, "ld32": N}))[1] == kind
    got = run(A, W, M, N, K, kind, kw, x0, bn, kind)
    want = run(A, W, M, N, K, kind, kw, x0, bn, "general")
    torch.cuda.synchronize()
    assert not torch.isnan(got.float()).any()
    assert torch.equal(got, want)


# M = 576: 4.5 row tiles.  N = 200 / 328: a partial column tile, 200 = 128 + 72 and 328 = 256 + 72 end inside a chunk;
# N = 196 / 332 (multiples of 4, not of 8) end inside an octet, which goes through the scalar tail.  alpha != 1 as
# the split-precision operands use it.
@pytest.mark.parametrize("alpha", [1.0, 0.0625])
@pytest.mark.parametrize("N", [200, 328, 196, 332])
@pytest.mark.parametrize("bn", [128, 256])
@pytest.mark.parametrize("kind", KINDS)
def test_kinds_equal_general_partial_tiles(cuda_dev, kind, bn, N, alpha):
    M, K = 576, 192
    g = torch.Generator(device="cuda").manual_seed(N + bn)
    A, W, kw, x0 = operands(M, N, K, kind, g, alpha)
    if kind != "bias_resid_f32" and N % 8:
        pytest.skip("fp16 rows of N % 8 != 0 columns have no 16-byte pitch")
    got = run(A, W, M, N, K, kind, kw, x0, bn, kind)
    want = run(A, W, M, N, K, kind, kw, x0, bn, "general")
    torch.cuda.synchronize()
    assert not torch.isnan(got.float()).any()
    assert torch.equal(got, want)


def test_misaligned_operands_fall_back_to_general(cuda_dev):
    M, N, K = 576, 200, 192
    g = torch.Generator(device="cuda").manual_seed(3)
    A, W, kw, _ = operands(M, N, K, "bias_f16", g)
    out = torch.zeros(M * (N + 8) + 8, dtype=torch.float16, device="cuda")
    assert gemm_probe.plan(A, W, M, N, K, out16=out, ld16=N, force_bn=128, **kw)[1] == "bias_f16"
    assert gemm_probe.plan(A, W, M, N, K, out16=out, ld16=N + 4, force_bn=128, **kw)[1] == "general"    # pitch
    assert gemm_probe.plan(A, W, M, N, K, out16=out[4:], ld16=N, force_bn=128, **kw)[1] == "general"    # base
    b = torch.zeros(N + 1, device="cuda")
    assert gemm_probe.plan(A, W, M, N, K, out16=out, ld16=N, force_bn=128, alpha=1.0, bias=b[1:])[1] == "general"
    x = torch.zeros(M * (N + 4) + 4, device="cuda")
    rk = dict(force_bn=256, **kw)
    assert gemm_probe.plan(A, W, M, N, K, resid=x, ldr=N, out32=x, ld32=N, **rk)[1] == "bias_resid_f32"
    assert gemm_probe.plan(A, W, M, N, K, resid=x, ldr=N + 2, out32=x, ld32=N + 2, **rk)[1] == "general"
    assert gemm_probe.plan(A, W, M, N, K, resid=x[1:], ldr=N, out32=x[1:], ld32=N, **rk)[1] == "general"
    # options no specialised kind has, and the narrow tiles, stay general too
    assert gemm_probe.plan(A, W, M, N, K, out16=out, ld16=N, force_bn=64, **kw)[1] == "general"
    assert gemm_probe.plan(A, W, M, N, K, out16=out, ld16=N, out32=x, ld32=N, force_bn=128, **kw)[1] == "general"
    assert gemm_probe.plan(A, W, M, N, K, out16=out, ld16=N, seq=(8, 1, 7), force_bn=128, **kw)[1] == "general"
    # a forced kind that does not fit is refused
    with pytest.raises(RuntimeError, match="does not fit"):
        gemm_probe.plan(A, W, M, N, K, out16=out, ld16=N + 4, force_bn=128, epi="bias_f16", **kw)


@pytest.mark.parametrize("kind", ["general", None])
@pytest.mark.parametrize("bn", [128, 256])
def test_timeline_records_each_ctas_tiles(cuda_dev, bn, kind):
    M, N, K = 12288, 3840, 256
    g = torch.Generator(device="cuda").manual_seed(5)
    A, W, kw, _ = operands(M, N, K, "bias_f16", g)
    out = torch.empty(M, N, dtype=torch.float16, device="cuda")
    _, _, grid = gemm_probe.plan(A, W, M, N, K, out16=out, ld16=N, force_bn=bn, epi=kind, **kw)
    tiles = (M // 128) * (N // bn)
    slots = (tiles + grid - 1) // grid
    tl, sm = gemm_probe.timeline(A, W, M, N, K, slots + 2, out16=out, ld16=N, force_bn=bn, epi=kind, **kw)
    ref = torch.empty_like(out)
    gemm_probe.gemm(A, W, M, N, K, out16=ref, ld16=N, force_bn=bn, epi=kind, **kw)
    torch.cuda.synchronize()
    assert torch.equal(out, ref)   # the timeline changes nothing the kernel computes
    tl, sm = tl.cpu(), sm.cpu()
    assert ((sm >= 0) & (sm < torch.cuda.get_device_properties(0).multi_processor_count)).all()
    for cta in range(grid):
        given = len(range(cta, tiles, grid))
        rec = tl[cta]
        assert (rec[:given] > 0).all() and (rec[given:] == 0).all(), f"CTA {cta}: {given} tiles"
        stamps = rec[:given].permute(1, 0, 2)   # [wg, tile, 4]: monotone within a tile and from tile to tile
        flat = stamps.reshape(2, -1)
        assert (flat[:, 1:] >= flat[:, :-1]).all(), f"CTA {cta}: stamps not monotone"

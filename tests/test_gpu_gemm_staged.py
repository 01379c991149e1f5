"""The GEMM's element-wise epilogue on its 16-byte vector paths: N, ld32, ld16 and ldr multiples of 8 (or of 4), against
torch fp64 through the kernel probe.  test_gpu_kernels.py checks the same epilogue options at N = 197 / 198, where every
access falls back to scalars; here the same cases run where bases and pitches allow row vectors, with partial row and
column tiles, column counts that are not a multiple of the 32- or 64-column staging chunk, and the CTA pair."""
import pytest
import torch

import probe
import test_gpu_kernels as kernels

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _flags(cuda_dev, built_lib):
    yield
    assert probe.flags() == 0, "probe device flags set"
    assert built_lib.thmr_check_device_flags() == 0, built_lib.thmr_last_error()


# M = 576 = 4.5 row tiles of 128 (2.25 tile pairs).  N = 200: one partial octet-aligned column tile at every width, not a
# multiple of either chunk; N = 328 = 256 + 72: a full and a partial tile at block_n 256, 72 = 64 + 8 columns into the
# last chunk.  The cases' pitch offsets keep ld16 = N + 8 / + 16 and ld32 = N + 4 on the vector path, ld32 = N + 2 (the
# aliased in-place residual of "all_act32_alias") on the scalar one.
@pytest.mark.parametrize("N", [200, 328])
@pytest.mark.parametrize("bn", [32, 64, 128, 256, 512])
@pytest.mark.parametrize("case", list(kernels.EPILOGUES))
def test_gemm_epilogue_options_vector_paths(cuda_dev, case, bn, N):
    kernels.test_gemm_epilogue_options(cuda_dev, case, bn, N)


@pytest.mark.parametrize("bn", [0, 128, 256, 512])
def test_gemm_inplace_residual_matches_separate_output(cuda_dev, bn):
    """The ViT's in-place residual add (out32 aliasing resid) at a proj-like shape with a partial last row tile is
    bitwise equal to the same GEMM writing a separate output, and fp16 / fp32 outputs of one launch agree with two
    single-output launches: each element is computed once, by one thread, in one operation order."""
    g = torch.Generator(device="cuda").manual_seed(7 + bn)
    M, N, K = 1000, 1280, 320
    A = torch.randn(M, K, device=cuda_dev, generator=g).half()
    W = (0.1 * torch.randn(N, K, device=cuda_dev, generator=g)).half()
    bias = torch.randn(N, device=cuda_dev, generator=g)
    x0 = torch.randn(M, N, device=cuda_dev, generator=g)
    x = x0.clone()
    probe.gemm(A, W, M, N, K, bias=bias, resid=x, ldr=N, out32=x, ld32=N, force_bn=bn)
    y = torch.full_like(x0, float("nan"))
    y16 = torch.full((M, N), float("nan"), device=cuda_dev, dtype=torch.float16)
    probe.gemm(A, W, M, N, K, bias=bias, resid=x0, ldr=N, act="gelu", out32=y, ld32=N, out16=y16, ld16=N, force_bn=bn)
    z16 = torch.full_like(y16, float("nan"))
    probe.gemm(A, W, M, N, K, bias=bias, resid=x0, ldr=N, act="gelu", out16=z16, ld16=N, force_bn=bn)
    torch.cuda.synchronize()
    assert torch.equal(x, y)
    assert torch.equal(y16, z16)
    ref = (A.double() @ W.double().t() + bias.double() + x0.double())
    assert ((y.double() - ref).abs() <= kernels.C_ACC * (A.double().abs() @ W.double().abs().t())
            + 3 * probe.U32 * (ref.abs() + bias.double().abs() + x0.double().abs())).all()

"""The fp16-output epilogue kinds (kEpiF16, kEpiBiasF16, kEpiBiasGeluF16) store their tiles with TMA, which clips each
64 x 64 box at the output's [M, N] bounds.  Into a pitched output (ld16 = N + 8) filled with a sentinel, a kind must
write exactly the interior: the pad columns and the rows past M keep the sentinel, and the interior equals the general
epilogue's output.  M = 576 ends inside a row tile (and inside the second warpgroup's rows); N = 200 / 328 end inside
a 128-column pass and inside a 64-column box."""
import pytest
import torch

import gemm_probe

pytestmark = pytest.mark.gpu

SENTINEL = -1234.0   # exactly representable in fp16


@pytest.fixture(autouse=True)
def _flags(cuda_dev, built_lib):
    yield
    assert gemm_probe.flags() == 0, "GEMM probe pipeline timeout"
    assert built_lib.thmr_check_device_flags() == 0, built_lib.thmr_last_error()


@pytest.mark.parametrize("N", [200, 328])
@pytest.mark.parametrize("bn", [128, 256])
@pytest.mark.parametrize("kind", ["f16", "bias_f16", "bias_gelu_f16"])
def test_tma_store_writes_only_inside_bounds(cuda_dev, kind, bn, N):
    M, K, ld, rows = 576, 192, N + 8, 640   # rows: the output buffer runs 64 rows past M
    g = torch.Generator(device="cuda").manual_seed(7 * N + bn)
    A = torch.randn(M, K, device="cuda", generator=g).half()
    W = (K ** -0.5 * torch.randn(N, K, device="cuda", generator=g)).half()
    kw = {"force_bn": bn}
    if kind != "f16":
        kw["bias"] = torch.randn(N, device="cuda", generator=g)
    if kind == "bias_gelu_f16":
        kw["act"] = "gelu"
    got = torch.full((rows, ld), SENTINEL, dtype=torch.float16, device="cuda")
    assert gemm_probe.plan(A, W, M, N, K, out16=got, ld16=ld, **kw)[1] == kind
    gemm_probe.gemm(A, W, M, N, K, out16=got, ld16=ld, epi=kind, **kw)
    want = torch.full((M, N), float("nan"), dtype=torch.float16, device="cuda")
    gemm_probe.gemm(A, W, M, N, K, out16=want, ld16=N, epi="general", **kw)
    torch.cuda.synchronize()
    assert (got[:M, N:] == SENTINEL).all(), "pad columns written"
    assert (got[M:] == SENTINEL).all(), "rows past M written"
    assert not torch.isnan(want.float()).any()
    assert torch.equal(got[:M, :N], want)

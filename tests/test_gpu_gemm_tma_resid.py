"""The in-place fp32 residual kind (kEpiBiasResidF32, x = alpha * acc + bias + x) writes alpha * acc + bias into a
shared-memory ring and adds it into x with TMA reductions through a tensor map over x, which clips them at [M, N].
Into a pitched x (ld32 = N + 8) whose pad columns and rows past M hold a sentinel, the kind must write exactly the
interior, bit for bit what the general epilogue writes, and leave the sentinel alone.  Also: one k-block per tile (the
reductions of one tile right behind the next), the ViT's M = 12288 (the ring wraps many times per CTA), back-to-back
launches on the same x, a CUDA-graph replay, and a residual that does not alias the output (the general epilogue)."""
import pytest
import torch

import gemm_probe

pytestmark = pytest.mark.gpu

SENTINEL = -1234.5


@pytest.fixture(autouse=True)
def _flags(cuda_dev, built_lib):
    yield
    assert gemm_probe.flags() == 0, "GEMM probe pipeline timeout"
    assert built_lib.thmr_check_device_flags() == 0, built_lib.thmr_last_error()


def operands(M, N, K, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    A = torch.randn(M, K, device="cuda", generator=g).half()
    W = (K ** -0.5 * torch.randn(N, K, device="cuda", generator=g)).half()
    bias = torch.randn(N, device="cuda", generator=g)
    x0 = torch.randn(M, N, device="cuda", generator=g)
    return A, W, bias, x0


def pitched(x0, ld, rows):
    """x0 in the top-left corner of a [rows, ld] buffer of sentinels."""
    M, N = x0.shape
    buf = torch.full((rows, ld), SENTINEL, device="cuda")
    buf[:M, :N] = x0
    return buf


def launch(A, W, x, M, N, K, bias, bn, epi, alpha=1.0):
    ld = x.stride(0)
    gemm_probe.gemm(A, W, M, N, K, bias=bias, resid=x, ldr=ld, out32=x, ld32=ld, force_bn=bn, epi=epi, alpha=alpha)


@pytest.mark.parametrize("K", [192, 64])
@pytest.mark.parametrize("N", [200, 328, 1280])
@pytest.mark.parametrize("bn", [128, 256])
def test_resid_kind_writes_only_inside_bounds(cuda_dev, bn, N, K):
    M, ld, rows = 576, N + 8, 640   # rows: the buffer runs 64 rows past M
    A, W, bias, x0 = operands(M, N, K, 13 * N + bn + K)
    got = pitched(x0, ld, rows)
    assert gemm_probe.plan(A, W, M, N, K, bias=bias, resid=got, ldr=ld, out32=got, ld32=ld, force_bn=bn)[1] == \
        "bias_resid_f32"
    want = got.clone()
    launch(A, W, got, M, N, K, bias, bn, "bias_resid_f32", alpha=0.0625)
    launch(A, W, want, M, N, K, bias, bn, "general", alpha=0.0625)
    torch.cuda.synchronize()
    assert (got[:M, N:] == SENTINEL).all(), "pad columns written"
    assert (got[M:] == SENTINEL).all(), "rows past M written"
    assert not torch.isnan(got).any()
    assert not torch.equal(got[:M, :N], x0)
    assert torch.equal(got, want)


@pytest.mark.parametrize("bn", [128, 256])
def test_resid_kind_vit_shape_back_to_back(cuda_dev, bn):
    M, N, K = 12288, 1280, 1280
    A, W, bias, x0 = operands(M, N, K, bn)
    got, want = x0.clone(), x0.clone()
    for _ in range(2):   # the second launch reads what the first one stored
        launch(A, W, got, M, N, K, bias, bn, "bias_resid_f32")
        launch(A, W, want, M, N, K, bias, bn, "general")
    torch.cuda.synchronize()
    assert torch.equal(got, want)


@pytest.mark.parametrize("bn", [128, 256])
def test_resid_kind_graph_replay(cuda_dev, bn):
    M, N, K = 1536, 1280, 320
    A, W, bias, x0 = operands(M, N, K, 3 + bn)
    x = x0.clone()
    launch(A, W, x, M, N, K, bias, bn, "bias_resid_f32")   # configures the kernel outside the capture
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s), torch.cuda.graph(graph, stream=s):
        launch(A, W, x, M, N, K, bias, bn, "bias_resid_f32")
    want = x0.clone()
    launch(A, W, want, M, N, K, bias, bn, "general")
    for _ in range(2):
        x.copy_(x0)
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(x, want)


def test_non_aliased_residual_takes_the_general_epilogue(cuda_dev):
    M, N, K = 576, 328, 192
    A, W, bias, x0 = operands(M, N, K, 29)
    out = torch.full((M, N), SENTINEL, device="cuda")
    kw = dict(bias=bias, resid=x0, ldr=N, out32=out, ld32=N, force_bn=256)
    assert gemm_probe.plan(A, W, M, N, K, **kw)[1] == "general"
    with pytest.raises(RuntimeError, match="does not fit"):
        gemm_probe.plan(A, W, M, N, K, epi="bias_resid_f32", **kw)
    # the same residual with a pitch other than the output's does not alias it either
    y = pitched(x0, N + 8, M)
    assert gemm_probe.plan(A, W, M, N, K, bias=bias, resid=y, ldr=N + 8, out32=y, ld32=N, force_bn=256)[1] == "general"
    gemm_probe.gemm(A, W, M, N, K, **kw)
    want = x0.clone()
    launch(A, W, want, M, N, K, bias, 256, "general")
    torch.cuda.synchronize()
    assert torch.equal(out, want)

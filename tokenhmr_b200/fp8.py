"""The block-scaled e4m3 quantisation of the FP8 mode (DESIGN.md §2), in torch on any device.

A block of values x gets the smallest power-of-two scale s with amax(|x|) / s <= 448 (s = 1 when amax = 0) and the
codes e4m3(x / s), rounded to nearest even.  s is a power of two, so x / s is exact and the codes are a pure function
of the fp32 input: torch.float8_e4m3fn reproduces the kernels' cvt.rn.satfinite bit for bit (its NaN on overflow is
unreachable because |x / s| <= 448).

  weights      one scale per 128 x 128 block of the [N, K] matrix: scales [ceil(N / 128), K / 128]
  activations  one scale per (row, 128 consecutive columns), k-block-major: scales [K / 128, rows]
"""
from __future__ import annotations

import torch

E4M3_MAX = 448.0
BLOCK = 128


def e4m3_scale(amax: torch.Tensor) -> torch.Tensor:
    """Smallest power of two s with amax / s <= 448, element-wise (1 where amax == 0).  amax = m 2^E with m in
    [0.5, 1): amax <= 448 2^(E-9) iff m <= 0.875 (448 = 0.875 2^9), else amax <= 448 2^(E-8)."""
    amax = amax.float()
    m, E = torch.frexp(amax)
    e = torch.where(m <= 0.875, E - 9, E - 8)
    s = torch.ldexp(torch.ones_like(amax), e)
    return torch.where(amax > 0, s, torch.ones_like(amax))


def quantize_rows(x: torch.Tensor):
    """fp32 [R, K] (K % 128 == 0) -> (codes float8_e4m3fn [R, K], scales fp32 [K / 128, R])."""
    R, K = x.shape
    if K % BLOCK:
        raise ValueError(f"quantize_rows: K={K} is not a multiple of {BLOCK}")
    xb = x.float().reshape(R, K // BLOCK, BLOCK)
    s = e4m3_scale(xb.abs().amax(-1))                                   # [R, K/128]
    codes = (xb / s.unsqueeze(-1)).to(torch.float8_e4m3fn).reshape(R, K)
    return codes, s.t().contiguous()


def quantize_weight_blocks(w: torch.Tensor):
    """fp32 [N, K] (K % 128 == 0) -> (codes float8_e4m3fn [N, K], scales fp32 [ceil(N / 128), K / 128])."""
    N, K = w.shape
    if K % BLOCK:
        raise ValueError(f"quantize_weight_blocks: K={K} is not a multiple of {BLOCK}")
    nb = (N + BLOCK - 1) // BLOCK
    wp = torch.zeros(nb * BLOCK, K, dtype=torch.float32, device=w.device)
    wp[:N] = w.float()
    blocks = wp.reshape(nb, BLOCK, K // BLOCK, BLOCK)
    s = e4m3_scale(blocks.abs().amax(dim=(1, 3)))                       # [nb, K/128]
    codes = (blocks / s[:, None, :, None]).to(torch.float8_e4m3fn).reshape(nb * BLOCK, K)[:N].contiguous()
    return codes, s.contiguous()


def dequantize_rows(codes: torch.Tensor, scales: torch.Tensor) -> torch.Tensor:
    """Inverse of quantize_rows (exact): fp32 [R, K]."""
    R, K = codes.shape
    return (codes.float().reshape(R, K // BLOCK, BLOCK) * scales.t().unsqueeze(-1)).reshape(R, K)


def dequantize_weight_blocks(codes: torch.Tensor, scales: torch.Tensor) -> torch.Tensor:
    """Inverse of quantize_weight_blocks (exact): fp32 [N, K]."""
    N, K = codes.shape
    s = scales.repeat_interleave(BLOCK, 0)[:N].repeat_interleave(BLOCK, 1)
    return codes.float() * s

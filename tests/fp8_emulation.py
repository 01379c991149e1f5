"""CPU emulation of the engine's FP8 mode (DESIGN.md §2) on top of the oracle's fp16-contract restatement.

The ViT's QKV, fc1 and fc2 GEMMs quantise both operands exactly as the contract says (tokenhmr_b200/fp8.py: e4m3 codes
with power-of-two scales per (row, 128 columns) of the activation and per 128 x 128 block of the weight), compute each
128-wide k-block's partial sum of the dequantised operands in fp64 and promote it into an fp32 accumulator, then add
the bias in fp32.  Every other operation follows the oracle's emulate_fp16=True path unchanged."""
from __future__ import annotations

import contextlib

import torch
import torch.nn.functional as F

from oracle import tokenhmr_oracle as O
from tokenhmr_b200 import fp8


def fp8_linear(x: torch.Tensor, w: torch.Tensor, b: torch.Tensor | None) -> torch.Tensor:
    """y = x @ w^T + b under the FP8 contract: x fp32 [..., K], w fp32 [N, K]."""
    shape = x.shape
    x2 = x.reshape(-1, shape[-1]).float()
    qa, sa = fp8.quantize_rows(x2)
    qw, sw = fp8.quantize_weight_blocks(w.float())
    A = fp8.dequantize_rows(qa, sa).double()
    W = fp8.dequantize_weight_blocks(qw, sw).double()
    acc = torch.zeros(A.shape[0], W.shape[0], dtype=torch.float32)
    for k0 in range(0, A.shape[1], fp8.BLOCK):
        acc = acc + (A[:, k0:k0 + fp8.BLOCK] @ W[:, k0:k0 + fp8.BLOCK].t()).float()
    if b is not None:
        acc = acc + b.float()
    return acc.reshape(*shape[:-1], W.shape[0])


class Fp8Numerics(O.Numerics):
    """The oracle's fp16 contract, except for the linears whose weight is one of `fp8_weights` (by identity)."""

    def __init__(self, fp8_weights):
        super().__init__(emulate_fp16=True)
        self.fp8_ids = {id(t) for t in fp8_weights}

    def linear(self, x, w, b=None):
        if id(w) in self.fp8_ids:
            return fp8_linear(x, w, b)
        return F.linear(self.q(x), self.q(w), b)


def vit_fp8_weights(sd, cfg):
    return [sd[f"backbone.blocks.{i}.{n}.weight"] for i in range(cfg.vit_depth)
            for n in ("attn.qkv", "mlp.fc1", "mlp.fc2")]


@contextlib.contextmanager
def _numerics(factory):
    saved = O.Numerics
    O.Numerics = factory
    try:
        yield
    finally:
        O.Numerics = saved


def forward_fp8(sd, smpl, img, cfg, return_intermediates: bool = False):
    """oracle.tokenhmr_oracle.forward with the FP8 mode's numerics (emulate_fp16=True everywhere else)."""
    weights = vit_fp8_weights(sd, cfg)
    with _numerics(lambda emulate_fp16: Fp8Numerics(weights)):
        return O.forward(sd, smpl, img, cfg, emulate_fp16=True, return_intermediates=return_intermediates)

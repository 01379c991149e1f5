"""Writes tests/golden/regression_head_grads.npz: the LIVE reference SMPLTransformerDecoderHead (heads/smpl_head.py)
in float64 with autograd, on seeded features (B = 4) and seeded upstream gradients for the 24 rotations, betas and
pred_cam, with the synthetic regression state dict of tiny_config (the release decoder).

    TOKENHMR_REFERENCE=<checkout> python scripts/regression_grads_golden.py

The file holds the outputs and, for the gradient G of every parameter, four projections <G, R_k> on seeded
standard-normal R_k (projection_matrix below) and the Frobenius norm; for the vector parameters (LayerNorms, biases,
pos_embedding, to_token_embedding.*) also every SAMPLE-th element in full.  So it stays small (~0.1 MB).  The reference leaves
to_token_embedding.weight without a gradient (its input is zero); it is stored as zeros.
"""
from __future__ import annotations

import sys
import zlib
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))

W_SEED, FEAT_SEED, UP_SEED, B, NPROJ, SAMPLE = 1234, 4, 5, 4, 4, 8


def is_matrix(shape) -> bool:
    """The weight matrices (two dimensions above 1); everything else is a vector parameter."""
    return sum(int(d) > 1 for d in shape) > 1


def sampled(g: torch.Tensor) -> torch.Tensor:
    return g.reshape(-1)[::SAMPLE]


def projection_matrix(name: str, k: int, shape) -> torch.Tensor:
    g = torch.Generator().manual_seed(zlib.crc32(f"{name}/{k}".encode()))
    return torch.randn(*shape, generator=g, dtype=torch.float64)


def inputs(cfg):
    """(features (B,1280,16,12), upstream rotations (B,24,3,3), betas (B,10), cam (B,3)), float64."""
    g = torch.Generator().manual_seed(FEAT_SEED)
    feats = torch.randn(B, cfg.vit_dim, cfg.grid_h, cfg.grid_w, generator=g, dtype=torch.float64)
    g = torch.Generator().manual_seed(UP_SEED)
    up = (torch.randn(B, 24, 3, 3, generator=g, dtype=torch.float64),
          torch.randn(B, 10, generator=g, dtype=torch.float64), torch.randn(B, 3, generator=g, dtype=torch.float64))
    return feats, up


def main() -> None:
    from oracle import ref_import
    from oracle import regression_oracle as R
    from tokenhmr_b200 import synth
    from tokenhmr_b200.config import tiny_config
    cfg = tiny_config(vit_depth=2, head="transformer_decoder")
    sd = synth.make_state_dict(cfg, W_SEED)
    head = R.build_regression_head(ref_import.load_modules(), sd, cfg).double()
    feats, up = inputs(cfg)
    torch.set_default_dtype(torch.float64)      # the head builds its zero query with torch.zeros (smpl_head.py:73)
    params, cam, _ = head(feats)
    torch.set_default_dtype(torch.float32)
    rot = torch.cat([params["global_orient"], params["body_pose"]], 1)
    loss = (rot * up[0]).sum() + (params["betas"] * up[1]).sum() + (cam * up[2]).sum()
    named = [(n, p) for n, p in head.named_parameters()]
    grads = torch.autograd.grad(loss, [p for _, p in named], allow_unused=True)
    arrays = {"meta": np.array([W_SEED, FEAT_SEED, UP_SEED, B, NPROJ, SAMPLE]), "rotmats": rot.detach().numpy(),
              "betas": params["betas"].detach().numpy(), "cam": cam.detach().numpy()}
    for (name, p), g in zip(named, grads):
        g = torch.zeros_like(p) if g is None else g.detach()
        arrays["proj/" + name] = np.array([(g * projection_matrix(name, k, g.shape)).sum().item()
                                           for k in range(NPROJ)])
        arrays["norm/" + name] = np.array(g.norm().item())
        if not is_matrix(g.shape):
            arrays["grad/" + name] = sampled(g).numpy()
    out = ROOT / "tests" / "golden" / "regression_head_grads.npz"
    np.savez_compressed(out, **arrays)
    print("wrote", out)


if __name__ == "__main__":
    main()

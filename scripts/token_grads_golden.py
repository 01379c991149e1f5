"""Writes tests/golden/token_head_grads.npz: the LIVE reference SMPLTokenDecoderHead (heads/token_head.py) in float64 with
autograd, on seeded features (B = 4) and seeded upstream gradients for the 24 rotations, betas, pred_cam and
cls_logits_softmax, with the synthetic token-head state dict of tiny_config (the release decoder, classifier and
tokenizer).

    TOKENHMR_REFERENCE=<checkout> python scripts/token_grads_golden.py

The synthetic class_pred_layer has gain 20, so its softmax is peaky and carries little gradient back to the
classifier.  The file therefore holds two sets, under the prefixes "cls1/" (the weights as made) and "cls005/"
(class_pred_layer.weight scaled by CLS_SCALE), each with the outputs and, for the gradient G of every trainable
parameter, four projections <G, R_k> and the Frobenius norm (regression_grads_golden's format); for the vector
parameters also every SAMPLE-th element (for the second set, of the
classifier's and read-outs' vectors only).  cls_logits_softmax is stored the same way (projections, norm, every
PROBS_SAMPLE-th element), so the file stays small (~0.2 MB; each set's summaries are stacked into a few arrays).  The tokenizer is frozen (the reference reaches it
through a Proxy, not as a submodule): it is converted to float64 on its own and has no gradient.
"""
from __future__ import annotations

import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))

from scripts.regression_grads_golden import is_matrix, projection_matrix, sampled  # noqa: E402

W_SEED, FEAT_SEED, UP_SEED, B, NPROJ, SAMPLE, PROBS_SAMPLE = 1234, 14, 15, 4, 4, 8, 509
CLS_SCALE = 0.05
SETS = (("cls1/", 1.0), ("cls005/", CLS_SCALE))


def state_dict(cfg, scale: float):
    """The tiny_config token-head state dict with class_pred_layer.weight scaled by `scale`."""
    from tokenhmr_b200 import synth
    sd = synth.make_state_dict(cfg, W_SEED)
    sd["smpl_head.decpose.class_pred_layer.weight"] = sd["smpl_head.decpose.class_pred_layer.weight"] * scale
    return sd


def inputs(cfg):
    """(features (B,1280,16,12), upstream rotations (B,24,3,3), betas (B,10), cam (B,3), cls_logits_softmax
    (B,160,2048)), float64."""
    g = torch.Generator().manual_seed(FEAT_SEED)
    feats = torch.randn(B, cfg.vit_dim, cfg.grid_h, cfg.grid_w, generator=g, dtype=torch.float64)
    g = torch.Generator().manual_seed(UP_SEED)
    up = (torch.randn(B, 24, 3, 3, generator=g, dtype=torch.float64),
          torch.randn(B, 10, generator=g, dtype=torch.float64), torch.randn(B, 3, generator=g, dtype=torch.float64),
          torch.randn(B, cfg.token_num, cfg.token_class_num, generator=g, dtype=torch.float64))
    return feats, up


def loss_of(rot, betas, cam, probs, up):
    return (rot * up[0]).sum() + (betas * up[1]).sum() + (cam * up[2]).sum() + (probs * up[3]).sum()


def has_samples(key: str) -> bool:
    """Sampled elements are stored for every vector of the first set, and for the second set's classifier and
    read-outs only (its decoder is the first set's, reached through a different softmax)."""
    return key.startswith(SETS[0][0]) or not key.startswith(SETS[1][0] + "transformer.")


def summarise(tab: dict, key: str, g: torch.Tensor, every: int) -> None:
    """Projections, norm and (for vectors, or with every != SAMPLE) sampled elements of g under key, into the set's
    table."""
    tab["names"].append(key)
    tab["proj"].append([(g * projection_matrix(key, k, g.shape)).sum().item() for k in range(NPROJ)])
    tab["norm"].append(g.norm().item())
    if has_samples(key) and (every != SAMPLE or not is_matrix(g.shape)):
        v = g.reshape(-1)[::every].numpy() if every != SAMPLE else sampled(g).numpy()
        tab["sampled_names"].append(key)
        tab["sampled"].append(v)


def table(arrays: dict, tag: str) -> dict:
    """{key: (projections, norm, sampled elements or None)} of one set, from the stacked arrays."""
    names, proj, norm = arrays[tag + "names"], arrays[tag + "proj"], arrays[tag + "norm"]
    cut = np.cumsum(arrays[tag + "sampled_len"])[:-1]
    samples = dict(zip(arrays[tag + "sampled_names"], np.split(arrays[tag + "sampled"], cut)))
    return {str(n): (proj[i], norm[i], samples.get(n)) for i, n in enumerate(names)}


def main() -> None:
    from oracle import ref_import
    from tokenhmr_b200.config import tiny_config
    cfg = tiny_config(vit_depth=2)
    ns = ref_import.load_modules()
    feats, up = inputs(cfg)
    arrays = {"meta": np.array([W_SEED, FEAT_SEED, UP_SEED, B, NPROJ, SAMPLE, PROBS_SAMPLE]),
              "cls_scale": np.array(CLS_SCALE)}
    for tag, scale in SETS:
        head = ref_import.build_head(ns, state_dict(cfg, scale), cfg).double()
        tokenizer = head.decpose.tokenize.__self__          # the Proxy: its tokenizer is not a submodule
        tokenizer.tokenizer = tokenizer.tokenizer.double()
        torch.set_default_dtype(torch.float64)              # the head builds its zero query with torch.zeros
        params, cam, lst = head(feats)
        torch.set_default_dtype(torch.float32)
        rot = torch.cat([params["global_orient"], params["body_pose"]], 1)
        probs = lst["cls_logits_softmax"]
        loss = loss_of(rot, params["betas"], cam, probs, up)
        named = [(n, p) for n, p in head.named_parameters()]
        grads = torch.autograd.grad(loss, [p for _, p in named], allow_unused=True)
        arrays[tag + "rotmats"] = rot.detach().numpy()
        arrays[tag + "betas"] = params["betas"].detach().numpy()
        arrays[tag + "cam"] = cam.detach().numpy()
        tab = {"names": [], "proj": [], "norm": [], "sampled_names": [], "sampled": []}
        summarise(tab, tag + "cls_logits_softmax", probs.detach(), PROBS_SAMPLE)
        for (name, p), g in zip(named, grads):
            g = torch.zeros_like(p) if g is None else g.detach()
            summarise(tab, tag + name, g, SAMPLE)
        arrays[tag + "names"] = np.array(tab["names"])
        arrays[tag + "proj"] = np.array(tab["proj"])
        arrays[tag + "norm"] = np.array(tab["norm"])
        arrays[tag + "sampled_names"] = np.array(tab["sampled_names"])
        arrays[tag + "sampled_len"] = np.array([len(v) for v in tab["sampled"]])
        arrays[tag + "sampled"] = np.concatenate(tab["sampled"])
    out = ROOT / "tests" / "golden" / "token_head_grads.npz"
    np.savez_compressed(out, **arrays)
    print("wrote", out, out.stat().st_size, "bytes")


if __name__ == "__main__":
    main()

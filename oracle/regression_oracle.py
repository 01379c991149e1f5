"""HMR 2.0's regression head (MODEL.SMPL_HEAD.TYPE: transformer_decoder) for the oracle.  TEST INFRASTRUCTURE ONLY.

  * build_regression_head: the LIVE reference SMPLTransformerDecoderHead (heads/smpl_head.py:9-50), built by its own
    constructor from a state dict, with the same duck-typed cfg and temporary MEAN_PARAMS .npz as
    ref_import.build_head.
  * regression_head_forward / forward: the plain-PyTorch restatement of SMPLTransformerDecoderHead.forward and of
    TokenHMR.forward_step with that head (tokenhmr.py:135-188: no cls_logits_softmax, :157-158), under the same
    Numerics switch (fp32, or the engine's fp16-operand emulation) as tokenhmr_oracle.head_forward.
  * main: writes tests/golden/forward_regression_*.npz from the live reference head:

    TOKENHMR_REFERENCE=<checkout> python -m oracle.regression_oracle            # tiny (depth-2, B = 2)
    TOKENHMR_REFERENCE=<checkout> python -m oracle.regression_oracle --release  # also ViT-H depth 32, B = 64
"""
from __future__ import annotations

import argparse
import contextlib
import importlib
import io
import os
import tempfile
from typing import Dict

import numpy as np
import torch

from . import ref_import, smpl_oracle
from . import tokenhmr_oracle as O

Tensor = torch.Tensor
W_SEED, SMPL_SEED, IMG_SEED = 1234, 3, 0


def build_regression_head(ns, sd: Dict[str, Tensor], cfg):
    """SMPLTransformerDecoderHead (smpl_head.py:14-50) from the reference's own constructor, loaded with the
    smpl_head.* entries of `sd` (strict: no missing and no unused key), eval mode."""
    mod = importlib.import_module("lib.models.heads.smpl_head")
    with tempfile.TemporaryDirectory() as td:
        npz = os.path.join(td, "smpl_mean_params.npz")
        np.savez(npz, pose=sd["smpl_head.init_body_pose"][0].numpy(), shape=sd["smpl_head.init_betas"][0].numpy(),
                 cam=sd["smpl_head.init_cam"][0].numpy())
        rcfg = ref_import._Cfg({
            "MODEL": {"SMPL_HEAD": {"TYPE": "transformer_decoder", "JOINT_REP": "6d", "TRANSFORMER_INPUT": "zero",
                                    "IEF_ITERS": 1,
                                    "TRANSFORMER_DECODER": {"depth": cfg.dec_depth, "heads": cfg.dec_heads,
                                                            "mlp_dim": cfg.dec_mlp_dim,
                                                            "dim_head": cfg.dec_dim_head, "dropout": 0.0,
                                                            "emb_dropout": 0.0, "norm": "layer",
                                                            "context_dim": cfg.vit_dim}}},
            "SMPL": {"NUM_BODY_JOINTS": cfg.num_joints - 1, "MEAN_PARAMS": npz},
        })
        with contextlib.redirect_stdout(io.StringIO()):
            head = mod.SMPLTransformerDecoderHead(rcfg)
    own = {k[len("smpl_head."):]: v for k, v in sd.items() if k.startswith("smpl_head.")}
    head.load_state_dict(own, strict=True)
    head.eval()
    return head


def regression_head_forward(sd: Dict[str, Tensor], context: Tensor, cfg, nm: O.Numerics, prefix: str = "smpl_head."):
    """SMPLTransformerDecoderHead.forward with IEF_ITERS=1, TRANSFORMER_INPUT='zero', JOINT_REP='6d'
    (smpl_head.py:52-105).  context (B,192,1280) -> (pred_smpl_params, pred_cam, aux)."""
    g = lambda n: sd[prefix + n]
    B = context.shape[0]
    tok = O.decoder_forward(sd, context, cfg, nm, prefix + "transformer.")                        # :77-79
    pred_body_pose = nm.linear(tok, g("decpose.weight"), g("decpose.bias")) + g("init_body_pose")  # :82
    pred_betas = nm.linear(tok, g("decshape.weight"), g("decshape.bias")) + g("init_betas")        # :83
    pred_cam = nm.linear(tok, g("deccam.weight"), g("deccam.bias")) + g("init_cam")                # :84
    rotmats = O.rot6d_to_rotmat(pred_body_pose).view(B, cfg.num_joints, 3, 3)                      # :89-99
    return {"global_orient": rotmats[:, [0]], "body_pose": rotmats[:, 1:], "betas": pred_betas}, pred_cam, \
        {"token_out": tok, "pred_body_pose_6d": pred_body_pose}


def _forward_tail(ns_projection, smpl, params, pred_cam, cfg, B: int, dtype) -> Dict[str, Tensor]:
    """forward_step after the head (tokenhmr.py:159-187), without cls_logits_softmax (:157-158)."""
    out: Dict[str, Tensor] = {"pred_cam": pred_cam, "pred_smpl_params": {k: v.clone() for k, v in params.items()}}
    focal = cfg.focal_length * torch.ones(B, 2, dtype=dtype)                                          # :165
    cam_t = torch.stack([pred_cam[:, 1], pred_cam[:, 2],
                         2 * focal[:, 0] / (cfg.image_size * pred_cam[:, 0] + 1e-9)], dim=-1)         # :166-168
    out["pred_cam_t"], out["focal_length"] = cam_t, focal
    verts, joints = smpl_oracle.smpl_forward(smpl, params["global_orient"], params["body_pose"], params["betas"])
    out["pred_keypoints_3d"] = joints.reshape(B, -1, 3)
    out["pred_vertices"] = verts.reshape(B, -1, 3)
    out["pred_keypoints_2d"] = ns_projection(joints, cam_t, focal / cfg.image_size)                  # :183-187
    return out


def forward(sd: Dict[str, Tensor], smpl: Dict[str, Tensor], img: Tensor, cfg, emulate_fp16: bool = False,
            return_intermediates: bool = False) -> Dict[str, Tensor]:
    """TokenHMR.forward(batch) for either head: cfg.head 'token' is tokenhmr_oracle.forward, 'transformer_decoder'
    the regression head's forward_step."""
    if cfg.head == "token":
        return O.forward(sd, smpl, img, cfg, emulate_fp16=emulate_fp16, return_intermediates=return_intermediates)
    nm = O.Numerics(emulate_fp16)
    feats = O.vit_forward(sd, img, cfg, nm)
    params, pred_cam, aux = regression_head_forward(sd, feats, cfg, nm)
    out = _forward_tail(O.perspective_projection, smpl, params, pred_cam, cfg, img.shape[0], img.dtype)
    if return_intermediates:
        out["_vit_tokens"], out["_token_out"], out["_pred_body_pose_6d"] = feats, aux["token_out"], aux["pred_body_pose_6d"]
    return out


def reference_forward(ns, backbone, head, smpl, img, cfg) -> Dict[str, Tensor]:
    """forward_step with TYPE transformer_decoder around the LIVE reference backbone, head and projection; only the
    smplx call goes to the restatement in smpl_oracle (as in ref_import.reference_forward)."""
    with torch.no_grad():
        feats = backbone(img)
        params, pred_cam, _ = head(feats)
        proj = lambda j, t, f: ns.geometry.perspective_projection(j, translation=t, focal_length=f)
        out = _forward_tail(proj, smpl, params, pred_cam, cfg, img.shape[0], img.dtype)
        out["_vit_tokens"] = feats.flatten(2).transpose(1, 2).contiguous()
    return out


def write_golden(ns, cfg, batch: int, name: str, img_seed: int = IMG_SEED, vert_stride: int = 1) -> None:
    from pathlib import Path
    from tokenhmr_b200 import synth
    golden = Path(__file__).resolve().parent.parent / "tests" / "golden"
    sd, smpl = synth.make_state_dict(cfg, W_SEED), synth.make_smpl(cfg, SMPL_SEED)
    img = synth.make_images(batch, cfg, img_seed)
    out = reference_forward(ns, ref_import.build_backbone(ns, sd, cfg), build_regression_head(ns, sd, cfg), smpl, img,
                            cfg)
    p = out["pred_smpl_params"]
    arrays = dict(meta=np.array([W_SEED, SMPL_SEED, img_seed, batch, cfg.vit_depth, cfg.num_verts, vert_stride]),
                  pred_cam=out["pred_cam"].numpy(), pred_cam_t=out["pred_cam_t"].numpy(),
                  focal_length=out["focal_length"].numpy(), global_orient=p["global_orient"].numpy(),
                  body_pose=p["body_pose"].numpy(), betas=p["betas"].numpy(),
                  pred_keypoints_3d=out["pred_keypoints_3d"].numpy(),
                  pred_vertices_sub=out["pred_vertices"][:, ::vert_stride].numpy(),
                  pred_keypoints_2d=out["pred_keypoints_2d"].numpy())
    if vert_stride == 1:
        arrays["vit_tokens_sub"] = out["_vit_tokens"][:, ::8].numpy()
    np.savez_compressed(golden / name, **arrays)
    print("wrote", name)


def main() -> None:
    from tokenhmr_b200.config import TokenHMRConfig, tiny_config
    ap = argparse.ArgumentParser()
    ap.add_argument("--release", action="store_true", help="also the ViT-H depth-32 forward at B = 64 (~3 GB RAM)")
    args = ap.parse_args()
    ns = ref_import.load_modules()
    write_golden(ns, tiny_config(vit_depth=2, head="transformer_decoder"), 2, "forward_regression_tiny_d2.npz")
    if args.release:
        write_golden(ns, TokenHMRConfig(head="transformer_decoder"), 64, "forward_regression_release_d32.npz",
                     img_seed=5, vert_stride=16)


if __name__ == "__main__":
    main()

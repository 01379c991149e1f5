"""TokenHMR's training and validation loss on the GPU, and the differentiable tail of forward_step.

    crit = TokenHMRLoss(cfg)                          # cfg.MODEL.LOOSE_SUP / LOOSE_WEIGHT, cfg.LOSS_WEIGHTS
    out = differentiable_tail(model.smpl, pred_smpl_params, pred_cam, focal_length, image_size)
    loss = crit(batch, out, train=True)               # TokenHMR.compute_loss: sets out['losses']
    loss.backward()                                   # -> rotations, betas and pred_cam

The loss is one CUDA call (thmr_tokenhmr_loss: per-sample terms and their gradients in one pass, then a fixed-order
batch sum), so a step has no host synchronisation and can be captured in a CUDA graph.  Unlike the reference it never
writes into the caller's batch (the reference masks gt_keypoints_2d's confidence and has_smpl_params['betas'] in place;
its returned values do not depend on that).
"""
from __future__ import annotations

import ctypes
from typing import Dict, Optional

import torch

from . import _lib
from ._lib import check, lib
from .ops import SMPLModel, _req, _stream, camera_tail

# tokenhmr.py:226: the datasets whose 3-D supervision TALS always trusts
VALID_3D_DATASETS = ("H36M-TRAIN-WMASK", "BEDLAM")
LOSS_TERMS = ("loss", "loss_keypoints_2d", "loss_keypoints_3d", "loss_global_orient", "loss_body_pose", "loss_betas")
TALS_JOINTS = 44


class TokenHMRLoss:
    """TokenHMR.compute_loss (tokenhmr.py:190-277) on the GPU.  The settings come from `model_cfg` (a CfgNode or a dict
    with MODEL.LOOSE_SUP, MODEL.LOOSE_WEIGHT and LOSS_WEIGHTS) unless given as keywords."""

    def __init__(self, model_cfg=None, *, loose_sup: Optional[bool] = None, loose_weight: Optional[float] = None,
                 loss_weights: Optional[Dict[str, float]] = None, pelvis_id: int = 25 + 14):
        if model_cfg is not None:
            model = model_cfg["MODEL"]          # a yacs CfgNode is a dict
            loose_sup = model["LOOSE_SUP"] if loose_sup is None else loose_sup
            loose_weight = model["LOOSE_WEIGHT"] if loose_weight is None else loose_weight
            loss_weights = model_cfg["LOSS_WEIGHTS"] if loss_weights is None else loss_weights
        if loose_sup is None or loss_weights is None or (loose_sup and loose_weight is None):
            raise _lib.ThmrError("TokenHMRLoss: give model_cfg, or loose_sup, loose_weight and loss_weights")
        self.loose_sup = bool(loose_sup)
        self.loose_weight = float(loose_weight) if loose_weight is not None else 0.0
        self.weights = {k: float(loss_weights[k])
                        for k in ("KEYPOINTS_2D", "KEYPOINTS_3D", "GLOBAL_ORIENT", "BODY_POSE", "BETAS")}
        self.pelvis_id = int(pelvis_id)

    def __call__(self, batch: Dict, output: Dict, train: bool = True) -> torch.Tensor:
        """compute_loss(batch, output, train): returns the scalar loss and sets output['losses'] (the six detached
        terms).  batch['dataset'] (read by the TALS branch only) is the list of dataset names, or a (B,) tensor that is
        1 for an H36M-TRAIN-WMASK or BEDLAM sample and 0 otherwise (no host-to-device copy: graph-capturable)."""
        tals = self.loose_sup and train
        params = output["pred_smpl_params"]
        kp2d, kp3d = output["pred_keypoints_2d"], output["pred_keypoints_3d"]
        B = params["body_pose"].shape[0]
        rot = torch.cat([params["global_orient"].reshape(B, -1, 3, 3), params["body_pose"].reshape(B, -1, 3, 3)], 1)
        betas = params["betas"].reshape(B, -1)
        valid_3d = self._valid_3d(batch["dataset"], B, kp2d.device) if tals else None
        terms = _LossFn.apply(self, tals, batch, valid_3d, kp2d, kp3d, rot, betas)
        output["losses"] = dict(zip(LOSS_TERMS, terms.detach().unbind(0)))
        return terms[0]

    @staticmethod
    def _valid_3d(dataset, B: int, device) -> torch.Tensor:
        if isinstance(dataset, torch.Tensor):
            return dataset
        if len(dataset) != B:
            raise _lib.ThmrError(f"TokenHMRLoss: batch['dataset'] has {len(dataset)} names for {B} samples")
        v = torch.tensor([float(n in VALID_3D_DATASETS) for n in dataset], dtype=torch.float32)
        return v.pin_memory().to(device, non_blocking=True)

    def _run(self, tals: bool, batch: Dict, valid_3d, kp2d, kp3d, rot, betas, grads: bool):
        kp2d, kp3d = _req(kp2d, torch.float32, "pred_keypoints_2d"), _req(kp3d, torch.float32, "pred_keypoints_3d")
        rot, betas = _req(rot, torch.float32, "pred rotations"), _req(betas, torch.float32, "pred betas")
        B, J, nb = kp2d.shape[0], kp2d.shape[1], betas.shape[1]
        f32 = lambda t, name: _req(t.to(torch.float32), torch.float32, name)
        flag = lambda t, name: _req(t.to(torch.bool), torch.bool, name)
        gt2, gt3 = f32(batch["keypoints_2d"], "keypoints_2d"), f32(batch["keypoints_3d"], "keypoints_3d")
        gt, has, aa = batch["smpl_params"], batch["has_smpl_params"], batch["smpl_params_is_axis_angle"]
        g_go, g_bp = f32(gt["global_orient"], "global_orient").reshape(B, -1), f32(gt["body_pose"], "body_pose").reshape(B, -1)
        g_be = f32(gt["betas"], "betas").reshape(B, -1)
        h = {k: f32(has[k], f"has_smpl_params[{k}]").reshape(-1) for k in ("global_orient", "body_pose", "betas")}
        a = {k: flag(aa[k], f"smpl_params_is_axis_angle[{k}]").reshape(-1) for k in ("global_orient", "body_pose", "betas")}
        shapes_ok = (kp2d.shape == (B, J, 2) and kp3d.shape == (B, J, 3) and gt2.shape == (B, J, 3)
                     and gt3.shape == (B, J, 4) and rot.shape == (B, 24, 3, 3) and 1 <= nb <= 10
                     and g_go.shape == (B, 3) and g_bp.shape == (B, 69) and g_be.shape == (B, nb)
                     and all(t.shape == (B,) for t in (*h.values(), *a.values())))
        if not shapes_ok:
            raise _lib.ThmrError(
                f"TokenHMRLoss: shapes do not match: pred keypoints_2d {tuple(kp2d.shape)}, keypoints_3d "
                f"{tuple(kp3d.shape)}, rotations {tuple(rot.shape)}, betas {tuple(betas.shape)}; GT keypoints_2d "
                f"{tuple(gt2.shape)}, keypoints_3d {tuple(gt3.shape)}, global_orient {tuple(g_go.shape)}, body_pose "
                f"{tuple(g_bp.shape)} (axis-angle), betas {tuple(g_be.shape)}")
        if tals and J != TALS_JOINTS:
            raise _lib.ThmrError(f"TokenHMRLoss: the TALS branch needs {TALS_JOINTS} keypoints (the size of the "
                                 f"reference's kp2D_err_valid_thresh), got {J}")
        if tals:
            valid_3d = f32(valid_3d, "valid_3d").reshape(-1)
            if valid_3d.shape != (B,):
                raise _lib.ThmrError(f"TokenHMRLoss: valid_3d {tuple(valid_3d.shape)} for {B} samples")
        dev = kp2d.device
        terms = torch.empty(6, device=dev)
        g = [torch.empty_like(t) for t in (kp2d, kp3d, rot, betas)] if grads else [None] * 4
        w = self.weights
        p = lambda t: 0 if t is None else t.data_ptr()
        d = _lib.LossDesc(B, J, nb, int(tals), self.pelvis_id, self.loose_weight, w["KEYPOINTS_2D"], w["KEYPOINTS_3D"],
                          w["GLOBAL_ORIENT"], w["BODY_POSE"], w["BETAS"],
                          kp2d.data_ptr(), kp3d.data_ptr(), rot.data_ptr(), betas.data_ptr(), gt2.data_ptr(),
                          gt3.data_ptr(), g_go.data_ptr(), g_bp.data_ptr(), g_be.data_ptr(),
                          h["global_orient"].data_ptr(), h["body_pose"].data_ptr(), h["betas"].data_ptr(),
                          p(valid_3d), a["global_orient"].data_ptr(), a["body_pose"].data_ptr(),
                          a["betas"].data_ptr(), terms.data_ptr(), *(p(t) for t in g))
        ws = torch.empty(lib().thmr_tokenhmr_loss_workspace_bytes(B), device=dev, dtype=torch.uint8)
        check(lib().thmr_tokenhmr_loss(ctypes.byref(d), ws.data_ptr(), _stream()))
        return terms, g


class _LossFn(torch.autograd.Function):
    """The six terms (loss first).  Only the loss is differentiable, as in the reference, whose other terms are
    detached: its gradient for a unit upstream comes from the same kernel pass and is scaled in the backward."""

    @staticmethod
    def forward(ctx, crit: TokenHMRLoss, tals: bool, batch: Dict, valid_3d, kp2d, kp3d, rot, betas):
        ctx.set_materialize_grads(False)
        grads = any(ctx.needs_input_grad[4:])
        terms, g = crit._run(tals, batch, valid_3d, kp2d, kp3d, rot, betas, grads)
        if grads:
            ctx.save_for_backward(*g)
        return terms

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad_terms):
        if grad_terms is None:
            return (None,) * 8
        grad_loss = grad_terms[0]
        g = [t * grad_loss if need else None for t, need in zip(ctx.saved_tensors, ctx.needs_input_grad[4:])]
        return (None, None, None, None, *g)


def differentiable_tail(smpl, pred_smpl_params: Dict[str, torch.Tensor], pred_cam: torch.Tensor,
                        focal_length: float, image_size: float) -> Dict[str, torch.Tensor]:
    """The tail of forward_step (tokenhmr.py:162-187) after the head: pred_smpl_params (global_orient (B,1,3,3),
    body_pose (B,23,3,3), betas (B,10)) and pred_cam (B,3) -> pred_cam_t, focal_length, pred_keypoints_3d,
    pred_vertices, pred_keypoints_2d.  `smpl` is model.smpl or an ops.SMPLModel.  focal_length and image_size are the
    model's EXTRA.FOCAL_LENGTH and MODEL.IMAGE_SIZE (model.cfg.focal_length and model.cfg.image_size of an engine);
    they are required because the body model does not carry them.  Differentiable to the rotations,
    betas and pred_cam: the body model's CUDA backward chained with the camera tail's (ops.camera_tail)."""
    model = getattr(smpl, "_model", smpl)
    if not isinstance(model, SMPLModel):
        raise _lib.ThmrError("differentiable_tail: smpl must be model.smpl or a tokenhmr_b200.ops.SMPLModel")
    B = pred_cam.shape[0]
    verts, joints = model.forward(pred_smpl_params["global_orient"].reshape(B, -1, 3, 3),
                                  pred_smpl_params["body_pose"].reshape(B, -1, 3, 3),
                                  pred_smpl_params["betas"].reshape(B, -1))
    cam_t, focal, kp2d = camera_tail(joints, pred_cam, focal_length, image_size)
    return {"pred_cam_t": cam_t, "focal_length": focal, "pred_keypoints_3d": joints, "pred_vertices": verts,
            "pred_keypoints_2d": kp2d}

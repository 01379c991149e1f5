"""SMPLify-inverse: refine SMPL predictions against 2D keypoints while pushing the 3D joints away from given ones
(tokenhmr/lib/utils/smplify_invert.py:32-156).  Same constructor, call arguments, return tuple and loop semantics as the
reference's SMPLifyInv.

The optimiser loop stays in PyTorch, as in the reference.  On the GPU the body model is the engine's: pass `model.smpl`
(TokenHMREngine) and the forward and backward of every iteration run in libtokenhmr_b200.so (thmr_smpl_forward /
thmr_smpl_backward).  Any callable with the reference SMPL wrapper's signature works, e.g. an fp64 CPU body model:

    fit = SMPLifyInv(model.smpl, step_size=1e-3, num_iters=100)
    verts, joints, pj2d, go, bp, betas, cam_t, reproj = fit(go, bp, betas, cam_t, focal, kp2d, kp3d)

FusedSMPLifyInv takes the same arguments with the engine's body model and runs the whole loop, Adam included, on the
GPU as one call (thmr_smplify_inv).
"""
from __future__ import annotations

from typing import List, Tuple

import torch


def perspective_projection(points: torch.Tensor, translation: torch.Tensor, focal_length: torch.Tensor) -> torch.Tensor:
    """tokenhmr/lib/utils/geometry.py:86-124 with no rotation and the principal point at 0: (B,N,3) -> (B,N,2),
    f * (p + t)_xy / (p + t)_z per axis."""
    p = points + translation.unsqueeze(1)
    return focal_length.unsqueeze(1) * (p[..., :2] / p[..., 2:])


def camera_fitting_loss(model_joints: torch.Tensor, pred_cam_t: torch.Tensor, focal_length: torch.Tensor,
                        joints_2d: torch.Tensor) -> torch.Tensor:
    """Mean over the batch of the summed (unweighted) L2 reprojection error, at focal_length / 256
    (smplify_invert.py:17-29)."""
    projected = perspective_projection(model_joints, pred_cam_t, focal_length / 256)
    return torch.sqrt(((joints_2d - projected) ** 2).sum(-1)).sum(1).mean()


class SMPLifyInv:
    """Single-stage SMPLify-inverse: Adam over body_pose, global_orient and pred_cam_t (betas fixed) on
    loss = 4 fit2D - mean(push3D) / 2 + margin, where fit2D is camera_fitting_loss and push3D the per-sample summed
    distance of the model's joints to gt_keypoints_3d.  The loop stops before the step at the first iteration where
    loss < loss_thresh_f3d and fit2D < loss_thresh_f2d.

    After a call, `history` holds one (loss, fit2D, mean push3D) triple of detached 0-d tensors per iteration run."""

    def __init__(self, smpl_model, step_size: float = 1e-3, num_iters: int = 100, margin: float = 20,
                 loss_thresh_f2d: float = 1, loss_thresh_f3d: float = 0, device=torch.device("cuda")):
        self.smpl = smpl_model
        self.step_size = step_size
        self.num_iters = num_iters
        self.margin = margin
        self.loss_thresh_f2d = loss_thresh_f2d
        self.loss_thresh_f3d = loss_thresh_f3d
        self.device = device
        self.history: List[Tuple[torch.Tensor, torch.Tensor, torch.Tensor]] = []

    def __call__(self, global_orient: torch.Tensor, body_pose: torch.Tensor, betas: torch.Tensor,
                 pred_cam_t: torch.Tensor, focal_length: torch.Tensor, gt_keypoints_2d: torch.Tensor,
                 gt_keypoints_3d: torch.Tensor):
        """global_orient / body_pose: the body model's pose input (rotation matrices for the SMPL wrapper), betas,
        pred_cam_t (B,3), focal_length (B,2), gt_keypoints_2d (B,J,3) with a confidence column that is read but not
        used (as in the reference), gt_keypoints_3d (B,J,3).  body_pose, global_orient and pred_cam_t are optimised in
        place (they must be leaf tensors).  Returns (vertices, joints, pj2ds, global_orient, body_pose, betas,
        pred_cam_t, reprojection_loss)."""
        joints_2d = gt_keypoints_2d[:, :, :2]
        _ = gt_keypoints_2d[:, :, -1]   # confidences: unused by the reference's loss
        for t, flag in ((body_pose, True), (betas, False), (global_orient, True), (pred_cam_t, True)):
            t.requires_grad = flag
        opt = torch.optim.Adam([body_pose, global_orient, pred_cam_t], lr=self.step_size, betas=(0.9, 0.999))
        self.history = []
        for _ in range(self.num_iters):
            joints = self.smpl(global_orient=global_orient, body_pose=body_pose, betas=betas).joints
            fit2d = camera_fitting_loss(joints, pred_cam_t, focal_length, joints_2d)
            push3d = torch.sqrt(((joints - gt_keypoints_3d) ** 2).sum(2)).sum(1)
            loss = 4 * fit2d - push3d.mean() / 2 + self.margin
            self.history.append((loss.detach(), fit2d.detach(), push3d.mean().detach()))
            if loss.item() < self.loss_thresh_f3d and fit2d.item() < self.loss_thresh_f2d:
                break
            opt.zero_grad()
            loss.backward()
            opt.step()
        with torch.no_grad():
            out = self.smpl(global_orient=global_orient, body_pose=body_pose, betas=betas)
            reprojection_loss = camera_fitting_loss(out.joints, pred_cam_t, focal_length, joints_2d)
        vertices, joints = out.vertices.detach(), out.joints.detach()
        pj2ds = perspective_projection(joints, pred_cam_t, focal_length / 256).reshape(joints.shape[0], -1, 2)
        return (vertices, joints, pj2ds, global_orient.detach(), body_pose.detach(), betas.detach(), pred_cam_t,
                reprojection_loss)


class FusedSMPLifyInv:
    """SMPLifyInv as one GPU call (thmr_smplify_inv): the loss, its gradient, the stop test and Adam run in CUDA kernels
    next to the body model's forward and backward, with no host round trip per iteration.  Same constructor, call
    arguments, 8-tuple return, in-place updates and `history` as SMPLifyInv; the body model must be the engine's
    (`model.smpl` or an `ops.SMPLModel`), other callables raise ThmrError and keep using SMPLifyInv.

    `run(...)` only enqueues work on the current stream (it can be captured in a CUDA graph) and returns the 8-tuple
    plus the device history [num_iters, 3] and iteration count [1] (int32); `__call__` is `run` plus one device-to-host
    read of the count, which trims `history`."""

    def __init__(self, smpl_model, step_size: float = 1e-3, num_iters: int = 100, margin: float = 20,
                 loss_thresh_f2d: float = 1, loss_thresh_f3d: float = 0, device=torch.device("cuda")):
        from .engine import _SmplFacade
        from .ops import SMPLModel
        from ._lib import ThmrError
        if isinstance(smpl_model, _SmplFacade):
            smpl_model = smpl_model._model
        if not isinstance(smpl_model, SMPLModel):
            raise ThmrError(f"FusedSMPLifyInv needs the engine's body model (model.smpl or ops.SMPLModel), got "
                            f"{type(smpl_model).__name__}; use SMPLifyInv for other body models")
        self.smpl = smpl_model
        self.step_size = step_size
        self.num_iters = num_iters
        self.margin = margin
        self.loss_thresh_f2d = loss_thresh_f2d
        self.loss_thresh_f3d = loss_thresh_f3d
        self.device = device
        self.history: List[Tuple[torch.Tensor, torch.Tensor, torch.Tensor]] = []
        self._ws = None

    def run(self, global_orient: torch.Tensor, body_pose: torch.Tensor, betas: torch.Tensor, pred_cam_t: torch.Tensor,
            focal_length: torch.Tensor, gt_keypoints_2d: torch.Tensor, gt_keypoints_3d: torch.Tensor):
        """Enqueues the fit.  Returns (vertices, joints, pj2ds, global_orient, body_pose, betas, pred_cam_t,
        reprojection_loss, history [num_iters, 3], iters_run [1] int32), all on the device."""
        import ctypes
        from . import _lib
        from .ops import _req, _stream
        m = self.smpl
        for t, flag in ((body_pose, True), (betas, False), (global_orient, True), (pred_cam_t, True)):
            t.requires_grad = flag
        B = betas.shape[0]
        J = 25 + m.n_extra
        for t, name, shape in ((global_orient, "global_orient", (B, 1, 3, 3)), (body_pose, "body_pose", (B, 23, 3, 3)),
                               (pred_cam_t, "pred_cam_t", (B, 3))):
            _req(t, torch.float32, name)
            if tuple(t.shape) != shape or not t.is_contiguous():
                raise _lib.ThmrError(f"{name}: expected a contiguous {shape} tensor (it is updated in place), got "
                                     f"{tuple(t.shape)}")
        betas_c = _req(betas.detach(), torch.float32, "betas")
        focal = _req(focal_length.detach(), torch.float32, "focal_length")
        kp2 = _req(gt_keypoints_2d.detach(), torch.float32, "gt_keypoints_2d")
        kp3 = _req(gt_keypoints_3d.detach(), torch.float32, "gt_keypoints_3d")
        if betas_c.shape != (B, m.num_betas) or focal.shape != (B, 2) or kp2.shape != (B, J, 3) \
                or kp3.shape != (B, J, 3):
            raise _lib.ThmrError(f"FusedSMPLifyInv: betas {tuple(betas_c.shape)}, focal_length {tuple(focal.shape)}, "
                                 f"gt_keypoints_2d {tuple(kp2.shape)}, gt_keypoints_3d {tuple(kp3.shape)} do not match "
                                 f"B = {B}, {m.num_betas} betas and J = {J} joints")
        dev = pred_cam_t.device
        verts = torch.empty(B, m.num_verts, 3, device=dev)
        joints = torch.empty(B, J, 3, device=dev)
        pj2ds = torch.empty(B, J, 2, device=dev)
        reproj = torch.empty((), device=dev)
        history = torch.zeros(self.num_iters, 3, device=dev)
        iters_run = torch.zeros(1, device=dev, dtype=torch.int32)
        need = _lib.lib().thmr_smplify_workspace_bytes(m.handle, B, self.num_iters)
        if need == 0:
            raise _lib.ThmrError(f"FusedSMPLifyInv: B = {B}, num_iters = {self.num_iters}")
        if self._ws is None or self._ws.numel() < need or self._ws.device != dev:
            self._ws = torch.empty(need, device=dev, dtype=torch.uint8)
        d = _lib.SmplifyDesc(B, self.num_iters, J, float(self.step_size), float(self.margin),
                             float(self.loss_thresh_f2d), float(self.loss_thresh_f3d), global_orient.data_ptr(),
                             body_pose.data_ptr(), pred_cam_t.data_ptr(), betas_c.data_ptr(), focal.data_ptr(),
                             kp2.data_ptr(), kp3.data_ptr(), verts.data_ptr(), joints.data_ptr(), pj2ds.data_ptr(),
                             reproj.data_ptr(), history.data_ptr() if self.num_iters else None, iters_run.data_ptr())
        _lib.check(_lib.lib().thmr_smplify_inv(m.handle, ctypes.byref(d), self._ws.data_ptr(), _stream()))
        for t in (global_orient, body_pose, pred_cam_t):      # updated in place, as the reference's optimiser does
            torch.autograd.graph.increment_version(t)
        return (verts, joints, pj2ds, global_orient.detach(), body_pose.detach(), betas.detach(), pred_cam_t, reproj,
                history, iters_run)

    def __call__(self, global_orient: torch.Tensor, body_pose: torch.Tensor, betas: torch.Tensor,
                 pred_cam_t: torch.Tensor, focal_length: torch.Tensor, gt_keypoints_2d: torch.Tensor,
                 gt_keypoints_3d: torch.Tensor):
        """As SMPLifyInv.__call__; afterwards `history` holds one (loss, fit2D, mean push3D) triple of 0-d tensors per
        iteration run."""
        out = self.run(global_orient, body_pose, betas, pred_cam_t, focal_length, gt_keypoints_2d, gt_keypoints_3d)
        history, iters_run = out[8], int(out[9].item())
        self.history = [(history[i, 0], history[i, 1], history[i, 2]) for i in range(iters_run)]
        return out[:8]

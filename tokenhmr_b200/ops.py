"""Stand-alone operators over the C ABI, mirroring the inner seams the reference exposes
(SURVEY.md §8b): QuantizeEMAReset.{quantize,dequantize,dequantize_logits}, smplx.lbs.lbs, the SMPL wrapper,
rot6d_to_rotmat, the ViT attention core, nn.Linear / LayerNorm / Conv1d on the engine's numeric contract.

Every function takes CUDA tensors, launches on torch's current stream and returns CUDA tensors.  There is
no CPU path: a missing library or a CPU tensor raises.
"""
from __future__ import annotations

import ctypes
from typing import Dict, Optional, Tuple

import torch

from . import _lib
from ._lib import check, lib
from .config import SMPL_TO_OPENPOSE

ACT = {"none": 0, "gelu": 1, "relu": 2}


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def _ptr(t: Optional[torch.Tensor]) -> Optional[int]:
    return None if t is None else t.data_ptr()


def _req(t: torch.Tensor, dtype, name: str) -> torch.Tensor:
    if not t.is_cuda:
        raise _lib.ThmrError(f"{name}: expected a CUDA tensor (tokenhmr_b200 has no CPU path)")
    if t.dtype != dtype:
        raise _lib.ThmrError(f"{name}: expected dtype {dtype}, got {t.dtype}")
    return t.contiguous()


# ------------------------------------------------------------------------------------------------
def linear_f16(x16: torch.Tensor, w16: torch.Tensor, bias: Optional[torch.Tensor] = None,
               resid: Optional[torch.Tensor] = None, act: str = "none", out32: bool = True, out16: bool = False,
               block_n: int = 0) -> Tuple[Optional[torch.Tensor], Optional[torch.Tensor]]:
    """F.linear on the tensor cores: x16 (M,K) f16, w16 (N,K) f16 -> fp32 and/or f16 (M,N)."""
    x16, w16 = _req(x16, torch.float16, "x"), _req(w16, torch.float16, "w")
    M, K = x16.shape
    N = w16.shape[0]
    o32 = torch.empty(M, N, device=x16.device, dtype=torch.float32) if out32 else None
    o16 = torch.empty(M, N, device=x16.device, dtype=torch.float16) if out16 else None
    check(lib().thmr_gemm_f16(x16.data_ptr(), K, w16.data_ptr(), K, M, N, K, _ptr(bias), _ptr(resid), N, ACT[act],
                              _ptr(o32), N, _ptr(o16), N, block_n, _stream()))
    return o32, o16


def conv1d_k3_f16(x16: torch.Tensor, w16: torch.Tensor, bias: torch.Tensor, L: int, pad: int, dilation: int = 1,
                  act: str = "none") -> Tuple[torch.Tensor, torch.Tensor]:
    """Conv1d(k=3, padding=dilation) on zero-padded channels-last sequences x16 (B, L+2*pad, Cin);
    w16 (Cout, 3*Cin) tap-major.  Returns (fp32, f16) outputs in the same padded layout."""
    x16, w16 = _req(x16, torch.float16, "x"), _req(w16, torch.float16, "w")
    B, Lp, Cin = x16.shape
    assert Lp == L + 2 * pad
    Cout = w16.shape[0]
    o32 = torch.empty(B, Lp, Cout, device=x16.device, dtype=torch.float32)
    o16 = torch.empty(B, Lp, Cout, device=x16.device, dtype=torch.float16)
    check(lib().thmr_conv1d_k3_f16(x16.data_ptr(), B, L, pad, Cin, w16.data_ptr(), Cout, _ptr(bias), dilation,
                                   ACT[act], o32.data_ptr(), o16.data_ptr(), _stream()))
    return o32, o16


def layernorm(x: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, eps: float, relu: bool = False,
              out16: bool = True, out32: bool = False):
    x = _req(x, torch.float32, "x")
    R, C = x.shape
    y16 = torch.empty(R, C, device=x.device, dtype=torch.float16) if out16 else None
    y32 = torch.empty(R, C, device=x.device, dtype=torch.float32) if out32 else None
    check(lib().thmr_layernorm(x.data_ptr(), gamma.data_ptr(), beta.data_ptr(), R, C, eps, int(relu), _ptr(y16),
                               _ptr(y32), _stream()))
    return y16, y32


def vit_attention(qkv16: torch.Tensor, batch: int, heads: int, return_scores: bool = False):
    """softmax(q k^T / sqrt(80)) v for all heads.  qkv16 (B*192, 3*H*80) f16 -> (B*192, H*80) f16."""
    qkv16 = _req(qkv16, torch.float16, "qkv")
    assert qkv16.shape == (batch * 192, 3 * heads * 80)
    out = torch.empty(batch * 192, heads * 80, device=qkv16.device, dtype=torch.float16)
    dbg = torch.empty(batch * heads, 192, 192, device=qkv16.device, dtype=torch.float32) if return_scores else None
    check(lib().thmr_vit_attention(qkv16.data_ptr(), batch, heads, out.data_ptr(), _ptr(dbg), _stream()))
    return (out, dbg) if return_scores else out


# ------------------------------------------------------------------------------------------------ VQ
def vq_quantize(x: torch.Tensor, codebook: torch.Tensor) -> torch.Tensor:
    """QuantizeEMAReset.quantize (quantize_cnn.py:80-86): x (Q,D) fp32, codebook (K,D) fp32 -> int64 (Q,)."""
    x, codebook = _req(x, torch.float32, "x"), _req(codebook, torch.float32, "codebook")
    Q, D = x.shape
    K = codebook.shape[0]
    idx = torch.empty(Q, device=x.device, dtype=torch.int64)
    ws = torch.empty(lib().thmr_vq_workspace_bytes(Q, K, D), device=x.device, dtype=torch.uint8)
    check(lib().thmr_vq_argmin(x.data_ptr(), Q, codebook.data_ptr(), K, D, idx.data_ptr(), ws.data_ptr(), _stream()))
    return idx


def vq_dequantize(idx: torch.Tensor, codebook: torch.Tensor) -> torch.Tensor:
    """QuantizeEMAReset.dequantize (quantize_cnn.py:88-90)."""
    idx, codebook = _req(idx, torch.int64, "idx"), _req(codebook, torch.float32, "codebook")
    out = torch.empty(idx.numel(), codebook.shape[1], device=idx.device, dtype=torch.float32)
    check(lib().thmr_vq_dequantize(idx.data_ptr(), idx.numel(), codebook.data_ptr(), codebook.shape[1], out.data_ptr(),
                                   _stream()))
    return out


def vq_dequantize_logits(probs: torch.Tensor, codebook: torch.Tensor) -> torch.Tensor:
    """QuantizeEMAReset.dequantize_logits (quantize_cnn.py:92-93): probs (Q,K) @ codebook (K,D) -> (Q,D) fp32
    (f16 operands, fp32 accumulate)."""
    p16 = probs.to(torch.float16).contiguous()
    ct16 = codebook.t().to(torch.float16).contiguous()
    Q, K = p16.shape
    D = ct16.shape[0]
    out = torch.empty(Q, D, device=probs.device, dtype=torch.float32)
    check(lib().thmr_vq_dequant_logits(p16.data_ptr(), Q, K, ct16.data_ptr(), D, out.data_ptr(), _stream()))
    return out


def rot6d_to_rotmat(x: torch.Tensor) -> torch.Tensor:
    """tokenhmr/lib/utils/geometry.py:64-84."""
    x = _req(x.reshape(-1, 6), torch.float32, "x")
    out = torch.empty(x.shape[0], 3, 3, device=x.device, dtype=torch.float32)
    check(lib().thmr_rot6d_to_rotmat(x.data_ptr(), x.shape[0], out.data_ptr(), _stream()))
    return out


# ------------------------------------------------------------------------------------------------ evaluation
def regress_joints(jreg: torch.Tensor, verts: torch.Tensor) -> torch.Tensor:
    """torch.matmul(J_regressor, vertices) (tokenhmr/lib/utils/pose_utils.py:213,219): (J,V) x (B,V,3) -> (B,J,3)."""
    jreg = _req(jreg, torch.float32, "jreg")
    verts = _req(verts, torch.float32, "verts")
    if jreg.dim() != 2 or verts.dim() != 3 or verts.shape[1] != jreg.shape[1] or verts.shape[2] != 3:
        raise ValueError(f"regress_joints: jreg {tuple(jreg.shape)} vs verts {tuple(verts.shape)}")
    out = torch.empty(verts.shape[0], jreg.shape[0], 3, device=verts.device, dtype=torch.float32)
    check(lib().thmr_regress_joints(jreg.data_ptr(), jreg.shape[0], verts.data_ptr(), verts.shape[1], verts.shape[0],
                                    out.data_ptr(), _stream()))
    return out


def eval_pose(pred_kp: torch.Tensor, gt_kp: torch.Tensor, keypoint_list: torch.Tensor, pelvis: Tuple[int, int],
              pred_verts: Optional[torch.Tensor] = None, gt_verts: Optional[torch.Tensor] = None):
    """Pelvis alignment + MPJPE + Procrustes-aligned MPJPE (+ PVE) in mm for one batch
    (tokenhmr/lib/utils/pose_utils.py:61-143,201-275).  gt_kp may still carry the confidence column (B,J,4).
    Returns (mpjpe, re, pve-or-None), each (B,) fp32 on the GPU."""
    pred_kp = _req(pred_kp, torch.float32, "pred_kp")
    gt_kp = _req(gt_kp, torch.float32, "gt_kp")
    keypoint_list = _req(keypoint_list, torch.int32, "keypoint_list")
    B, J = pred_kp.shape[0], pred_kp.shape[1]
    if pred_kp.dim() != 3 or pred_kp.shape[2] != 3 or gt_kp.dim() != 3 or gt_kp.shape[:2] != pred_kp.shape[:2] \
            or gt_kp.shape[2] not in (3, 4):
        raise ValueError(f"eval_pose: pred_kp {tuple(pred_kp.shape)} vs gt_kp {tuple(gt_kp.shape)}")
    mpjpe = torch.empty(B, device=pred_kp.device, dtype=torch.float32)
    re = torch.empty_like(mpjpe)
    pve, pv, gv, V = None, 0, 0, 0
    if pred_verts is not None or gt_verts is not None:
        pred_verts = _req(pred_verts, torch.float32, "pred_verts")
        gt_verts = _req(gt_verts, torch.float32, "gt_verts")
        if pred_verts.shape != gt_verts.shape or pred_verts.shape[0] != B or pred_verts.shape[-1] != 3:
            raise ValueError(f"eval_pose: vertices {tuple(pred_verts.shape)} vs {tuple(gt_verts.shape)}")
        pve = torch.empty_like(mpjpe)
        pv, gv, V = pred_verts.data_ptr(), gt_verts.data_ptr(), pred_verts.shape[1]
    check(lib().thmr_eval_pose(pred_kp.data_ptr(), gt_kp.data_ptr(), gt_kp.shape[2], J, keypoint_list.data_ptr(),
                               keypoint_list.numel(), int(pelvis[0]), int(pelvis[1]), pv, gv, V, B, mpjpe.data_ptr(),
                               re.data_ptr(), pve.data_ptr() if pve is not None else 0, _stream()))
    return mpjpe, re, pve


def cam_crop_to_full(cam_bbox: torch.Tensor, box_center: torch.Tensor, box_size: torch.Tensor, img_size: torch.Tensor,
                     focal_length: float = 5000.0) -> torch.Tensor:
    """tokenhmr/lib/utils/renderer.py:13-23 (same argument order)."""
    cam_bbox = _req(cam_bbox, torch.float32, "cam_bbox")
    box_center = _req(box_center, torch.float32, "box_center")
    box_size = _req(box_size.reshape(-1), torch.float32, "box_size")
    img_size = _req(img_size, torch.float32, "img_size")
    B = cam_bbox.shape[0]
    if cam_bbox.shape != (B, 3) or box_center.shape != (B, 2) or box_size.shape != (B,) or img_size.shape != (B, 2):
        raise ValueError("cam_crop_to_full: expected cam (B,3), center (B,2), size (B,), img_size (B,2)")
    out = torch.empty(B, 3, device=cam_bbox.device, dtype=torch.float32)
    check(lib().thmr_cam_crop_to_full(cam_bbox.data_ptr(), box_center.data_ptr(), box_size.data_ptr(),
                                      img_size.data_ptr(), float(focal_length), B, out.data_ptr(), _stream()))
    return out


# ------------------------------------------------------------------------------------------------ SMPL
class SMPLModel:
    """Device-resident SMPL model (thmr_smpl).  `smpl` holds the smplx buffers: v_template, shapedirs, posedirs,
    J_regressor, lbs_weights, parents, joint_regressor_extra, extra_vertex_ids (tokenhmr_b200.synth.make_smpl or a
    real SMPL pkl converted by the caller)."""

    def __init__(self, smpl: Dict[str, torch.Tensor], device: torch.device):
        self.device = device
        dev = lambda n: smpl[n].to(device=device, dtype=torch.float32).contiguous()
        vt, sd, pd, jr, lw = dev("v_template"), dev("shapedirs"), dev("posedirs"), dev("J_regressor"), dev("lbs_weights")
        jx = smpl.get("joint_regressor_extra")
        jx = None if jx is None else jx.to(device=device, dtype=torch.float32).contiguous()
        self.num_verts = vt.shape[0]
        self.num_betas = sd.shape[2]
        self.n_extra = 0 if jx is None else jx.shape[0]
        arr = lambda vals: (ctypes.c_int32 * len(vals))(*[int(v) for v in vals])
        parents = arr(smpl["parents"].tolist())
        evid = arr(smpl["extra_vertex_ids"].tolist())
        jmap = arr(SMPL_TO_OPENPOSE)
        d = _lib.SmplDesc(self.num_verts, self.num_betas, vt.data_ptr(), sd.data_ptr(), pd.data_ptr(), jr.data_ptr(),
                          lw.data_ptr(), parents, _ptr(jx), self.n_extra, evid, jmap)
        h = ctypes.c_void_p()
        check(lib().thmr_smpl_create(ctypes.byref(d), ctypes.byref(h)))
        torch.cuda.synchronize(device)
        self.handle = h
        self._ws: Optional[torch.Tensor] = None
        self._bws: Optional[torch.Tensor] = None
        self.faces = smpl.get("faces")

    def __del__(self):
        try:
            if getattr(self, "handle", None):
                lib().thmr_smpl_destroy(self.handle)
                self.handle = None
        except Exception:
            pass

    def workspace(self, batch: int) -> torch.Tensor:
        need = lib().thmr_smpl_workspace_bytes(self.handle, batch)
        if self._ws is None or self._ws.numel() < need:
            self._ws = torch.empty(need, device=self.device, dtype=torch.uint8)
        return self._ws

    def backward_workspace(self, batch: int) -> torch.Tensor:
        need = lib().thmr_smpl_backward_workspace_bytes(self.handle, batch)
        if self._bws is None or self._bws.numel() < need:
            self._bws = torch.empty(need, device=self.device, dtype=torch.uint8)
        return self._bws

    def lbs(self, betas: torch.Tensor, pose: torch.Tensor, pose2rot: bool = True):
        """smplx.lbs.lbs: returns (verts (B,V,3), J_transformed (B,24,3)).  Differentiable in pose and betas when grad
        mode is on and one of them requires grad (thmr_lbs_backward)."""
        if _wants_grad(betas, pose):
            return _LbsFn.apply(self, betas, pose, bool(pose2rot))
        return self._lbs(betas, pose, pose2rot)

    def _lbs(self, betas: torch.Tensor, pose: torch.Tensor, pose2rot: bool):
        betas, pose = _req(betas, torch.float32, "betas"), _req(pose, torch.float32, "pose")
        B = betas.shape[0]
        verts = torch.empty(B, self.num_verts, 3, device=self.device)
        joints = torch.empty(B, 24, 3, device=self.device)
        check(lib().thmr_lbs(self.handle, pose.data_ptr(), int(pose2rot), betas.data_ptr(), B, verts.data_ptr(),
                             joints.data_ptr(), self.workspace(B).data_ptr(), _stream()))
        return verts, joints

    def forward(self, global_orient: torch.Tensor, body_pose: torch.Tensor, betas: torch.Tensor,
                pred_cam: Optional[torch.Tensor] = None, focal_length: float = 5000.0, image_size: float = 256.0):
        """tokenhmr SMPL wrapper forward (smpl_wrapper.py:27-41): rotation matrices -> (vertices, 44 joints)
        [+ (cam_t, focal, keypoints_2d) when pred_cam is given: tokenhmr.py:165-187].  Without pred_cam it is
        differentiable in global_orient, body_pose and betas when grad mode is on and one of them requires grad
        (thmr_smpl_backward); the camera tail has no backward, so pred_cam with such inputs raises."""
        if _wants_grad(global_orient, body_pose, betas):
            if pred_cam is not None:
                raise _lib.ThmrError("SMPLModel.forward: the camera tail (pred_cam) has no backward; call it without "
                                     "pred_cam and project in PyTorch, or run it under torch.no_grad()")
            B = betas.shape[0]
            rot = torch.cat([global_orient.reshape(B, -1, 3, 3), body_pose.reshape(B, -1, 3, 3)], 1)
            return _SmplForwardFn.apply(self, rot, betas)
        return self._forward(global_orient, body_pose, betas, pred_cam, focal_length, image_size)

    def _forward(self, global_orient: torch.Tensor, body_pose: torch.Tensor, betas: torch.Tensor,
                 pred_cam: Optional[torch.Tensor] = None, focal_length: float = 5000.0, image_size: float = 256.0):
        B = betas.shape[0]
        rot = torch.cat([global_orient.reshape(B, -1, 3, 3), body_pose.reshape(B, -1, 3, 3)], 1)
        rot, betas = _req(rot, torch.float32, "rotmats"), _req(betas, torch.float32, "betas")
        nj = 25 + self.n_extra
        verts = torch.empty(B, self.num_verts, 3, device=self.device)
        joints = torch.empty(B, nj, 3, device=self.device)
        cam_t = focal = kp2d = None
        if pred_cam is not None:
            pred_cam = _req(pred_cam, torch.float32, "pred_cam")
            cam_t = torch.empty(B, 3, device=self.device)
            focal = torch.empty(B, 2, device=self.device)
            kp2d = torch.empty(B, nj, 2, device=self.device)
        check(lib().thmr_smpl_forward(self.handle, rot.data_ptr(), betas.data_ptr(), B, verts.data_ptr(),
                                      joints.data_ptr(), _ptr(pred_cam), focal_length, image_size, _ptr(cam_t),
                                      _ptr(focal), _ptr(kp2d), self.workspace(B).data_ptr(), _stream()))
        return (verts, joints) if pred_cam is None else (verts, joints, cam_t, focal, kp2d)

    def smpl_backward(self, rotmats: torch.Tensor, betas: torch.Tensor, grad_verts: Optional[torch.Tensor],
                      grad_joints: Optional[torch.Tensor]) -> Tuple[torch.Tensor, torch.Tensor]:
        """thmr_smpl_backward: rotmats (B,24,3,3), betas (B,nb), cotangents of (vertices, joints) (None = zero) ->
        (grad_rotmats (B,24,3,3), grad_betas (B,nb))."""
        rotmats, betas = _req(rotmats, torch.float32, "rotmats"), _req(betas, torch.float32, "betas")
        B = betas.shape[0]
        gv = None if grad_verts is None else _req(grad_verts, torch.float32, "grad_verts")
        gj = None if grad_joints is None else _req(grad_joints, torch.float32, "grad_joints")
        g_rot = torch.empty(B, 24, 3, 3, device=self.device)
        g_betas = torch.empty(B, self.num_betas, device=self.device)
        check(lib().thmr_smpl_backward(self.handle, rotmats.data_ptr(), betas.data_ptr(), B, _ptr(gv), _ptr(gj),
                                       g_rot.data_ptr(), g_betas.data_ptr(), self.backward_workspace(B).data_ptr(),
                                       _stream()))
        return g_rot, g_betas

    def lbs_backward(self, betas: torch.Tensor, pose: torch.Tensor, pose2rot: bool, grad_verts: Optional[torch.Tensor],
                     grad_joints: Optional[torch.Tensor]) -> Tuple[torch.Tensor, torch.Tensor]:
        """thmr_lbs_backward: cotangents of (verts, J_transformed) (None = zero) -> (grad_pose shaped as pose,
        grad_betas (B,nb))."""
        betas, pose = _req(betas, torch.float32, "betas"), _req(pose, torch.float32, "pose")
        B = betas.shape[0]
        gv = None if grad_verts is None else _req(grad_verts, torch.float32, "grad_verts")
        gj = None if grad_joints is None else _req(grad_joints, torch.float32, "grad_joints")
        g_pose = torch.empty(B, 24, 3, device=self.device) if pose2rot else torch.empty(B, 24, 3, 3, device=self.device)
        g_betas = torch.empty(B, self.num_betas, device=self.device)
        check(lib().thmr_lbs_backward(self.handle, pose.data_ptr(), int(pose2rot), betas.data_ptr(), B, _ptr(gv),
                                      _ptr(gj), g_pose.data_ptr(), g_betas.data_ptr(),
                                      self.backward_workspace(B).data_ptr(), _stream()))
        return g_pose.view(pose.shape), g_betas


def _wants_grad(*ts: torch.Tensor) -> bool:
    return torch.is_grad_enabled() and any(t.requires_grad for t in ts)


# ------------------------------------------------------------------------------------------------ camera tail
def camera_tail(joints: torch.Tensor, pred_cam: torch.Tensor, focal_length: float = 5000.0,
                image_size: float = 256.0) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """The camera tail of forward_step (tokenhmr.py:162-187): joints (B,J,3) and pred_cam (B,3) -> (pred_cam_t (B,3),
    focal_length (B,2), keypoints_2d (B,J,2)), the numbers SMPLModel.forward(..., pred_cam=) gives for the same joints.
    Differentiable in joints and pred_cam when grad mode is on and one of them requires grad
    (thmr_camera_tail_backward)."""
    if _wants_grad(joints, pred_cam):
        return _CameraTailFn.apply(joints, pred_cam, float(focal_length), float(image_size))
    return _camera_tail(joints, pred_cam, float(focal_length), float(image_size))


def _camera_tail(joints: torch.Tensor, pred_cam: torch.Tensor, focal_length: float, image_size: float):
    joints, pred_cam = _req(joints, torch.float32, "joints"), _req(pred_cam, torch.float32, "pred_cam")
    if joints.dim() != 3 or joints.shape[2] != 3 or pred_cam.shape != (joints.shape[0], 3):
        raise _lib.ThmrError(f"camera_tail: joints {tuple(joints.shape)} must be (B,J,3) and pred_cam "
                             f"{tuple(pred_cam.shape)} (B,3)")
    B, J = joints.shape[:2]
    cam_t = torch.empty(B, 3, device=joints.device)
    focal = torch.empty(B, 2, device=joints.device)
    kp2d = torch.empty(B, J, 2, device=joints.device)
    check(lib().thmr_camera_tail(joints.data_ptr(), pred_cam.data_ptr(), B, J, focal_length, image_size,
                                 cam_t.data_ptr(), focal.data_ptr(), kp2d.data_ptr(), _stream()))
    return cam_t, focal, kp2d


class _CameraTailFn(torch.autograd.Function):
    """camera_tail with thmr_camera_tail_backward as its backward (focal_length carries no gradient)."""

    @staticmethod
    def forward(ctx, joints: torch.Tensor, pred_cam: torch.Tensor, focal_length: float, image_size: float):
        ctx.set_materialize_grads(False)
        ctx.focal_length, ctx.image_size = focal_length, image_size
        joints, pred_cam = joints.contiguous(), pred_cam.contiguous()
        ctx.save_for_backward(joints, pred_cam)
        cam_t, focal, kp2d = _camera_tail(joints, pred_cam, focal_length, image_size)
        ctx.mark_non_differentiable(focal)
        return cam_t, focal, kp2d

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad_cam_t, _grad_focal, grad_kp2d):
        joints, pred_cam = ctx.saved_tensors
        if grad_cam_t is None and grad_kp2d is None:
            return None, None, None, None
        B, J = joints.shape[:2]
        gk = None if grad_kp2d is None else _req(grad_kp2d, torch.float32, "grad_kp2d")
        gc = None if grad_cam_t is None else _req(grad_cam_t, torch.float32, "grad_cam_t")
        g_joints = torch.empty_like(joints)
        g_cam = torch.empty_like(pred_cam)
        check(lib().thmr_camera_tail_backward(joints.data_ptr(), pred_cam.data_ptr(), B, J, ctx.focal_length,
                                              ctx.image_size, _ptr(gk), _ptr(gc), g_joints.data_ptr(),
                                              g_cam.data_ptr(), _stream()))
        return (g_joints if ctx.needs_input_grad[0] else None, g_cam if ctx.needs_input_grad[1] else None, None, None)


class _SmplForwardFn(torch.autograd.Function):
    """SMPLModel.forward without the camera tail, with thmr_smpl_backward as its backward."""

    @staticmethod
    def forward(ctx, model: SMPLModel, rot: torch.Tensor, betas: torch.Tensor):
        ctx.set_materialize_grads(False)
        ctx.model = model
        ctx.save_for_backward(rot, betas)
        return model._forward(rot[:, :1], rot[:, 1:], betas)

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad_verts, grad_joints):
        rot, betas = ctx.saved_tensors
        if grad_verts is None and grad_joints is None:
            return None, None, None
        g_rot, g_betas = ctx.model.smpl_backward(rot.reshape(rot.shape[0], 24, 3, 3), betas, grad_verts, grad_joints)
        return (None, g_rot.view(rot.shape) if ctx.needs_input_grad[1] else None,
                g_betas if ctx.needs_input_grad[2] else None)


class _LbsFn(torch.autograd.Function):
    """SMPLModel.lbs with thmr_lbs_backward as its backward."""

    @staticmethod
    def forward(ctx, model: SMPLModel, betas: torch.Tensor, pose: torch.Tensor, pose2rot: bool):
        ctx.set_materialize_grads(False)
        ctx.model, ctx.pose2rot = model, pose2rot
        ctx.save_for_backward(betas, pose)
        return model._lbs(betas, pose, pose2rot)

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad_verts, grad_joints):
        betas, pose = ctx.saved_tensors
        if grad_verts is None and grad_joints is None:
            return None, None, None, None
        g_pose, g_betas = ctx.model.lbs_backward(betas, pose, ctx.pose2rot, grad_verts, grad_joints)
        return (None, g_betas if ctx.needs_input_grad[1] else None, g_pose if ctx.needs_input_grad[2] else None, None)

"""Training-loss golden: TokenHMR.compute_loss (tokenhmr/lib/models/tokenhmr.py:190-277) on the LIVE reference
lib/models/losses.py and lib/utils/geometry.aa_to_rotmat (loaded file by file through oracle/ref_import.py; losses.py
needs only rotation_utils.py), run on the CPU in fp64 with autograd.  TEST INFRASTRUCTURE ONLY.

    TOKENHMR_REFERENCE=<checkout> python -m oracle.loss_oracle      # writes tests/golden/tals_loss.npz

tokenhmr.py itself needs pytorch_lightning, so compute_loss's body is restated below (`compute_loss`), with the loss
modules chosen as TokenHMR.__init__ chooses them (tokenhmr.py:67-74) and the release config's LOOSE_WEIGHT and
LOSS_WEIGHTS.  Two seeded cases at B = 16 with 44 keypoints and mixed dataset names: "tals" (LOOSE_SUP, train=True:
training_step) and "plain" (LOOSE_SUP, train=False: validation_step).  Confidences are 0, 1 or fractional,
has_smpl_params is 0 for some samples, sample 0 is a BEDLAM sample without pose parameters and sample 1 an
H36M-TRAIN-WMASK sample without betas (the two TALS quirks: full-weight pose loss, betas gated by has * valid_3D), and every 2-D error c |pred - gt|^2 and every pose angle lies at least MARGIN
from its threshold, on both sides (asserted).  Stored per case: the inputs (fp32-representable), the six terms of
output['losses'] and d loss / d (pred_keypoints_2d, pred_keypoints_3d, global_orient, body_pose, betas), in fp64.
"""
from __future__ import annotations

import importlib
from pathlib import Path
from typing import Dict

import numpy as np
import torch

from oracle import ref_import

GOLDEN = Path(__file__).resolve().parent.parent / "tests" / "golden" / "tals_loss.npz"
B, J = 16, 44
MARGIN = 1e-4            # distance of every 2-D error and pose angle from its threshold
LOOSE_WEIGHT = 0.05      # tokenhmr_release.yaml:53
LOSS_WEIGHTS = {"KEYPOINTS_3D": 0.05, "KEYPOINTS_2D": 0.01, "GLOBAL_ORIENT": 0.001, "BODY_POSE": 0.001,
                "BETAS": 0.0005}   # tokenhmr_release.yaml:83-88
CASES = {"tals": dict(seed=21, train=True), "plain": dict(seed=22, train=False)}
DATASETS = ["H36M-TRAIN-WMASK", "BEDLAM", "COCO-TRAIN-2014", "MPII-TRAIN", "AIC-TRAIN", "INSTA-TRAIN"]
PRED_KEYS = ("pred_keypoints_2d", "pred_keypoints_3d", "pred_global_orient", "pred_body_pose", "pred_betas")


def modules():
    ref_import.load_modules()
    return importlib.import_module("lib.models.losses"), importlib.import_module("lib.utils.geometry")


def compute_loss(L, geometry, batch: Dict, output: Dict, train: bool, loose_sup: bool = True):
    """tokenhmr.py:201-277 with the modules of tokenhmr.py:67-74 (cfg.MODEL.LOOSE_SUP = loose_sup)."""
    aa_to_rotmat = geometry.aa_to_rotmat
    if loose_sup:
        keypoint_3d_loss, keypoint_2d_loss = L.Keypoint3DLossPCKT("l1"), L.Keypoint2DLossPCKT("l1")
        smpl_parameter_loss = L.ParameterLossPCKT()
    else:
        keypoint_3d_loss, keypoint_2d_loss = L.Keypoint3DLoss("l1"), L.Keypoint2DLoss("l1")
        smpl_parameter_loss = L.ParameterLoss()
    pred_smpl_params = output["pred_smpl_params"]
    pred_keypoints_2d = output["pred_keypoints_2d"]
    pred_keypoints_3d = output["pred_keypoints_3d"]
    batch_size = pred_smpl_params["body_pose"].shape[0]
    gt_keypoints_2d = batch["keypoints_2d"]
    gt_keypoints_3d = batch["keypoints_3d"]
    gt_smpl_params = batch["smpl_params"]
    has_smpl_params = batch["has_smpl_params"]
    is_axis_angle = batch["smpl_params_is_axis_angle"]
    if loose_sup and train:
        dataset_names = batch["dataset"]
        batch_size = pred_keypoints_2d.shape[0]
        kp2D_err = gt_keypoints_2d[:, :, -1] * torch.nn.functional.mse_loss(
            pred_keypoints_2d, gt_keypoints_2d[:, :, :-1], reduction="none").sum(dim=2)
        valid_mask2D = kp2D_err > L.kp2D_err_valid_thresh[None].repeat(batch_size, 1).to(kp2D_err.device)
        weak_mask = gt_keypoints_2d[:, :, -1] * (~valid_mask2D).float()
        gt_keypoints_2d[:, :, -1] = gt_keypoints_2d[:, :, -1] * valid_mask2D
        loss_keypoints_2d = keypoint_2d_loss(pred_keypoints_2d, gt_keypoints_2d, weak_mask, LOOSE_WEIGHT)
        valid_3D_mask = torch.Tensor([name in ["H36M-TRAIN-WMASK", "BEDLAM"] for name in dataset_names]).float().to(
            gt_keypoints_3d.device)
        gt_keypoints_3d[:, :, -1] = gt_keypoints_3d[:, :, -1] * ((valid_3D_mask.unsqueeze(-1) + gt_keypoints_2d[:, :, -1]) > 0.5)
        loss_keypoints_3d = keypoint_3d_loss(pred_keypoints_3d, gt_keypoints_3d, pelvis_id=25 + 14)
        loss_smpl_params = {}
        for k, pred in pred_smpl_params.items():
            gt = gt_smpl_params[k].view(batch_size, -1)
            if is_axis_angle[k].all():
                gt = aa_to_rotmat(gt.reshape(-1, 3)).view(batch_size, -1, 3, 3)
            has_gt = has_smpl_params[k]
            if k in ["betas"]:
                valid_mask3D = None
                weak_mask = None
                has_gt *= valid_3D_mask
            elif k in ["body_pose", "global_orient"]:
                angle_error = L.joint_angle_error(pred, gt)
                valid_mask3D = angle_error > L.angle_valid_thresh[k][None].repeat(batch_size, 1).to(angle_error.device)
                valid_mask3D = (valid_mask3D * has_gt.unsqueeze(1) + valid_3D_mask.unsqueeze(1)).bool()
                weak_mask = (~valid_mask3D * has_gt.unsqueeze(1)).float()
                valid_mask3D = valid_mask3D.float()
            loss_smpl_params[k] = smpl_parameter_loss(pred, gt, has_gt, valid_mask3D, weak_mask, LOOSE_WEIGHT)
    else:
        loss_keypoints_2d = keypoint_2d_loss(pred_keypoints_2d, gt_keypoints_2d)
        loss_keypoints_3d = keypoint_3d_loss(pred_keypoints_3d, gt_keypoints_3d, pelvis_id=25 + 14)
        loss_smpl_params = {}
        for k, pred in pred_smpl_params.items():
            gt = gt_smpl_params[k].view(batch_size, -1)
            if is_axis_angle[k].all():
                gt = aa_to_rotmat(gt.reshape(-1, 3)).view(batch_size, -1, 3, 3)
            has_gt = has_smpl_params[k]
            loss_smpl_params[k] = smpl_parameter_loss(pred.reshape(batch_size, -1), gt.reshape(batch_size, -1), has_gt)
    loss = LOSS_WEIGHTS["KEYPOINTS_3D"] * loss_keypoints_3d + \
        LOSS_WEIGHTS["KEYPOINTS_2D"] * loss_keypoints_2d + \
        sum([loss_smpl_params[k] * LOSS_WEIGHTS[k.upper()] for k in loss_smpl_params])
    losses = dict(loss=loss.detach(), loss_keypoints_2d=loss_keypoints_2d.detach(),
                  loss_keypoints_3d=loss_keypoints_3d.detach())
    for k, v in loss_smpl_params.items():
        losses["loss_" + k] = v.detach()
    output["losses"] = losses
    return loss


def _angles(L, geometry, pred_rot, gt_aa):
    """joint_angle_error of (B,K,3,3) predictions against (B,3K) GT axis-angles (fp64)."""
    gt = geometry.aa_to_rotmat(gt_aa.reshape(-1, 3)).view(pred_rot.shape)
    return L.joint_angle_error(pred_rot, gt)


def make_inputs(seed: int) -> Dict[str, torch.Tensor]:
    """fp32-representable fp64 inputs with every 2-D error and pose angle at least MARGIN from its threshold."""
    L, geometry = modules()
    g = torch.Generator().manual_seed(seed)
    f32 = lambda t: t.float().double()
    rnd = lambda *s: torch.rand(*s, generator=g, dtype=torch.float64)
    nrm = lambda *s: torch.randn(*s, generator=g, dtype=torch.float64)

    def conf(*s):   # a third each of 0, 1 and fractional
        u, c = rnd(*s), rnd(*s)
        return torch.where(u < 1 / 3, torch.zeros_like(c), torch.where(u < 2 / 3, torch.ones_like(c), c))

    # 2-D: pred = gt + d along a random direction, |d|^2 c at a random factor in [0.3, 0.9] or [1.1, 3] of the
    # joint's threshold (0 where c = 0)
    thr2 = L.kp2D_err_valid_thresh.double()
    gt2 = f32(torch.cat([0.4 * nrm(B, J, 2), conf(B, J, 1)], -1))
    c = gt2[..., 2]
    fac = torch.where(rnd(B, J) < 0.5, 0.3 + 0.6 * rnd(B, J), 1.1 + 1.9 * rnd(B, J))
    r = torch.sqrt(fac * thr2 / c.clamp_min(0.05))
    phi = 2 * torch.pi * rnd(B, J)
    pred2 = f32(gt2[..., :2] + r[..., None] * torch.stack([phi.cos(), phi.sin()], -1))
    # 3-D: pelvis-aligned L1 with zero / one / fractional confidences
    gt3 = f32(torch.cat([0.5 * nrm(B, J, 3), conf(B, J, 1)], -1))
    pred3 = f32(gt3[..., :3] + 0.05 * nrm(B, J, 3) + 0.1 * nrm(B, 1, 3))
    # poses: pred = R(gt) R(delta) with |delta| a random factor in [0.3, 0.9] or [1.1, 3] of the threshold
    thr_go = L.angle_valid_thresh["global_orient"].double()
    thr_bp = L.angle_valid_thresh["body_pose"].double()
    thr = torch.cat([thr_go, thr_bp])                                       # (24,)
    gt_aa = f32(0.5 * nrm(B, 24, 3))
    fac = torch.where(rnd(B, 24) < 0.5, 0.3 + 0.6 * rnd(B, 24), 1.1 + 1.9 * rnd(B, 24))
    axis = nrm(B, 24, 3)
    axis = axis / axis.norm(dim=-1, keepdim=True)
    delta = axis * (fac * thr)[..., None]
    R = geometry.aa_to_rotmat(gt_aa.reshape(-1, 3)) @ geometry.aa_to_rotmat(delta.reshape(-1, 3))
    R = f32(R.view(B, 24, 3, 3))
    has_pose = (rnd(B) < 0.75).double()
    has_betas = (rnd(B) < 0.75).double()
    names = [DATASETS[i] for i in torch.randint(len(DATASETS), (B,), generator=g).tolist()]
    names[0], has_pose[0], has_betas[0] = "BEDLAM", 0.0, 1.0               # valid_3D = 1, has pose = 0
    names[1], has_pose[1], has_betas[1] = "H36M-TRAIN-WMASK", 1.0, 0.0     # valid_3D = 1, has betas = 0
    x = dict(pred_keypoints_2d=pred2, pred_keypoints_3d=pred3, pred_global_orient=R[:, :1].contiguous(),
             pred_body_pose=R[:, 1:].contiguous(), pred_betas=f32(nrm(B, 10)), gt_keypoints_2d=gt2,
             gt_keypoints_3d=gt3, gt_global_orient=gt_aa[:, 0].contiguous(),
             gt_body_pose=gt_aa[:, 1:].reshape(B, 69).contiguous(), gt_betas=f32(nrm(B, 10)),
             has_global_orient=has_pose, has_body_pose=has_pose.clone(), has_betas=has_betas,
             valid_3d=torch.tensor([float(n in ("H36M-TRAIN-WMASK", "BEDLAM")) for n in names], dtype=torch.float64))
    # the margins hold on the stored (fp32-rounded) values, as the reference computes them
    e2 = x["gt_keypoints_2d"][..., 2] * ((x["pred_keypoints_2d"] - x["gt_keypoints_2d"][..., :2]) ** 2).sum(-1)
    assert ((e2 - thr2).abs() >= MARGIN).all(), "a 2-D error is too close to its threshold"
    ang = torch.cat([_angles(L, geometry, x["pred_global_orient"], x["gt_global_orient"]),
                     _angles(L, geometry, x["pred_body_pose"], x["gt_body_pose"])], 1)
    assert ((ang - thr).abs() >= MARGIN).all(), "a pose angle is too close to its threshold"
    assert ((ang > thr).any() and (ang < thr).any() and (e2 > thr2).any() and (e2[c > 0] < thr2.expand(B, J)[c > 0]).any())
    return x, names


def run_reference(x: Dict[str, torch.Tensor], names, train: bool) -> Dict[str, np.ndarray]:
    """One compute_loss call on fresh copies of the inputs, then autograd of the loss to the five predictions."""
    L, geometry = modules()
    pred = {k: x[k].clone().requires_grad_(True) for k in PRED_KEYS}
    batch = {"keypoints_2d": x["gt_keypoints_2d"].clone(), "keypoints_3d": x["gt_keypoints_3d"].clone(),
             "smpl_params": {"global_orient": x["gt_global_orient"].clone(), "body_pose": x["gt_body_pose"].clone(),
                             "betas": x["gt_betas"].clone()},
             "has_smpl_params": {"global_orient": x["has_global_orient"].clone(),
                                 "body_pose": x["has_body_pose"].clone(), "betas": x["has_betas"].clone()},
             "smpl_params_is_axis_angle": {"global_orient": torch.ones(B, dtype=torch.bool),
                                           "body_pose": torch.ones(B, dtype=torch.bool),
                                           "betas": torch.zeros(B, dtype=torch.bool)},
             "dataset": list(names)}
    output = {"pred_smpl_params": {"global_orient": pred["pred_global_orient"], "body_pose": pred["pred_body_pose"],
                                   "betas": pred["pred_betas"]},
              "pred_keypoints_2d": pred["pred_keypoints_2d"], "pred_keypoints_3d": pred["pred_keypoints_3d"]}
    loss = compute_loss(L, geometry, batch, output, train)
    grads = torch.autograd.grad(loss, [pred[k] for k in PRED_KEYS])
    terms = output["losses"]
    out = {"losses": np.array([terms[k].item() for k in ("loss", "loss_keypoints_2d", "loss_keypoints_3d",
                                                         "loss_global_orient", "loss_body_pose", "loss_betas")])}
    out.update({"grad_" + k[len("pred_"):]: gr.numpy() for k, gr in zip(PRED_KEYS, grads)})
    return out


def build_cases() -> Dict[str, np.ndarray]:
    arrays: Dict[str, np.ndarray] = {}
    for name, c in CASES.items():
        x, names = make_inputs(c["seed"])
        got = run_reference(x, names, c["train"])
        arrays.update({f"{name}_{k}": v.numpy() for k, v in x.items()})
        arrays[f"{name}_dataset"] = np.array(names)
        arrays.update({f"{name}_{k}": v for k, v in got.items()})
        arrays[f"{name}_config"] = np.array([1.0, float(c["train"]), LOOSE_WEIGHT], np.float64)
    return arrays


def main() -> None:
    np.savez_compressed(GOLDEN, **build_cases())
    print(f"wrote {GOLDEN}")


if __name__ == "__main__":
    main()


# ---- the same loss in plain torch, without the reference tree (a timing baseline that runs on the GPU) -------------
KP2D_ERR_THRESH = [0.0085024, 0.00648666, 0.00747825, 0.01103439, 0.01355629, 0.00741691, 0.01096735, 0.01414461,
                   0.00974212, 0.01127469, 0.01663222, 0.00564927, 0.01126335, 0.01615757, 0.00532595, 0.00829731,
                   0.00831497, 0.00737241, 0.00743286, 0.00543739, 0.00550524, 0.00535504, 0.00565414, 0.00581685,
                   0.00573041, 0.00554029, 0.01515258, 0.00986267, 0.00997563, 0.01519944, 0.00511402, 0.01288267,
                   0.01105894, 0.00710525, 0.00709785, 0.01092387, 0.01388091, 0.00648326, 0.00766487, 0.00931454,
                   0.00646622, 0.00677057, 0.00744011, 0.00752381]
BODY_ANGLE_THRESH = [0.273709, 0.26481161, 0.1838198, 0.41490657, 0.37521194, 0.20793171, 0.24905021, 0.33887333,
                     0.14481062, 0.35632194, 0.34944217, 0.30542146, 0.32835298, 0.33110567, 0.34813467, 0.36357761,
                     0.40062272, 0.43493496, 0.4400709, 0.78017052, 0.7375746, 0.24927082, 0.24966981]


def _aa_to_rotmat(theta):
    angle = torch.norm(theta + 1e-8, p=2, dim=1).unsqueeze(-1)
    q = torch.cat([torch.cos(angle * 0.5), torch.sin(angle * 0.5) * (theta / angle)], 1)
    q = q / q.norm(p=2, dim=1, keepdim=True)
    w, x, y, z = q.unbind(1)
    return torch.stack([w * w + x * x - y * y - z * z, 2 * x * y - 2 * w * z, 2 * w * y + 2 * x * z,
                        2 * w * z + 2 * x * y, w * w - x * x + y * y - z * z, 2 * y * z - 2 * w * x,
                        2 * x * z - 2 * w * y, 2 * w * x + 2 * y * z, w * w - x * x - y * y + z * z], 1).view(-1, 3, 3)


def _angle(m):
    """|matrix_to_axis_angle(m)| as rotation_utils computes it (first best-conditioned quaternion candidate)."""
    m = m.reshape(-1, 9)
    m00, m01, m02, m10, m11, m12, m20, m21, m22 = m.unbind(1)
    t = torch.stack([1 + m00 + m11 + m22, 1 + m00 - m11 - m22, 1 - m00 + m11 - m22, 1 - m00 - m11 + m22], 1)
    qa = torch.where(t > 0, t.clamp_min(0).sqrt(), torch.zeros_like(t))
    cand = torch.stack([torch.stack([qa[:, 0] ** 2, m21 - m12, m02 - m20, m10 - m01], 1),
                        torch.stack([m21 - m12, qa[:, 1] ** 2, m10 + m01, m02 + m20], 1),
                        torch.stack([m02 - m20, m10 + m01, qa[:, 2] ** 2, m12 + m21], 1),
                        torch.stack([m10 - m01, m20 + m02, m21 + m12, qa[:, 3] ** 2], 1)], 1)
    k = qa.argmax(1)
    q = cand[torch.arange(m.shape[0], device=m.device), k] / (2 * qa.gather(1, k[:, None]).clamp_min(0.1))
    half = torch.atan2(q[:, 1:].norm(dim=1), q[:, 0])
    ang = 2 * half
    s = torch.where(ang.abs() < 1e-6, 0.5 - ang * ang / 48, torch.sin(half) / ang).clamp_min(torch.finfo(m.dtype).tiny)
    return (q[:, 1:] / s[:, None]).norm(dim=1)


def torch_loss(pred: Dict[str, torch.Tensor], gt: Dict[str, torch.Tensor], valid_3d: torch.Tensor, tals: bool,
               loose_weight: float = LOOSE_WEIGHT, weights: Dict[str, float] = LOSS_WEIGHTS, pelvis_id: int = 39):
    """compute_loss's arithmetic in plain torch ops (no host round trip, no in-place write to gt).  pred: the five
    PRED_KEYS; gt: gt_keypoints_2d / 3d, gt_global_orient, gt_body_pose, gt_betas, has_*.  Returns the six terms."""
    B = pred["pred_keypoints_2d"].shape[0]
    dt, dev = pred["pred_keypoints_2d"].dtype, pred["pred_keypoints_2d"].device
    p2, g2 = pred["pred_keypoints_2d"], gt["gt_keypoints_2d"]
    p3, g3 = pred["pred_keypoints_3d"], gt["gt_keypoints_3d"]
    c = g2[..., 2]
    l1 = (p2 - g2[..., :2]).abs()
    c3 = g3[..., 3]
    if tals:
        thr2 = torch.tensor(KP2D_ERR_THRESH, dtype=torch.float32, device=dev)
        valid = c * ((p2 - g2[..., :2]) ** 2).sum(2) > thr2
        cm = c * valid
        l2 = (cm[..., None] * l1).sum() + loose_weight * ((c * ~valid)[..., None] * l1).sum()
        c3 = c3 * ((valid_3d[:, None] + cm) > 0.5)
    else:
        l2 = (c[..., None] * l1).sum()
    e3 = (p3 - p3[:, pelvis_id:pelvis_id + 1]) - (g3[..., :3] - g3[:, pelvis_id:pelvis_id + 1, :3])
    l3 = (c3[..., None] * e3.abs()).sum()
    thr = {"global_orient": torch.tensor([0.46], dtype=torch.float32, device=dev),
           "body_pose": torch.tensor(BODY_ANGLE_THRESH, dtype=torch.float32, device=dev) * 0.8}
    terms = {}
    for k in ("global_orient", "body_pose"):
        P = pred["pred_" + k]
        G = _aa_to_rotmat(gt["gt_" + k].reshape(-1, 3)).view(P.shape)
        e = ((P - G) ** 2).sum((2, 3))
        has = gt["has_" + k][:, None]
        if tals:
            valid = _angle(P.reshape(-1, 3, 3) @ G.reshape(-1, 3, 3).transpose(1, 2)).view(B, -1) > thr[k]
            mask = (valid * has + valid_3d[:, None]).bool()
            terms[k] = (mask * e).sum() + loose_weight * ((~mask * has) * e).sum()
        else:
            terms[k] = (has * e).sum()
    hb = gt["has_betas"] * valid_3d if tals else gt["has_betas"]
    terms["betas"] = (hb[:, None] * (pred["pred_betas"] - gt["gt_betas"]) ** 2).sum()
    loss = weights["KEYPOINTS_3D"] * l3 + weights["KEYPOINTS_2D"] * l2 + \
        sum(terms[k] * weights[k.upper()] for k in ("global_orient", "body_pose", "betas"))
    return torch.stack([loss, l2, l3, terms["global_orient"], terms["body_pose"], terms["betas"]]).to(dt)

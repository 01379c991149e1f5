"""SMPLify-inverse golden: the LIVE reference lib/utils/smplify_invert.py (loaded file by file through
oracle/ref_import.py; it needs only geometry.py and rotation_utils.py) run on the CPU in fp64, with
oracle.smpl_oracle.smpl_forward on synth.make_smpl(release_config()) as its body model.  TEST INFRASTRUCTURE ONLY.

    TOKENHMR_REFERENCE=<checkout> python -m oracle.smplify_oracle      # writes tests/golden/smplify_inv.npz

Two seeded cases (B = 4, 30 iterations): (a) default thresholds, every iteration runs; (b) step size 5e-3 and
thresholds that stop the loop mid-run, with the crossing asserted to be at least 1e-3 relative away from every
iteration's loss (so fp32 cannot move the break).  Per case: the inputs, per iteration the parameters the body model
was called with and the gradients left by loss.backward() (both stored in fp32), loss, fit2D and mean push3D, the break iteration (-1 when none)
and the outputs (vertices every VERT_STRIDE-th).

The per-iteration values are recorded without touching the reference's code: the body model passed in records its
inputs and the gradients of the previous iteration, and the module's camera_fitting_loss is wrapped to record fit2D.
push3D and loss are the two lines of smplify_invert.py:127-128 evaluated on the recorded joints.
"""
from __future__ import annotations

import importlib
import types
from pathlib import Path
from typing import Dict

import numpy as np
import torch

from oracle import ref_import
from oracle import smpl_oracle as S

GOLDEN = Path(__file__).resolve().parent.parent / "tests" / "golden" / "smplify_inv.npz"
B, NUM_ITERS, VERT_STRIDE, MARGIN = 4, 30, 53, 20.0
CASES = {"a": dict(seed=11, step_size=1e-3), "b": dict(seed=12, step_size=5e-3)}
BREAK_AT = 15          # case (b): the loop stops here
CROSS_REL = 1e-3       # case (b): |loss_i - thresh| >= CROSS_REL |thresh| for every iteration up to the break
FOCAL = 5000.0


def body_model():
    from tokenhmr_b200 import synth
    from tokenhmr_b200.config import release_config
    smpl = synth.make_smpl(release_config())
    return {k: (v.double() if v.is_floating_point() else v) for k, v in smpl.items()}


def smpl_callable(smpl64):
    """The reference SMPL wrapper's call surface on the fp64 oracle: rotation matrices in, .vertices / .joints out."""
    def call(global_orient, body_pose, betas, pose2rot=False):
        v, j = S.smpl_forward(smpl64, global_orient, body_pose, betas, dtype=torch.float64)
        return types.SimpleNamespace(vertices=v, joints=j)
    return call


def make_inputs(smpl64, seed: int) -> Dict[str, torch.Tensor]:
    """fp32-representable fp64 inputs: a start pose, 2D keypoints projected from a nearby pose (plus noise) and 3D
    keypoints from another pose.  Rotation matrices come from Rodrigues of random axis-angles."""
    g = torch.Generator().manual_seed(seed)
    f32 = lambda t: t.float().double()
    rot = lambda aa: S.batch_rodrigues(aa.reshape(-1, 3)).view(B, 24, 3, 3)
    aa = 0.3 * torch.randn(B, 24, 3, generator=g, dtype=torch.float64)
    R = f32(rot(aa))
    betas = f32(torch.randn(B, 10, generator=g, dtype=torch.float64))
    s = 0.8 + 0.2 * torch.rand(B, generator=g, dtype=torch.float64)
    cam_t = f32(torch.stack([0.1 * torch.randn(B, generator=g, dtype=torch.float64),
                             0.1 * torch.randn(B, generator=g, dtype=torch.float64), 2 * FOCAL / (256 * s)], 1))
    focal = torch.full((B, 2), FOCAL, dtype=torch.float64)
    _, j2 = S.smpl_forward(smpl64, rot(aa + 0.2 * torch.randn(aa.shape, generator=g, dtype=torch.float64))[:, :1],
                           rot(aa + 0.2 * torch.randn(aa.shape, generator=g, dtype=torch.float64))[:, 1:], betas,
                           dtype=torch.float64)
    p = j2 + cam_t[:, None]
    kp2 = (FOCAL / 256) * p[..., :2] / p[..., 2:] + 0.01 * torch.randn(B, 44, 2, generator=g, dtype=torch.float64)
    conf = torch.rand(B, 44, 1, generator=g, dtype=torch.float64)
    aa3 = 0.3 * torch.randn(B, 24, 3, generator=g, dtype=torch.float64)
    _, j3 = S.smpl_forward(smpl64, rot(aa3)[:, :1], rot(aa3)[:, 1:], betas, dtype=torch.float64)
    return dict(global_orient=R[:, :1].contiguous(), body_pose=R[:, 1:].contiguous(), betas=betas, pred_cam_t=cam_t,
                focal_length=focal, gt_keypoints_2d=f32(torch.cat([kp2, conf], -1)),
                gt_keypoints_3d=f32(j3 + 0.02 * torch.randn(j3.shape, generator=g, dtype=torch.float64)))


def run_reference(smpl64, inputs: Dict[str, torch.Tensor], step_size: float, f2d: float, f3d: float) -> Dict[str, np.ndarray]:
    """One live reference SMPLifyInv call with recording hooks; returns the golden arrays of one case."""
    ref_import.load_modules()
    mod = importlib.import_module("lib.utils.smplify_invert")
    x = {k: v.clone() for k, v in inputs.items()}
    go, bp, cam = x["global_orient"], x["body_pose"], x["pred_cam_t"]
    rec = {k: [] for k in ("go", "bp", "cam", "g_go", "g_bp", "g_cam", "joints", "fit2d")}
    model = smpl_callable(smpl64)
    seen = [None]

    def recording(global_orient, body_pose, betas, pose2rot=False):
        # gradients of the previous iteration's loss.backward(): zero_grad() sets .grad to None, so a new tensor is
        # a new step (after a break the final pass finds the last step's gradient again)
        if go.grad is not None and go.grad is not seen[0]:
            seen[0] = go.grad
            rec["g_go"].append(go.grad.clone()); rec["g_bp"].append(bp.grad.clone()); rec["g_cam"].append(cam.grad.clone())
        rec["go"].append(go.detach().clone()); rec["bp"].append(bp.detach().clone()); rec["cam"].append(cam.detach().clone())
        out = model(global_orient, body_pose, betas)
        rec["joints"].append(out.joints.detach().clone())
        return out

    live_loss = mod.camera_fitting_loss

    def fit_loss(*a, **k):
        v = live_loss(*a, **k)
        rec["fit2d"].append(v.detach().clone())
        return v

    mod.camera_fitting_loss = fit_loss
    try:
        fit = mod.SMPLifyInv(recording, step_size=step_size, num_iters=NUM_ITERS, margin=MARGIN, loss_thresh_f2d=f2d,
                             loss_thresh_f3d=f3d, device=torch.device("cpu"))
        out = fit(go, bp, x["betas"], cam, x["focal_length"], x["gt_keypoints_2d"], x["gt_keypoints_3d"])
    finally:
        mod.camera_fitting_loss = live_loss
    n_loop = len(rec["go"]) - 1                      # the last call is the final no-grad pass
    steps = len(rec["g_go"])
    fit2d = torch.stack(rec["fit2d"][:n_loop])
    push = torch.stack([torch.sqrt(((j - x["gt_keypoints_3d"]) ** 2).sum(2)).sum(1).mean() for j in rec["joints"][:n_loop]])
    loss = 4 * fit2d - push / 2 + MARGIN
    broke = steps < n_loop
    vertices, joints, pj2ds, go_o, bp_o, _, cam_o, reproj = out
    st = lambda xs: torch.stack(xs).float().numpy()     # per-iteration parameters and gradients: fp32 is enough
    return dict(
        global_orient_it=st(rec["go"][:n_loop]), body_pose_it=st(rec["bp"][:n_loop]), pred_cam_t_it=st(rec["cam"][:n_loop]),
        grad_global_orient_it=st(rec["g_go"]), grad_body_pose_it=st(rec["g_bp"]), grad_pred_cam_t_it=st(rec["g_cam"]),
        loss_it=loss.numpy(), fit2d_it=fit2d.numpy(), push3d_it=push.numpy(),
        break_iter=np.array(n_loop - 1 if broke else -1), steps=np.array(steps),
        vertices_sub=vertices[:, ::VERT_STRIDE].numpy(), joints=joints.numpy(), pj2ds=pj2ds.detach().numpy(),
        global_orient_out=go_o.numpy(), body_pose_out=bp_o.detach().numpy(), pred_cam_t_out=cam_o.detach().numpy(),
        reprojection_loss=reproj.detach().numpy())


def build_cases(smpl64) -> Dict[str, np.ndarray]:
    arrays: Dict[str, np.ndarray] = {}
    for name, c in CASES.items():
        x = make_inputs(smpl64, c["seed"])
        f2d, f3d = 1.0, 0.0
        if name == "b":
            probe = run_reference(smpl64, x, c["step_size"], 1e9, -1e9)
            loss = probe["loss_it"]
            f2d = 1e9
            f3d = 0.5 * (loss[BREAK_AT - 1] + loss[BREAK_AT])
            assert (loss[:BREAK_AT] - f3d >= CROSS_REL * abs(f3d)).all(), "case (b): earlier iterations too close"
            assert f3d - loss[BREAK_AT] >= CROSS_REL * abs(f3d), "case (b): the crossing is too narrow"
        got = run_reference(smpl64, x, c["step_size"], f2d, f3d)
        if name == "b":
            assert int(got["break_iter"]) == BREAK_AT
        else:
            assert int(got["break_iter"]) == -1
        cfg = np.array([c["step_size"], NUM_ITERS, MARGIN, f2d, f3d, VERT_STRIDE], np.float64)
        arrays.update({f"{name}_{k}": v.numpy() for k, v in x.items()})
        arrays.update({f"{name}_{k}": v for k, v in got.items()})
        arrays[f"{name}_config"] = cfg
    return arrays


def main() -> None:
    arrays = build_cases(body_model())
    np.savez_compressed(GOLDEN, **arrays)
    print(f"wrote {GOLDEN}")


if __name__ == "__main__":
    main()

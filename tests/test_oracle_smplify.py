"""SMPLify-inverse without a GPU: the golden (tests/golden/smplify_inv.npz, written from the live reference
smplify_invert.py by oracle/smplify_oracle.py) against a fresh reference run, and tokenhmr_b200.fitting.SMPLifyInv
driven by the fp64 oracle body model against the golden.  Also the backward entry points' ctypes signatures against the
header."""
import re
from pathlib import Path

import numpy as np
import pytest
import torch

from oracle import smplify_oracle as SO

ROOT = Path(__file__).resolve().parent.parent
GOLD = "smplify_inv.npz"


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(golden_dir / GOLD)


@pytest.fixture(scope="module")
def smpl64():
    return SO.body_model()


def _inputs(golden, case):
    names = ("global_orient", "body_pose", "betas", "pred_cam_t", "focal_length", "gt_keypoints_2d", "gt_keypoints_3d")
    return {n: torch.from_numpy(golden[f"{case}_{n}"].copy()) for n in names}


def test_golden_equals_fresh_reference_run(smpl64, golden):
    from oracle import ref_import
    if not ref_import.available():
        pytest.skip("reference checkout not configured (TOKENHMR_REFERENCE)")
    fresh = SO.build_cases(smpl64)
    assert set(fresh) == set(golden.files)
    for k, v in fresh.items():
        assert np.array_equal(v, golden[k]), k


def test_inputs_are_the_seeded_ones(smpl64, golden):
    """The stored inputs are what make_inputs gives (so a fresh run starts from the same point)."""
    for case, c in SO.CASES.items():
        x = SO.make_inputs(smpl64, c["seed"])
        for k, v in x.items():
            assert np.array_equal(v.numpy(), golden[f"{case}_{k}"]), (case, k)


@pytest.mark.parametrize("case", list(SO.CASES))
def test_fitting_with_oracle_body_model_matches_golden(smpl64, golden, case):
    """fitting.SMPLifyInv on the fp64 oracle body model: per-iteration loss, fit2D and push3D, the break iteration and
    every output within 1e-12 of the reference's."""
    from tokenhmr_b200.fitting import SMPLifyInv
    step, iters, margin, f2d, f3d, stride = golden[f"{case}_config"]
    x = _inputs(golden, case)
    fit = SMPLifyInv(SO.smpl_callable(smpl64), step_size=float(step), num_iters=int(iters), margin=float(margin),
                     loss_thresh_f2d=float(f2d), loss_thresh_f3d=float(f3d), device=torch.device("cpu"))
    go, bp, cam = x["global_orient"], x["body_pose"], x["pred_cam_t"]
    out = fit(go, bp, x["betas"], cam, x["focal_length"], x["gt_keypoints_2d"], x["gt_keypoints_3d"])
    hist = torch.tensor([[float(t) for t in h] for h in fit.history], dtype=torch.float64).numpy()
    n = len(golden[f"{case}_loss_it"])
    assert hist.shape[0] == n
    close = lambda a, b: np.testing.assert_allclose(a, b, rtol=1e-12, atol=1e-12)
    close(hist[:, 0], golden[f"{case}_loss_it"])
    close(hist[:, 1], golden[f"{case}_fit2d_it"])
    close(hist[:, 2], golden[f"{case}_push3d_it"])
    broke = int(golden[f"{case}_break_iter"])
    assert (n - 1 if n < int(iters) or broke >= 0 else -1) == broke
    vertices, joints, pj2ds, go_o, bp_o, betas_o, cam_o, reproj = out
    close(vertices[:, ::int(stride)].numpy(), golden[f"{case}_vertices_sub"])
    close(joints.numpy(), golden[f"{case}_joints"])
    close(pj2ds.detach().numpy(), golden[f"{case}_pj2ds"])
    close(go_o.numpy(), golden[f"{case}_global_orient_out"])
    close(bp_o.numpy(), golden[f"{case}_body_pose_out"])
    close(cam_o.detach().numpy(), golden[f"{case}_pred_cam_t_out"])
    close(reproj.numpy(), golden[f"{case}_reprojection_loss"])
    # the caller's tensors are the optimised ones (updated in place, as in the reference)
    assert torch.equal(go.detach(), go_o)
    close(bp.detach().numpy(), golden[f"{case}_body_pose_out"])
    close(cam.detach().numpy(), golden[f"{case}_pred_cam_t_out"])


def _prototype(name):
    text = re.sub(r"/\*.*?\*/", "", (ROOT / "include" / "tokenhmr_b200.h").read_text(), flags=re.S)
    m = re.search(rf"\b(\w+\*?)\s+{name}\s*\(([^)]*)\)", text)
    return m.group(1), [a.strip() for a in m.group(2).split(",")]


@pytest.mark.parametrize("name", ["thmr_smpl_backward_workspace_bytes", "thmr_smpl_backward", "thmr_lbs_backward"])
def test_backward_prototypes_match_ctypes(name):
    import ctypes
    from tokenhmr_b200._lib import SIGNATURES
    ret, args = _prototype(name)
    res, argtypes = SIGNATURES[name]
    assert len(args) == len(argtypes)
    assert res is (ctypes.c_size_t if ret == "size_t" else ctypes.c_int)
    for a, t in zip(args, argtypes):
        if "*" in a:
            assert t is ctypes.c_void_p, a
        else:
            assert t is ctypes.c_int, a

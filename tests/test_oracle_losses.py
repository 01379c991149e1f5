"""The training loss without a GPU: the golden (tests/golden/tals_loss.npz, written from the live reference losses.py by
oracle/loss_oracle.py) against a fresh reference run, the plain-torch restatement that scripts/bench_tals_loss.py times
against the golden, and the new C entry points and descriptor against their ctypes mirrors."""
import ctypes
import re
import shutil
import subprocess
from pathlib import Path

import numpy as np
import pytest
import torch

from oracle import loss_oracle as LO

ROOT = Path(__file__).resolve().parent.parent
HEADER = ROOT / "include" / "tokenhmr_b200.h"


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(golden_dir / "tals_loss.npz")


def test_golden_equals_fresh_reference_run(golden):
    from oracle import ref_import
    if not ref_import.available():
        pytest.skip("reference checkout not configured (TOKENHMR_REFERENCE)")
    fresh = LO.build_cases()
    assert set(fresh) == set(golden.files)
    for k, v in fresh.items():
        assert np.array_equal(v, golden[k]), k


def test_golden_covers_both_sides_of_every_decision(golden):
    """Both branches are stored, with zero / fractional / unit confidences, has_smpl_params 0 and 1, and valid_3d 0 and
    1 in every combination with has_smpl_params, so the TALS branch's masks take both values.  The TALS case holds the
    reference's two quirks, visible in its gradients: a valid_3D sample without pose parameters still gets the pose
    loss (at full weight), and a valid_3D sample without betas gets no betas loss (the gate is has * valid_3D)."""
    for case in LO.CASES:
        c2 = golden[f"{case}_gt_keypoints_2d"][..., 2]
        assert (c2 == 0).any() and (c2 == 1).any() and ((c2 > 0) & (c2 < 1)).any()
        v3d = golden[f"{case}_valid_3d"]
        assert np.array_equal(v3d, [float(n in ("H36M-TRAIN-WMASK", "BEDLAM")) for n in golden[f"{case}_dataset"]])
        for k in ("has_global_orient", "has_body_pose", "has_betas"):
            has = golden[f"{case}_{k}"]
            assert set(np.unique(has)) == {0.0, 1.0}
            for v in (0.0, 1.0):
                for h in (0.0, 1.0):
                    assert ((v3d == v) & (has == h)).any(), (case, k, v, h)
        assert np.isfinite(golden[f"{case}_losses"]).all()
    v3d = golden["tals_valid_3d"]
    no_pose = (v3d == 1) & (golden["tals_has_body_pose"] == 0) & (golden["tals_has_global_orient"] == 0)
    no_betas = (v3d == 1) & (golden["tals_has_betas"] == 0)
    for k in ("global_orient", "body_pose"):
        g = np.abs(golden[f"tals_grad_{k}"]).reshape(len(v3d), -1).max(1)
        assert (g[no_pose] > 0).all(), k
    g = np.abs(golden["tals_grad_betas"]).max(1)
    assert (g[no_betas] == 0).all() and (g[(v3d == 1) & (golden["tals_has_betas"] == 1)] > 0).all()
    assert (g[v3d == 0] == 0).all()           # has * valid_3D is 0 for every sample outside the two datasets


@pytest.mark.parametrize("case", list(LO.CASES))
def test_torch_restatement_matches_golden(golden, case):
    """oracle.loss_oracle.torch_loss (the timing baseline) gives the golden's terms and gradients in fp64."""
    pred = {k: torch.from_numpy(golden[f"{case}_{k}"].copy()).requires_grad_(True) for k in LO.PRED_KEYS}
    gt_keys = ("gt_keypoints_2d", "gt_keypoints_3d", "gt_global_orient", "gt_body_pose", "gt_betas",
               "has_global_orient", "has_body_pose", "has_betas")
    gt = {k: torch.from_numpy(golden[f"{case}_{k}"].copy()) for k in gt_keys}
    tals = bool(golden[f"{case}_config"][1])
    terms = LO.torch_loss(pred, gt, torch.from_numpy(golden[f"{case}_valid_3d"].copy()), tals)
    np.testing.assert_allclose(terms.detach().numpy(), golden[f"{case}_losses"], rtol=1e-12)
    grads = torch.autograd.grad(terms[0], [pred[k] for k in LO.PRED_KEYS])
    for k, g in zip(LO.PRED_KEYS, grads):
        np.testing.assert_allclose(g.numpy(), golden[f"{case}_grad_{k[len('pred_'):]}"], rtol=1e-12, atol=1e-15)


def _prototype(name):
    text = re.sub(r"/\*.*?\*/", "", HEADER.read_text(), flags=re.S)
    m = re.search(rf"\b(\w+\*?)\s+{name}\s*\(([^)]*)\)", text)
    return m.group(1), [a.strip() for a in m.group(2).split(",")]


@pytest.mark.parametrize("name", ["thmr_camera_tail", "thmr_camera_tail_backward",
                                  "thmr_tokenhmr_loss_workspace_bytes", "thmr_tokenhmr_loss"])
def test_prototypes_match_ctypes(name):
    from tokenhmr_b200 import _lib
    ret, args = _prototype(name)
    res, argtypes = _lib.SIGNATURES[name]
    assert len(args) == len(argtypes)
    assert res is (ctypes.c_size_t if ret == "size_t" else ctypes.c_int)
    for a, t in zip(args, argtypes):
        if a.startswith("const thmr_loss_desc*"):
            assert t is ctypes.POINTER(_lib.LossDesc), a
        elif "*" in a:
            assert t is ctypes.c_void_p, a
        elif a.startswith("float"):
            assert t is ctypes.c_float, a
        else:
            assert t is ctypes.c_int, a


def test_loss_desc_fields_in_header_order():
    from tokenhmr_b200 import _lib
    body = re.search(r"typedef struct thmr_loss_desc \{(.*?)\} thmr_loss_desc;", HEADER.read_text(), re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    assert re.findall(r"\b([A-Za-z_0-9]+)\s*(?=[,;])", body) == [n for n, _ in _lib.LossDesc._fields_]


def test_loss_desc_size_matches_c(tmp_path):
    from tokenhmr_b200 import _lib
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("no C compiler")
    src = tmp_path / "size.c"
    src.write_text(f'#include <stdio.h>\n#include "{HEADER}"\n'
                   'int main(void) { printf("%zu", sizeof(thmr_loss_desc)); return 0; }\n')
    exe = tmp_path / "size"
    subprocess.run([gcc, "-std=c99", "-Wall", "-Werror", "-o", str(exe), str(src)], check=True, capture_output=True)
    assert int(subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout) == \
        ctypes.sizeof(_lib.LossDesc)


def test_loss_workspace_is_arithmetic(built_lib):
    assert built_lib.thmr_tokenhmr_loss_workspace_bytes(0) == 0
    assert built_lib.thmr_tokenhmr_loss_workspace_bytes(48) >= 48 * 5 * 8


def test_loss_rejects_bad_descriptors_without_a_gpu(built_lib):
    """Argument checks run before any CUDA call.  Every pointer is set (to an address never dereferenced), so each
    descriptor breaks exactly one rule, and the error message names that rule."""
    from tokenhmr_b200 import _lib
    ws = ctypes.c_void_p(16)
    cases = ((dict(B=0), "B=0"), (dict(num_joints=43, tals=1), "needs 44 keypoints"),
             (dict(pelvis_id=44), "pelvis_id 44 outside"), (dict(num_betas=11), "num_betas 11"),
             (dict(tals=2), "tals 2"), (dict(valid_3d=None, tals=1), "missing input"),
             (dict(grad_betas=None), "all set or all NULL"))
    for fields, msg in cases:
        d = _lib.LossDesc(B=4, num_joints=44, num_betas=10, tals=0, pelvis_id=39)
        for name, typ in _lib.LossDesc._fields_:
            if typ is ctypes.c_void_p:
                setattr(d, name, 4096)
        for k, v in fields.items():
            setattr(d, k, v)
        assert built_lib.thmr_tokenhmr_loss(ctypes.byref(d), ws, None) == -1, fields
        assert msg in built_lib.thmr_last_error().decode(), (fields, built_lib.thmr_last_error())

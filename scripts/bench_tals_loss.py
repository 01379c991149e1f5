"""Forward + backward of TokenHMR's training loss: the fused CUDA call (tokenhmr_b200.losses.TokenHMRLoss) against the
same loss restated in plain torch ops (oracle.loss_oracle.torch_loss, fp32, on the same GPU), with CUDA events, at
B = 48 (TRAIN.BATCH_SIZE of the release config) and B = 512, in the TALS (training) and plain (validation) branches.
Inputs are the golden's cases tiled to B.  The torch arm reads valid_3d as a device tensor, as the fused call does, so
neither arm pays the reference's host round trips; the reference itself adds three .all() reads and a host-to-device
copy per step.  Prints one JSON line with the card's name, power limit and SM clock.

    python scripts/bench_tals_loss.py [--iters 200] [--warmup 20]
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

from oracle import loss_oracle as LO  # noqa: E402
from tokenhmr_b200.losses import TokenHMRLoss  # noqa: E402

GT_KEYS = ("gt_keypoints_2d", "gt_keypoints_3d", "gt_global_orient", "gt_body_pose", "gt_betas", "has_global_orient",
           "has_body_pose", "has_betas")


def inputs(golden, case, B, dev):
    reps = -(-B // golden[f"{case}_pred_betas"].shape[0])
    t = lambda k: torch.from_numpy(np.concatenate([golden[f"{case}_{k}"]] * reps)[:B].copy()).float().to(dev)
    pred = {k: t(k).requires_grad_(True) for k in LO.PRED_KEYS}
    gt = {k: t(k) for k in GT_KEYS}
    return pred, gt, t("valid_3d")


def time_ms(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--batches", type=int, nargs="+", default=[48, 512])
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_tals_loss needs a CUDA device")
    dev = torch.device("cuda:0")
    golden = np.load(ROOT / "tests" / "golden" / "tals_loss.npz")
    crit = TokenHMRLoss(loose_sup=True, loose_weight=LO.LOOSE_WEIGHT, loss_weights=LO.LOSS_WEIGHTS)
    res = {}
    for case in LO.CASES:
        tals = bool(golden[f"{case}_config"][1])
        for B in args.batches:
            pred, gt, v3d = inputs(golden, case, B, dev)
            ins = [pred[k] for k in LO.PRED_KEYS]
            batch = {"keypoints_2d": gt["gt_keypoints_2d"], "keypoints_3d": gt["gt_keypoints_3d"],
                     "smpl_params": {k: gt["gt_" + k] for k in ("global_orient", "body_pose", "betas")},
                     "has_smpl_params": {k: gt["has_" + k] for k in ("global_orient", "body_pose", "betas")},
                     "smpl_params_is_axis_angle": {"global_orient": torch.ones(B, dtype=torch.bool, device=dev),
                                                   "body_pose": torch.ones(B, dtype=torch.bool, device=dev),
                                                   "betas": torch.zeros(B, dtype=torch.bool, device=dev)},
                     "dataset": v3d}
            output = {"pred_smpl_params": {"global_orient": pred["pred_global_orient"],
                                           "body_pose": pred["pred_body_pose"], "betas": pred["pred_betas"]},
                      "pred_keypoints_2d": pred["pred_keypoints_2d"], "pred_keypoints_3d": pred["pred_keypoints_3d"]}
            fused = lambda: torch.autograd.grad(crit(batch, output, train=tals), ins)
            ref = lambda: torch.autograd.grad(LO.torch_loss(pred, gt, v3d, tals)[0], ins)
            lf, lr = crit(batch, output, train=tals), LO.torch_loss(pred, gt, v3d, tals)[0]
            rel = abs(lf.item() - lr.item()) / abs(lr.item())
            tf, tr = time_ms(fused, args.iters, args.warmup), time_ms(ref, args.iters, args.warmup)
            tf2 = time_ms(fused, args.iters, args.warmup)    # alternate the arms once more to see the spread
            res[f"{case}_B{B}"] = {"fused_ms": round(min(tf, tf2), 4), "fused_ms_runs": [round(tf, 4), round(tf2, 4)],
                                   "torch_ms": round(tr, 4), "speedup": round(tr / min(tf, tf2), 2),
                                   "loss_rel_diff": float(f"{rel:.3g}")}
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    print(json.dumps({"bench": "tals_loss_fwd_bwd", "gpu": q, "iters": args.iters, "results": res}))


if __name__ == "__main__":
    main()

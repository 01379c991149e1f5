"""Times one 100-iteration SMPLify-inverse call at B in {1, 64, 512} with thresholds that never stop the loop:
FusedSMPLifyInv (thmr_smplify_inv), SMPLifyInv(model.smpl), SMPLifyInv on fp32 torch autograd through
oracle/smpl_oracle.py, and the body model's forward + backward alone (one call, as one iteration runs it).  The variants
alternate within each round; each is timed with CUDA events after a warm-up call, and the median over rounds is
reported.  Prints one JSON line with the card's name and power limit read in the same run.

    python scripts/bench_smplify.py [--rounds 5]
"""
from __future__ import annotations

import argparse
import json
import statistics
import subprocess
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

from oracle import smpl_oracle as S                           # noqa: E402
from tokenhmr_b200 import synth                               # noqa: E402
from tokenhmr_b200.config import release_config               # noqa: E402
from tokenhmr_b200.engine import _SmplFacade                  # noqa: E402
from tokenhmr_b200.fitting import FusedSMPLifyInv, SMPLifyInv  # noqa: E402
from tokenhmr_b200.ops import SMPLModel                       # noqa: E402

ITERS = 100


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[torch.cuda.current_device()] if q else torch.cuda.get_device_name()


def timed(fn, reps):
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(reps):
        fn()
    t1.record()
    torch.cuda.synchronize()
    return t0.elapsed_time(t1) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_smplify.py needs a GPU")
    dev = torch.device("cuda:0")
    smpl = synth.make_smpl(release_config())
    m = SMPLModel(smpl, dev)
    facade = _SmplFacade(m)
    s32 = {k: (v.cuda() if not v.is_floating_point() else v.cuda().float()) for k, v in smpl.items()}

    def oracle_model(global_orient, body_pose, betas, pose2rot=False):
        with torch.device("cuda"):
            v, j = S.smpl_forward(s32, global_orient, body_pose, betas)
        return type("Out", (), {"vertices": v, "joints": j})

    res = {"card": card(), "unit": "ms per call", "iters": ITERS, "rounds": args.rounds}
    g = torch.Generator(device="cuda").manual_seed(0)
    for B in (1, 64, 512):
        with torch.device("cuda"):
            rot = S.batch_rodrigues(0.3 * torch.randn(B * 24, 3, device="cuda", generator=g)).view(B, 24, 3, 3)
        betas = torch.randn(B, 10, device="cuda", generator=g)
        focal = torch.full((B, 2), 5000.0, device="cuda")
        kp2 = torch.cat([0.3 * torch.randn(B, 44, 2, device="cuda", generator=g), torch.ones(B, 44, 1, device="cuda")],
                        -1)
        kp3 = 0.3 * torch.randn(B, 44, 3, device="cuda", generator=g)
        cam0 = torch.tensor([0.0, 0.0, 45.0], device="cuda").expand(B, 3)
        gj = torch.randn(B, 44, 3, device="cuda", generator=g)

        def fit_with(cls, model):
            fit = cls(model, num_iters=ITERS, loss_thresh_f2d=-1.0)

            def run():
                fit(rot[:, :1].clone(), rot[:, 1:].clone(), betas, cam0.clone(), focal, kp2, kp3)
            return run

        go, bp = rot[:, :1].clone().requires_grad_(), rot[:, 1:].clone().requires_grad_()

        def body_fwd_bwd():
            j = m.forward(go, bp, betas)[1]
            torch.autograd.backward(j, gj)

        variants = {"fused": (fit_with(FusedSMPLifyInv, facade), 3), "smplifyinv_engine": (fit_with(SMPLifyInv, facade), 1),
                    "smplifyinv_torch_fp32": (fit_with(SMPLifyInv, oracle_model), 1),
                    "body_fwd_bwd": (body_fwd_bwd, 50)}
        for fn, _ in variants.values():
            fn()                                    # warm-up: module loads, workspaces, torch's allocator
        times = {k: [] for k in variants}
        for _ in range(args.rounds):
            for k, (fn, reps) in variants.items():
                times[k].append(timed(fn, reps))
        row = {k: round(statistics.median(v), 4) for k, v in times.items()}
        row["spread"] = {k: round((max(v) - min(v)) / statistics.median(v), 3) for k, v in times.items()}
        row["fused_per_iter"] = round(row["fused"] / ITERS, 4)
        row["body_fwd_bwd_x100"] = round(row["body_fwd_bwd"] * ITERS, 2)
        res[f"B{B}"] = row
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()

"""Times the SMPL stage's forward and forward + backward (thmr_smpl_forward / thmr_smpl_backward through
SMPLModel's autograd Function) at B in {64, 512, 4096}, and one SMPLifyInv(model.smpl) call at B = 64 with 100
iterations, against fp32 torch.autograd through oracle/smpl_oracle.py on the same GPU (the smplx algorithm in eager
PyTorch).  CUDA events after warm-up; prints one JSON line with the card's name and power limit read in the same run.

    python scripts/bench_smpl_grad.py [--reps 20]
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

from oracle import smpl_oracle as S                      # noqa: E402
from tokenhmr_b200 import synth                          # noqa: E402
from tokenhmr_b200.config import release_config          # noqa: E402
from tokenhmr_b200.engine import _SmplFacade             # noqa: E402
from tokenhmr_b200.fitting import SMPLifyInv             # noqa: E402
from tokenhmr_b200.ops import SMPLModel                  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[torch.cuda.current_device()] if q else torch.cuda.get_device_name()


def timed(fn, reps):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(reps):
        fn()
    t1.record()
    torch.cuda.synchronize()
    return t0.elapsed_time(t1) / reps


def backward_work(V, nb, B):
    """Algorithmic bytes and FLOPs of one backward from shapes: the blend GEMM's recompute (fp16 basis 3V x 672 read
    once per 256-pose chunk, v_posed written and read), the v_posed cotangent written and read, the fp32 basis
    (207 + nb) x 3V read once per chunk, the cotangents read; FLOPs of the recompute (3 products over 218 features),
    the skinning transpose and A_bar sums (~4 x 12 x 2 per vertex and weight) and the 3V x (207 + nb) contraction."""
    chunks = (B + 255) // 256
    nf = 207 + nb
    bytes_ = (chunks * (3 * V * 672 * 2 + nf * 3 * V * 4) + B * (4 * 3 * V * 4 + 3 * V * 4 + 44 * 3 * 4))
    flops = B * (2 * 3 * 218 * 3 * V + V * 4 * (2 * 12 + 2 * 12) + 6 * 3 * V + 2 * nf * 3 * V)
    return bytes_, flops


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    smpl = synth.make_smpl(release_config())
    m = SMPLModel(smpl, dev)
    s32 = {k: (v.cuda() if not v.is_floating_point() else v.cuda().float()) for k, v in smpl.items()}
    res = {"card": card(), "unit": "ms"}
    g = torch.Generator(device="cuda").manual_seed(0)
    for B in (64, 512, 4096):
        with torch.device("cuda"):
            rot = S.batch_rodrigues(0.5 * torch.randn(B * 24, 3, device="cuda", generator=g)).view(B, 24, 3, 3)
        betas = torch.randn(B, 10, device="cuda", generator=g)
        gv = torch.randn(B, m.num_verts, 3, device="cuda", generator=g)
        gj = torch.randn(B, 44, 3, device="cuda", generator=g)
        go, bp = rot[:, :1].clone().requires_grad_(), rot[:, 1:].clone().requires_grad_()

        def fwd():
            with torch.no_grad():
                m.forward(go, bp, betas)

        def fwd_bwd():
            v, j = m.forward(go, bp, betas)
            torch.autograd.backward((v, j), (gv, gj))

        def oracle_fwd_bwd():
            with torch.device("cuda"):
                v, j = S.smpl_forward(s32, go, bp, betas)
            torch.autograd.backward((v, j), (gv, gj))

        def oracle_fwd():
            with torch.no_grad(), torch.device("cuda"):
                S.smpl_forward(s32, go, bp, betas)

        nb_, fl = backward_work(m.num_verts, m.num_betas, B)
        res[f"B{B}"] = {"fwd": timed(fwd, args.reps), "fwd_bwd": timed(fwd_bwd, args.reps),
                        "torch_fp32_fwd": timed(oracle_fwd, args.reps),
                        "torch_fp32_fwd_bwd": timed(oracle_fwd_bwd, args.reps),
                        "bwd_bytes": nb_, "bwd_flops": fl}
        del gv, gj
        torch.cuda.empty_cache()
    # one SMPLifyInv call, B = 64, 100 iterations (thresholds that never stop the loop)
    B = 64
    with torch.device("cuda"):
        rot = S.batch_rodrigues(0.3 * torch.randn(B * 24, 3, device="cuda", generator=g)).view(B, 24, 3, 3)
    betas = torch.randn(B, 10, device="cuda", generator=g)
    focal = torch.full((B, 2), 5000.0, device="cuda")
    kp2 = torch.cat([0.3 * torch.randn(B, 44, 2, device="cuda", generator=g), torch.ones(B, 44, 1, device="cuda")], -1)
    kp3 = 0.3 * torch.randn(B, 44, 3, device="cuda", generator=g)
    cam0 = torch.tensor([0.0, 0.0, 45.0], device="cuda").expand(B, 3)

    def fit_with(model):
        def run():
            fit = SMPLifyInv(model, num_iters=100, loss_thresh_f2d=-1.0)
            fit(rot[:, :1].clone(), rot[:, 1:].clone(), betas, cam0.clone(), focal, kp2, kp3)
        return run

    def oracle_model(global_orient, body_pose, betas, pose2rot=False):
        with torch.device("cuda"):
            v, j = S.smpl_forward(s32, global_orient, body_pose, betas)
        return type("Out", (), {"vertices": v, "joints": j})

    res["smplify_B64_100it"] = {"engine": timed(fit_with(_SmplFacade(m)), 3),
                                "torch_fp32": timed(fit_with(oracle_model), 3)}
    print(json.dumps(res))


if __name__ == "__main__":
    main()

"""Times one training step of HMR 2.0's regression head (forward + backward to every parameter, no feature gradient):
the CUDA head (tokenhmr_b200.heads.RegressionHead) against the same head restated in fp32 torch, which materialises K
and V with cuBLAS as the reference does (oracle.regression_oracle.regression_head_forward).  Both run on the same
features, parity is checked in the same run, and the step is compared with its byte floor: one pass over the features
per layer and direction plus the parameters read twice and their gradients written once.

    python scripts/bench_head_train.py [--batches 48 256] [--iters 20] [--warmup 5]
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))

HBM_BYTES_PER_S = 3.35e12          # H100 SXM5 80 GB HBM3 peak


def _card():
    name = torch.cuda.get_device_name()
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                            capture_output=True, text=True, timeout=20).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        pl = "unknown"
    return name, pl


def _time(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(iters)]
    for a, b in ev:
        a.record()
        fn()
        b.record()
    torch.cuda.synchronize()
    ts = sorted(a.elapsed_time(b) for a, b in ev)
    return ts[len(ts) // 2], ts[0]


def main() -> None:
    from oracle import regression_oracle as R
    from oracle import tokenhmr_oracle as O
    from tokenhmr_b200 import synth
    from tokenhmr_b200.config import tiny_config
    from tokenhmr_b200.heads import RegressionHead
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, nargs="+", default=[48, 256])
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    torch.backends.cuda.matmul.allow_tf32 = False
    dev = torch.device("cuda:0")
    cfg = tiny_config(vit_depth=1, head="transformer_decoder")
    sd = synth.make_state_dict(cfg)
    head = RegressionHead(cfg, sd, dev)
    tparams = {k: v.to(dev).clone().requires_grad_("init_" not in k) for k, v in sd.items() if k.startswith("smpl_head.")}
    n_params = sum(p.numel() for p in head.parameters())
    name, pl = _card()
    print(f"# {name}, power limit {pl}; decoder depth {cfg.dec_depth}, {n_params / 1e6:.1f} M parameters")
    for B in args.batches:
        g = torch.Generator(device="cpu").manual_seed(B)
        feats = torch.randn(B, cfg.vit_dim, cfg.grid_h, cfg.grid_w, generator=g).to(dev)
        up = torch.randn(B, 24, 3, 3, generator=g).to(dev)

        def cuda_step():
            head.zero_grad(set_to_none=True)
            p, cam, _ = head(feats)
            loss = (torch.cat([p["global_orient"], p["body_pose"]], 1) * up).sum() + p["betas"].sum() + cam.sum()
            loss.backward()

        def torch_step():
            for v in tparams.values():
                v.grad = None
            p, cam, _ = R.regression_head_forward(tparams, feats.flatten(2).transpose(1, 2), cfg, O.Numerics(False))
            loss = (torch.cat([p["global_orient"], p["body_pose"]], 1) * up).sum() + p["betas"].sum() + cam.sum()
            loss.backward()

        cuda_step()
        torch_step()
        worst = 0.0
        for k, p in head.named_parameters():
            ref = tparams["smpl_head." + k].grad
            ref = torch.zeros_like(p) if ref is None else ref
            worst = max(worst, ((p.grad - ref).abs().max() / ref.abs().max().clamp_min(1e-30)).item())
        t_cuda, t_cuda_min = _time(cuda_step, args.iters, args.warmup)
        t_torch, _ = _time(torch_step, args.iters, args.warmup)
        # the same CUDA step captured in a CUDA graph: the kernels' time without the host's launch cost
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            cuda_step()
        torch.cuda.current_stream().wait_stream(s)
        head.zero_grad(set_to_none=True)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            p, cam, _ = head(feats)
            loss = (torch.cat([p["global_orient"], p["body_pose"]], 1) * up).sum() + p["betas"].sum() + cam.sum()
            loss.backward()
        t_graph, _ = _time(graph.replay, args.iters, args.warmup)
        feat_bytes = B * cfg.vit_dim * cfg.num_tokens * 4
        floor_bytes = 2 * cfg.dec_depth * feat_bytes + 3 * n_params * 4
        floor_ms = floor_bytes / HBM_BYTES_PER_S * 1e3
        res = {"B": B, "cuda_ms": round(t_cuda, 3), "cuda_min_ms": round(t_cuda_min, 3), "cuda_graph_ms": round(t_graph, 3),
               "torch_fp32_ms": round(t_torch, 3),
               "speedup": round(t_torch / t_cuda, 2), "byte_floor_ms": round(floor_ms, 3),
               "floor_fraction_graph": round(floor_ms / t_graph, 3), "worst_grad_rel_vs_torch": float(f"{worst:.2e}")}
        print(json.dumps(res))


if __name__ == "__main__":
    main()

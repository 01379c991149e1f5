"""Times one training step of TokenHMR's token head (forward + backward to every trainable parameter, no feature or
tokenizer gradient): the CUDA head (tokenhmr_b200.heads.TokenHead), eager and as a CUDA graph, against the same head
restated in fp32 torch (oracle.tokenhmr_oracle.head_forward with autograd, cuBLAS / cuDNN underneath), in the same call
on the same features.  Also prints the step's FLOPs and compulsory bytes computed from the shapes, a torch.profiler
split of the CUDA step's kernel time (from a separate run), and the card's name and power limit.

    python scripts/bench_token_head_train.py [--batches 48 256] [--iters 20] [--warmup 5] [--out DIR]
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
from collections import defaultdict
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))

HBM_BYTES_PER_S = 3.35e12          # H100 SXM5 80 GB HBM3 data-sheet peak
FP32_FLOPS = 67e12                 # H100 SXM5 dense FP32 data-sheet peak


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


def step_cost(cfg, B: int, n_params: int, n_tok: int):
    """(FLOPs, bytes) of one forward + backward from the shapes: 2 flops per multiply-add, the backward twice the
    forward's contractions for trainable layers (input and weight gradient) and once for the frozen tokenizer (input
    gradient only); bytes: the features read once per decoder layer and direction, the parameters read twice and
    their gradients written once, the tokenizer read twice, and P (B x 160 x 2048) written, read and its gradient
    written and read."""
    E, C, T, L = cfg.dec_dim, cfg.vit_dim, cfg.num_tokens, cfg.dec_depth
    I, M = cfg.dec_inner, cfg.dec_mlp_dim
    dec = L * (E * I + E * I + 2 * C * I + E * I + E * M * 2 + 2 * T * C * cfg.dec_heads)   # per image, fwd macs
    tn, h = cfg.token_num, cfg.cls_hidden
    cls = E * tn * h + cfg.cls_blocks * (2 * h * tn * cfg.cls_token_inter + 2 * tn * h * cfg.cls_hidden_inter) + \
        tn * h * h + tn * h * cfg.token_class_num
    W = cfg.tok_width
    lens = [tn] + cfg.upsample_sizes
    tok = tn * cfg.nb_code * cfg.code_dim + tn * W * cfg.code_dim * 3 + \
        sum(l * W * W * 3 for l in lens[1:]) + cfg.tok_joints * W * W * (3 + 1) * cfg.tok_depth + \
        cfg.tok_joints * W * W * 3 + cfg.tok_joints * 6 * W * 3
    flops = 2 * B * (3 * (dec + cls) + 2 * tok)
    nbytes = 4 * (2 * L * B * C * T + 3 * n_params + 2 * n_tok + 4 * B * tn * cfg.token_class_num)
    return flops, nbytes


def main() -> None:
    from oracle import tokenhmr_oracle as O
    from tokenhmr_b200 import synth
    from tokenhmr_b200.config import tiny_config
    from tokenhmr_b200.heads import TokenHead
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, nargs="+", default=[48, 256])
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", default=None, help="directory for the profiler's kernel table")
    args = ap.parse_args()
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    dev = torch.device("cuda:0")
    cfg = tiny_config(vit_depth=1)
    sd = synth.make_state_dict(cfg)
    head = TokenHead(cfg, sd, dev)
    tparams = {k: v.to(dev).clone().requires_grad_(k.startswith("smpl_head.") and "init_" not in k)
               for k, v in sd.items() if k.startswith(("smpl_head.", "tokenizer."))}
    n_params = sum(p.numel() for p in head.parameters())
    n_tok = head._tokenizer.numel()
    name, pl = _card()
    print(f"# {name}, power limit {pl}; decoder depth {cfg.dec_depth}, {n_params / 1e6:.1f} M trainable parameters, "
          f"{n_tok / 1e6:.1f} M frozen tokenizer floats")
    for B in args.batches:
        g = torch.Generator(device="cpu").manual_seed(B)
        feats = torch.randn(B, cfg.vit_dim, cfg.grid_h, cfg.grid_w, generator=g).to(dev)
        up = torch.randn(B, 24, 3, 3, generator=g).to(dev)
        up_cls = torch.randn(B, cfg.token_num, cfg.token_class_num, generator=g).to(dev) * 1e-3

        def loss_of(p, cam, probs):
            return (torch.cat([p["global_orient"], p["body_pose"]], 1) * up).sum() + p["betas"].sum() + cam.sum() + \
                (probs * up_cls).sum()

        def cuda_step():
            head.zero_grad(set_to_none=True)
            p, cam, lst = head(feats)
            loss_of(p, cam, lst["cls_logits_softmax"]).backward()

        def torch_step():
            for v in tparams.values():
                v.grad = None
            p, cam, aux = O.head_forward(tparams, feats.flatten(2).transpose(1, 2), cfg, O.Numerics(False))
            loss_of(p, cam, aux["cls_logits_softmax"]).backward()

        cuda_step()
        torch_step()
        worst = 0.0
        for k, p in head.named_parameters():
            ref = tparams["smpl_head." + k].grad
            ref = torch.zeros_like(p) if ref is None else ref
            worst = max(worst, ((p.grad - ref).abs().max() / ref.abs().max().clamp_min(1e-30)).item())
        t_cuda, t_cuda_min = _time(cuda_step, args.iters, args.warmup)
        t_torch, _ = _time(torch_step, args.iters, args.warmup)
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            cuda_step()
        torch.cuda.current_stream().wait_stream(s)
        head.zero_grad(set_to_none=True)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            p, cam, lst = head(feats)
            loss_of(p, cam, lst["cls_logits_softmax"]).backward()
        t_graph, _ = _time(graph.replay, args.iters, args.warmup)
        del graph
        flops, nbytes = step_cost(cfg, B, n_params, n_tok)
        floor_ms = max(flops / FP32_FLOPS, nbytes / HBM_BYTES_PER_S) * 1e3
        # where the time goes: kernel time by name, from a profiled run of its own
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(3):
                cuda_step()
            torch.cuda.synchronize()
        by = defaultdict(float)
        for e in prof.key_averages():
            if e.device_type.name == "CUDA":
                by[e.key.split("<")[0].split("(")[0]] += e.self_device_time_total / 3e3
        total = sum(by.values())
        split = {k: round(v, 3) for k, v in sorted(by.items(), key=lambda kv: -kv[1])[:8]}
        if args.out:
            Path(args.out).mkdir(parents=True, exist_ok=True)
            (Path(args.out) / f"token_head_profile_B{B}.txt").write_text(
                prof.key_averages().table(sort_by="self_cuda_time_total", row_limit=40))
        res = {"B": B, "cuda_ms": round(t_cuda, 3), "cuda_min_ms": round(t_cuda_min, 3),
               "cuda_graph_ms": round(t_graph, 3), "torch_fp32_ms": round(t_torch, 3),
               "speedup_graph_vs_torch": round(t_torch / t_graph, 2), "gflop": round(flops / 1e9, 1),
               "mbytes": round(nbytes / 1e6, 1), "floor_ms": round(floor_ms, 3),
               "floor_fraction_graph": round(floor_ms / t_graph, 3), "kernel_ms_profiled": round(total, 3),
               "kernel_split_ms": split, "worst_grad_rel_vs_torch": float(f"{worst:.2e}")}
        print(json.dumps(res))


if __name__ == "__main__":
    main()

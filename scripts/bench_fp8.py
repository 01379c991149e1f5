"""Default mode vs FP8 mode (TokenHMREngine(fp8=True)) on the release config (synthetic weights), bs = 64, one process.

Prints, per mode: images/s of CUDA-graph replays on one stream and through TokenHMRPipeline(depth=4, streams=4),
alternating the two modes for --rounds rounds; the in-graph per-family GEMM times; the FP8 GEMMs' TFLOP/s next to the
H100 SXM data-sheet figure (1,979 dense FP8 TFLOP/s, a data-sheet number, not one reached here); the errors of both
modes against the fp32 reference golden (tests/golden/forward_release_d32_bs64.npz); and the card, read-only through
nvidia-smi.

    python scripts/bench_fp8.py [--rounds 3] [--iters 10]
"""
from __future__ import annotations

import argparse
import subprocess
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

FP8_DATASHEET_TFLOPS = 1979.0
GEMM_FAMILIES = ("vit.qkv_gemm", "vit.proj_gemm", "vit.fc1_gelu_gemm", "vit.fc2_gemm")


def card() -> str:
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return f"nvidia-smi unavailable ({e})"


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--batch", type=int, default=64)
    args = ap.parse_args()

    import numpy as np
    import torch

    from tokenhmr_b200 import synth
    from tokenhmr_b200.config import release_config
    from tokenhmr_b200.engine import TokenHMREngine, TokenHMRPipeline

    print("card:", card(), flush=True)
    cfg = release_config()
    sd, smpl = synth.make_state_dict(cfg, 1234), synth.make_smpl(cfg, 3)
    golden = np.load(ROOT / "tests" / "golden" / "forward_release_d32_bs64.npz")
    B = args.batch
    img = synth.make_images(B, cfg, int(golden["meta"][2])).cuda()
    models = {mode: TokenHMREngine(cfg, sd, smpl, device="cuda:0", concurrent=True, alias_outputs=True,
                                   max_cached_shapes=8, fp8=(mode == "fp8"))
              for mode in ("default", "fp8")}

    # accuracy against the fp32 reference (same images as the golden)
    stride = int(golden["meta"][6])

    def rel(a, b):
        a, b = a.detach().float().cpu(), torch.as_tensor(b).float()
        return float((a - b).abs().max() / (b.abs().max() + 1e-12))

    for mode, m in models.items():
        out = m({"img": img})
        errs = {k: rel(out[k], golden[k]) for k in ("pred_cam", "pred_cam_t", "pred_keypoints_3d", "pred_keypoints_2d")}
        errs["pred_vertices"] = rel(out["pred_vertices"][:, ::stride], golden["pred_vertices_sub"])
        errs["betas"] = rel(out["pred_smpl_params"]["betas"], golden["betas"])
        agree = float((out["cls_logits_softmax"].argmax(-1).cpu().numpy() == golden["cls_argmax"]).mean())
        print(f"[{mode}] rel err vs fp32 reference:", {k: f"{v:.2e}" for k, v in errs.items()},
              f"pose-token agreement {agree:.4f}", flush=True)

    # one stream: CUDA-graph replays, modes alternating
    def one_stream(m) -> float:
        m({"img": img})
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(args.iters):
            m({"img": img})
        torch.cuda.synchronize()
        return B * args.iters / (time.perf_counter() - t0)

    pinned = [synth.make_images(B, cfg, 100 + i).pin_memory() for i in range(8)]

    def four_streams(m) -> float:
        pipe = TokenHMRPipeline(m, depth=4, read_back=("pred_vertices",), streams=4)
        for b in pinned[:4]:
            pipe.result(pipe.submit({"img": b}))
        torch.cuda.synchronize()
        n = 2 * args.iters
        t0 = time.perf_counter()
        tickets = [pipe.submit({"img": pinned[i % len(pinned)]}) for i in range(min(4, n))]
        done = 0
        while done < n:
            pipe.result(tickets[done])
            done += 1
            if len(tickets) < n:
                tickets.append(pipe.submit({"img": pinned[len(tickets) % len(pinned)]}))
        torch.cuda.synchronize()
        return B * n / (time.perf_counter() - t0)

    rates = {mode: {"1 stream": [], "4 streams": []} for mode in models}
    for r in range(args.rounds):
        for mode, m in models.items():
            rates[mode]["1 stream"].append(one_stream(m))
            rates[mode]["4 streams"].append(four_streams(m))
        print(f"round {r}:", {mode: {k: f"{v[-1]:.1f}" for k, v in d.items()} for mode, d in rates.items()}, flush=True)
    for mode, d in rates.items():
        for k, v in d.items():
            print(f"[{mode}] {k}: best {max(v):.1f} img/s, median {sorted(v)[len(v) // 2]:.1f}, "
                  f"spread {(max(v) - min(v)) / max(v) * 100:.1f} %")
    for k in ("1 stream", "4 streams"):
        print(f"fp8 / default ({k}, best of {args.rounds}): {max(rates['fp8'][k]) / max(rates['default'][k]):.3f}")

    # in-graph per-family GEMM times
    for mode, m in models.items():
        rows = m.profile_in_graph(img, replays=10)
        fam = {}
        for name, ms, flops, _ in rows:
            t = fam.setdefault(name, [0.0, 0.0])
            t[0] += ms
            t[1] += flops
        total = sum(ms for _, ms, _, _ in rows)
        print(f"[{mode}] in-graph step {total:.2f} ms;", ", ".join(
            f"{n} {fam[n][0]:.2f} ms ({fam[n][1] / fam[n][0] / 1e9:.0f} TFLOP/s)" for n in GEMM_FAMILIES if n in fam))
        if mode == "fp8":
            ms = sum(fam[n][0] for n in ("vit.qkv_gemm", "vit.fc1_gelu_gemm", "vit.fc2_gemm"))
            fl = sum(fam[n][1] for n in ("vit.qkv_gemm", "vit.fc1_gelu_gemm", "vit.fc2_gemm"))
            print(f"[fp8] QKV + fc1 + fc2 on e4m3: {fl / ms / 1e9:.0f} TFLOP/s "
                  f"(H100 SXM data sheet: {FP8_DATASHEET_TFLOPS:.0f} dense FP8 TFLOP/s)")
    print("card:", card())


if __name__ == "__main__":
    main()

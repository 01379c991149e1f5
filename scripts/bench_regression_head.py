"""Token head vs regression head (TokenHMRConfig(head="transformer_decoder"), HMR 2.0's head) on the release config
(ViT-H/16 depth 32, synthetic weights), bs = 64, one process, one card.

Both engines share the backbone and decoder shapes; they differ only after the decoder's output token.  The script
replays each engine's CUDA graph, alternating the two for --rounds rounds of --iters forwards, times every round with
CUDA events after a warm-up, and prints the per-forward milliseconds, images/s, launches per forward and workspace
bytes of both, with the card's name and power limit (read-only through nvidia-smi).  Nothing is written.

    python scripts/bench_regression_head.py [--rounds 3] [--iters 20] [--batch 64]
"""
from __future__ import annotations

import argparse
import json
import statistics
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))


def card() -> str:
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return f"nvidia-smi unavailable ({e})"


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--batch", type=int, default=64)
    args = ap.parse_args()

    import torch

    from tokenhmr_b200 import synth
    from tokenhmr_b200._lib import lib
    from tokenhmr_b200.config import TokenHMRConfig
    from tokenhmr_b200.engine import TokenHMREngine

    if not torch.cuda.is_available():
        raise SystemExit("bench_regression_head.py needs a CUDA device (there is no CPU measurement)")
    B = args.batch
    models = {}
    for head in ("token", "transformer_decoder"):
        cfg = TokenHMRConfig(head=head)
        models[head] = TokenHMREngine(cfg, synth.make_state_dict(cfg, 1234), synth.make_smpl(cfg, 3), device="cuda:0",
                                      alias_outputs=True)
    img = synth.make_images(B, TokenHMRConfig(), 5).cuda()
    for m in models.values():
        for _ in range(args.warmup):
            m({"img": img})
    torch.cuda.synchronize()
    ms = {h: [] for h in models}
    for _ in range(args.rounds):
        for head, m in models.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.iters):
                m({"img": img})
            e1.record()
            e1.synchronize()
            ms[head].append(e0.elapsed_time(e1) / args.iters)
    res = {"card": card(), "batch": B, "rounds": args.rounds, "iters": args.iters}
    for head, m in models.items():
        med = statistics.median(ms[head])
        res[head] = {"ms_per_forward": [round(v, 3) for v in ms[head]], "images_per_s": round(B / med * 1e3, 1),
                     "launches": m.num_launches(), "workspace_bytes": lib().thmr_engine_workspace_bytes(m._h, B)}
    res["regression_over_token_speed"] = round(statistics.median(ms["token"]) / statistics.median(ms["transformer_decoder"]), 3)
    print(json.dumps(res))


if __name__ == "__main__":
    main()

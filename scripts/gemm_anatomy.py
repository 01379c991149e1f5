"""Where a ViT GEMM's time goes, tile by tile.

Runs the five M = 12288 GEMMs of the bs = 64 forward (QKV, proj, fc1 + GELU, fc2, decoder to_kv) with their real
epilogues through the test-only GEMM plan probe, at block_n 128 and 256, with the plan's epilogue kind and with the
general one, and prints one JSON line per case:
  (a) CUDA-event time per launch over 40 launches after warm-up, at the full K and at K = 64 (one k-block per tile,
      so almost only the fixed per-tile cost is left);
  (b) median, p90 and mean of each phase per tile from the kernel's %globaltimer timeline (GemmParams::timeline):
      wait = tile start -> first full barrier, mma = -> last wgmma retired, epilogue = -> epilogue done (for the
      TMA-stored kinds: the tile's stores issued, or handed to the residual kind's reduction thread, not completed);
  (c) torch.matmul fp16 at the same M, N, K, with no epilogue, as the card's own yardstick for these shapes;
  (d) card name, power limit and SM clocks, read in the same run.

    python scripts/gemm_anatomy.py [--out DIR/anatomy.jsonl] [--gemms qkv,fc2]

Needs tests/libthmr_gemm_probe.so, which tokenhmr_b200._build.build() compiles next to the tests.
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))

import torch  # noqa: E402

import gemm_probe  # noqa: E402

M = 12288
# name: (N, K, epilogue)
GEMMS = {
    "qkv": (3840, 1280, "bias_f16"),
    "proj": (1280, 1280, "bias_resid_f32"),
    "fc1_gelu": (5120, 1280, "bias_gelu_f16"),
    "fc2": (1280, 5120, "bias_resid_f32"),
    "to_kv": (6144, 1280, "f16"),
}
SLOTS = 64


def card() -> dict:
    q = "name,power.limit,clocks.sm,clocks.max.sm,clocks_throttle_reasons.sw_power_cap"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        return dict(zip(q.split(","), [v.strip() for v in out.split(",")]))
    except (OSError, IndexError, subprocess.SubprocessError) as e:
        return {"error": str(e)}


def operands(N: int, K: int, epi: str, g):
    A = (torch.randn(M, K, device="cuda", generator=g) * 0.5).half()
    W = (torch.randn(N, K, device="cuda", generator=g) * K ** -0.5).half()
    kw = {}
    if epi != "f16":
        kw["bias"] = torch.randn(N, device="cuda", generator=g)
    if epi == "bias_resid_f32":
        x = torch.randn(M, N, device="cuda", generator=g)
        kw.update(resid=x, ldr=N, out32=x, ld32=N)
    else:
        kw.update(out16=torch.empty(M, N, dtype=torch.float16, device="cuda"), ld16=N)
        if epi == "bias_gelu_f16":
            kw["act"] = "gelu"
    return A, W, kw


def event_ms(fn, n: int = 40) -> float:
    for _ in range(5):
        fn()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    s.record()
    for _ in range(n):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / n


def phases(tl) -> dict:
    t = tl.view(-1, 4).double()
    t = t[t[:, 0] > 0]
    d = {"wait": t[:, 1] - t[:, 0], "mma": t[:, 2] - t[:, 1], "epilogue": t[:, 3] - t[:, 2], "tile": t[:, 3] - t[:, 0]}
    return {k: {"median_us": round(float(v.median()) / 1e3, 3), "p90_us": round(float(v.quantile(0.9)) / 1e3, 3),
                "mean_us": round(float(v.mean()) / 1e3, 3)} for k, v in d.items()}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", type=Path, default=None)
    ap.add_argument("--gemms", default=",".join(GEMMS))
    args = ap.parse_args()
    assert torch.cuda.is_available(), "gemm_anatomy.py needs a GPU"
    g = torch.Generator(device="cuda").manual_seed(0)
    lines = [{"card": card()}]
    print(json.dumps(lines[0]), flush=True)
    for name in args.gemms.split(","):
        N, K, epi = GEMMS[name]
        for k in (K, 64):
            A, W, kw = operands(N, k, epi, g)
            mm = event_ms(lambda: torch.matmul(A, W.t()))
            for bn in (128, 256):
                for kind in (None, "general"):
                    run = dict(force_bn=bn, epi=kind, **kw)
                    _, chosen, _ = gemm_probe.plan(A, W, M, N, k, **run)
                    ms = event_ms(lambda: gemm_probe.gemm(A, W, M, N, k, **run))
                    tl, _ = gemm_probe.timeline(A, W, M, N, k, SLOTS, **run)
                    torch.cuda.synchronize()
                    rec = {"gemm": name, "N": N, "K": k, "block_n": bn, "epi": chosen, "ms": round(ms, 4),
                           "tflops": round(2.0 * M * N * k / ms / 1e9, 1), "torch_matmul_ms": round(mm, 4),
                           "phases": phases(tl)}
                    lines.append(rec)
                    print(json.dumps(rec), flush=True)
    lines.append({"card_after": card()})
    print(json.dumps(lines[-1]), flush=True)
    if args.out:
        args.out.parent.mkdir(parents=True, exist_ok=True)
        args.out.write_text("".join(json.dumps(r) + "\n" for r in lines))


if __name__ == "__main__":
    main()

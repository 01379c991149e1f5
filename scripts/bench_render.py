"""Times the CUDA rasterizer (tokenhmr_b200.render): render_crops of 64 crops at 256 x 256, 1920 x 1080 frames with
1, 8 and 32 people, and MeshRenderer.visualize_tensorboard (eval.py --render's prediction grid: two mesh views and two
OpenPose skeletons per crop) at B = 8 (what eval.py renders) and 64, on a closed synthetic mesh of SMPL's size (6890
vertices, 13776 faces).  CUDA events around
windows of back-to-back calls of at least --window-ms each, --repeats times after --warmup calls; prints one JSON line
with the median, the spread (max - min over median) and the card's name and power limit read in the same run.

There is no CPU or pyrender baseline: pyrender needs an OpenGL stack this project does not depend on, and the
reference's render_openpose no longer runs on NumPy >= 1.24 (np.int)."""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path[:0] = [str(ROOT), str(ROOT / "tests")]

from render_mesh import posed, synthetic_body  # noqa: E402
from tokenhmr_b200 import render as R  # noqa: E402


def _time(fn, warmup, window_ms, repeats):
    """ms per call: each repeat times as many back-to-back calls as fill `window_ms` (sized from a probe), so the
    window is long against clock and scheduler noise; returns the median and the spread over the repeats."""
    for _ in range(warmup):
        fn()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def window(n):
        torch.cuda.synchronize()
        start.record()
        for _ in range(n):
            fn()
        end.record()
        torch.cuda.synchronize()
        return start.elapsed_time(end) / n

    iters = max(40, int(window_ms / max(window(20), 1e-3)))
    runs = sorted(window(iters) for _ in range(repeats))
    med = runs[len(runs) // 2]
    return {"ms": med, "spread": (runs[-1] - runs[0]) / med, "calls_per_window": iters, "repeats": repeats}


def _card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        return q
    except Exception as e:   # the timings stand without it
        return f"unavailable ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--window-ms", type=float, default=300.0)
    ap.add_argument("--repeats", type=int, default=5)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_render needs a GPU"
    v0, faces = synthetic_body()
    ren = R.Renderer({"EXTRA": {"FOCAL_LENGTH": 5000.0}}, faces, "cuda:0")
    res = {"card": _card(), "mesh": {"verts": int(v0.shape[0]), "faces": int(faces.shape[0])}}
    rng = np.random.default_rng(0)
    B = 64
    v = torch.from_numpy(posed(v0, B)).cuda()
    t = torch.tensor(np.stack([rng.uniform(-.1, .1, B), rng.uniform(-.1, .1, B),
                               2 * 5000. / (256 * rng.uniform(.6, 1., B))], 1), dtype=torch.float32, device="cuda")
    imgs = torch.randn(B, 3, 256, 256, device="cuda")
    r = _time(lambda: ren.render_crops(v, t, imgs), a.warmup, a.window_ms, a.repeats)
    res["crops_64x256"] = dict(r, tris_per_s=B * faces.shape[0] / r["ms"] * 1e3, pix_per_s=B * 256 * 256 / r["ms"] * 1e3)
    f = 5000. / 256 * 1920
    for n in (1, 8, 32):
        vv = torch.from_numpy(posed(v0, n, seed=n)).cuda()
        z = rng.uniform(80, 250, n)
        sx, sy = rng.uniform(100, 1820, n), rng.uniform(200, 880, n)
        tt = torch.tensor(np.stack([(sx - 960) * z / f, (sy - 540) * z / f, z], 1), dtype=torch.float32, device="cuda")
        lights = R.multiple_lights()
        fn = lambda: ren.raster(vv, tt, 1920, 1080, f, rotate_translation=True, mesh_image=[0] * n, n_images=1,
                                lights=lights, outputs=("rgba",))
        r = _time(fn, a.warmup, a.window_ms, a.repeats)
        res[f"frame_1080p_{n}"] = dict(r, tris_per_s=n * faces.shape[0] / r["ms"] * 1e3,
                                       pix_per_s=1920 * 1080 / r["ms"] * 1e3)
    mr = R.MeshRenderer({"EXTRA": {"FOCAL_LENGTH": 5000.0}, "MODEL": {"IMAGE_SIZE": 256}}, faces, "cuda:0")
    for B in (8, 64):
        v = torch.from_numpy(posed(v0, B, seed=B)).cuda()
        t = torch.tensor(np.stack([rng.uniform(-.1, .1, B), rng.uniform(-.1, .1, B),
                                   2 * 5000. / (256 * rng.uniform(.6, 1., B))], 1), dtype=torch.float32, device="cuda")
        imgs = torch.rand(B, 3, 256, 256, device="cuda")
        pred = torch.rand(B, 44, 2, device="cuda") - 0.5
        gt = torch.cat([torch.rand(B, 44, 2, device="cuda") - 0.5, (torch.rand(B, 44, 1, device="cuda") > 0.3).float()],
                       -1)
        r = _time(lambda: mr.visualize_tensorboard(v, t, imgs, pred, gt), a.warmup, a.window_ms, a.repeats)
        res[f"visualize_tensorboard_{B}x256"] = dict(r, what="CUDA-tensor inputs, grid left on the GPU")
        args = [x.cpu().numpy() for x in (v, t, imgs, pred, gt)]
        r = _time(lambda: mr.visualize_tensorboard(*args).cpu().numpy(), a.warmup, a.window_ms, a.repeats)
        res[f"visualize_tensorboard_{B}x256_numpy"] = dict(r, what="numpy inputs and .cpu().numpy(), as eval.py calls it")
    print(json.dumps(res))


if __name__ == "__main__":
    main()

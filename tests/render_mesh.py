"""A closed synthetic mesh of SMPL's size for the renderer tests: 6890 vertices, 13776 faces (genus 0: F = 2V - 4).

A UV sphere of 84 rings x 82 segments plus the two poles, stretched to a person's proportions (0.4 x 1.7 x 0.25 m)
and dented with bumps so that it occludes itself.  Faces are wound outwards."""
from __future__ import annotations

import numpy as np

RINGS, SEGS = 84, 82


def synthetic_body(seed: int = 0):
    rng = np.random.default_rng(seed)
    th = np.pi * (np.arange(RINGS) + 1) / (RINGS + 1)          # polar angle of each ring
    ph = 2 * np.pi * np.arange(SEGS) / SEGS
    T, P = np.meshgrid(th, ph, indexing="ij")
    bump = 1 + 0.18 * np.sin(3 * P + rng.uniform(0, 6)) * np.sin(4 * T) + 0.08 * np.cos(7 * T)
    x = 0.20 * bump * np.sin(T) * np.cos(P)
    y = -0.85 * np.cos(T)                                       # model frame: y down in the image, head at -y
    z = 0.125 * bump * np.sin(T) * np.sin(P)
    ring = np.stack([x, y, z], -1).reshape(-1, 3)
    verts = np.concatenate([[[0, -0.85, 0]], ring, [[0, 0.85, 0]]]).astype(np.float32)
    top, bot = 0, RINGS * SEGS + 1
    idx = lambda r, s: 1 + r * SEGS + (s % SEGS)
    faces = []
    for s in range(SEGS):
        faces.append((top, idx(0, s + 1), idx(0, s)))
        faces.append((bot, idx(RINGS - 1, s), idx(RINGS - 1, s + 1)))
        for r in range(RINGS - 1):
            a, b, c, d = idx(r, s), idx(r, s + 1), idx(r + 1, s), idx(r + 1, s + 1)
            faces += [(a, b, d), (a, d, c)]
    faces = np.array(faces, np.int32)[:, [0, 2, 1]]
    assert verts.shape == (6890, 3) and faces.shape == (13776, 3)
    return verts, faces


def posed(verts: np.ndarray, n: int, seed: int = 1) -> np.ndarray:
    """n copies with a random rotation about y and a small random scale (fp32)."""
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(n):
        a = rng.uniform(-np.pi, np.pi)
        R = np.array([[np.cos(a), 0, np.sin(a)], [0, 1, 0], [-np.sin(a), 0, np.cos(a)]])
        out.append((verts.astype(np.float64) @ R.T) * rng.uniform(0.9, 1.1))
    return np.array(out, np.float32)


def ellipsoid(axes, rings: int = 10, segs: int = 16):
    """A coarse closed ellipsoid with semi-axes `axes` (large faces), wound outwards, fp32."""
    th = np.pi * (np.arange(rings) + 1) / (rings + 1)
    ph = 2 * np.pi * np.arange(segs) / segs
    T, P = np.meshgrid(th, ph, indexing="ij")
    ring = np.stack([np.sin(T) * np.cos(P), -np.cos(T), np.sin(T) * np.sin(P)], -1).reshape(-1, 3)
    verts = np.concatenate([[[0, -1, 0]], ring, [[0, 1, 0]]]) * np.asarray(axes, float)
    top, bot = 0, rings * segs + 1
    idx = lambda r, s: 1 + r * segs + (s % segs)
    faces = []
    for s in range(segs):
        faces.append((top, idx(0, s), idx(0, s + 1)))
        faces.append((bot, idx(rings - 1, s + 1), idx(rings - 1, s)))
        for r in range(rings - 1):
            a, b, c, d = idx(r, s), idx(r, s + 1), idx(r + 1, s), idx(r + 1, s + 1)
            faces += [(a, d, b), (a, c, d)]
    return verts.astype(np.float32), np.array(faces, np.int32)

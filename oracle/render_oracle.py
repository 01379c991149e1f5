"""float64 numpy restatement of the renderer contract (DESIGN.md §2 "Rendering").  TEST INFRASTRUCTURE.

* `crop_chain` / `multiple_chain` restate the reference's camera chain step by step (renderer.py:189-210 and
  :233-251, :338-347): x flip of the translation, the trimesh rotations, pyrender's IntrinsicsCamera projection matrix
  and the window transform, rows pointing down.  The tests show both reduce to perspective_projection of q = R v + t
  (or R (v + t)) with the principal point at (W/2, H/2), which is what `camera_q` / `project` compute.
* `raster` is an edge-function rasterizer with the kernel's sample points (pixel centres), fill rule (top-left, each
  edge evaluated in one canonical direction), z-test (nearest perspective-correct z, lower face id on ties) and znear
  drop.  Given per-vertex bounds on the kernel's fp32 screen / depth error it also marks the pixels whose coverage or
  depth order those errors could change.
* `shade` is the stated shading model: smooth area-weighted vertex normals, perspective-correct interpolation,
  base * clamp(ambient + sum_dir I max(0, n.l) + sum_point I max(0, n.l) / d^2, 0, 1), then k/255.
* `lights_from_reference` imports the reference's renderer.py through oracle/ref_import.py with a recording stand-in
  for pyrender and records the light nodes create_raymond_lights, add_lighting and add_point_lighting build.
"""
from __future__ import annotations

import types
from typing import Dict, Optional

import numpy as np

U32 = 2.0 ** -24          # unit round-off of fp32


# ---------------------------------------------------------------------------------------------- rotations
def rot_axis(angle_rad: float, axis) -> np.ndarray:
    """trimesh.transformations.rotation_matrix(angle, axis)[:3, :3]: Rodrigues' formula about a unit axis."""
    a = np.asarray(axis, float)
    a = a / np.linalg.norm(a)
    c, s = np.cos(angle_rad), np.sin(angle_rad)
    K = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
    return c * np.eye(3) + s * K + (1 - c) * np.outer(a, a)


# ---------------------------------------------------------------------------------------------- camera chain
def _pyrender_project(p_world: np.ndarray, cam_t: np.ndarray, focal: float, W: int, H: int):
    """Camera at cam_t with identity rotation, IntrinsicsCamera(fx = fy = focal, cx = W/2, cy = H/2): eye space,
    projection matrix, perspective divide, viewport, then rows from the top.  Returns (col, row, depth)."""
    cx, cy = W / 2.0, H / 2.0
    P = np.zeros((4, 4))
    P[0, 0], P[1, 1] = 2 * focal / W, 2 * focal / H
    P[0, 2], P[1, 2] = 1 - 2 * cx / W, 2 * cy / H - 1
    P[3, 2] = -1.0
    eye = p_world - cam_t
    clip = np.concatenate([eye, np.ones(eye.shape[:-1] + (1,))], -1) @ P.T
    ndc = clip[..., :2] / clip[..., 3:4]
    xw = (ndc[..., 0] + 1) * W / 2
    yw = (ndc[..., 1] + 1) * H / 2
    return xw, H - yw, -eye[..., 2]


def crop_chain(v, t, focal, W, H, side_view=False, rot_angle=90.0):
    """Renderer.__call__ (renderer.py:189-210): (col, row, depth) of every vertex."""
    t = np.array(t, float).copy()
    t[0] *= -1.0
    m = np.asarray(v, float)
    if side_view:
        m = m @ rot_axis(np.radians(rot_angle), [0, 1, 0]).T
    m = m @ rot_axis(np.radians(180), [1, 0, 0]).T
    return _pyrender_project(m, t, focal, W, H)


def multiple_chain(v, t, focal, W, H, axis=(1, 0, 0), angle=0.0):
    """render_rgba_multiple: vertices_to_trimesh (renderer.py:241-250) and an identity camera (:338-347)."""
    m = np.asarray(v, float) + np.asarray(t, float)
    m = m @ rot_axis(np.radians(angle), axis).T
    m = m @ rot_axis(np.radians(180), [1, 0, 0]).T
    return _pyrender_project(m, np.zeros(3), focal, W, H)


def camera_q(v, t, R=None, rotate_translation=False):
    """The model's camera frame (x right, y down, z forward): q = R v + t or R (v + t)."""
    v, t = np.asarray(v, float), np.asarray(t, float)
    R = np.eye(3) if R is None else np.asarray(R, float)
    return (v + t[..., None, :]) @ R.T if rotate_translation else v @ R.T + t[..., None, :]


def project(q, focal, W, H):
    """perspective_projection (geometry.py:86-124) with camera_center (W/2, H/2)."""
    return np.stack([focal * q[..., 0] / q[..., 2] + W / 2.0, focal * q[..., 1] / q[..., 2] + H / 2.0], -1)


def vertex_error_bounds(v, t, R, rotate_translation, focal, W, H):
    """Bounds on the kernel's fp32 vertex stage (render_vertex_kernel) against exact arithmetic on the same fp32
    inputs, per vertex: (screen coordinate error, camera z error, camera q component error).
    q component: a 3-term dot product plus the translation in fp32 (possibly fused) has error <= 4u sum |terms|;
    with rotate_translation the sum v + t adds u |v + t| per term, <= 5u sum |R| (|v| + |t|).  Screen: x / z carries
    the relative errors of x and z plus u, f * (.) + c one more rounding.  Each bound is doubled for head-room."""
    v, t = np.asarray(v, float), np.asarray(t, float)
    R = np.asarray(R, float)
    if rotate_translation:
        mag = (np.abs(v) + np.abs(t)[..., None, :]) @ np.abs(R).T
        eq = 5 * U32 * mag
    else:
        mag = np.abs(v) @ np.abs(R).T + np.abs(t)[..., None, :]
        eq = 4 * U32 * mag
    q = camera_q(v, t, R, rotate_translation)
    z = q[..., 2]
    ez = eq[..., 2]
    s = project(q, focal, W, H)
    es = np.stack([focal * (eq[..., k] + np.abs(q[..., k]) * ez / np.abs(z) + U32 * np.abs(q[..., k])) / np.abs(z)
                   + U32 * np.abs(s[..., k]) for k in (0, 1)], -1)
    return 2 * es.max(-1), 2 * ez, 2 * eq.max(-1)


# ---------------------------------------------------------------------------------------------- rasterizer
def _edges(faces):
    """Per face, for the edge opposite vertex k: the two vertex slots in canonical (lower vertex id first) order and
    the sign of the directed edge relative to it (the kernel's make_edge)."""
    pairs = [(1, 2), (2, 0), (0, 1)]
    out = []
    for a, b in pairs:
        ia, ib = faces[:, a], faces[:, b]
        swap = ib < ia
        lo = np.where(swap, ib, ia)
        hi = np.where(swap, ia, ib)
        out.append((lo, hi, np.where(swap, -1.0, 1.0)))
    return out


def raster(scr, qz, faces, W, H, mesh_image=None, n_images=None, znear=0.05, es=None, ez=None):
    """scr (n, V, 2) screen positions, qz (n, V) camera z.  Returns face_id (n_images, H, W) int64 (mesh * F + face,
    -1 = empty), depth, barycentrics {(img, pix): ...} as arrays, and -- given per-vertex bounds es / ez -- the mask of
    pixels whose coverage or winning depth those bounds could change."""
    scr, qz = np.asarray(scr, float), np.asarray(qz, float)
    faces = np.asarray(faces, np.int64)
    n, V = qz.shape
    F = faces.shape[0]
    n_images = n if n_images is None else n_images
    mesh_image = np.arange(n) if mesh_image is None else np.asarray(mesh_image)
    best_key = np.full(n_images * H * W, np.inf)
    best_fid = np.full(n_images * H * W, -1, np.int64)
    cand = []   # (pix, z, fid, dz) of every covered pair
    ambiguous = np.zeros(n_images * H * W, bool)
    edges = _edges(faces)
    for m in range(n):
        s, z = scr[m], qz[m]
        zf = z[faces]
        keep = np.all(zf >= znear, 1) & np.all(np.isfinite(s[faces]).reshape(F, -1), 1)
        sf = s[faces]                                       # (F, 3, 2)
        E_at = []
        for k, (lo, hi, sg) in enumerate(edges):
            E_at.append((s[lo], s[hi] - s[lo], sg))
        ax, d, sg = E_at[2]
        area = sg * (d[:, 0] * (sf[:, 2, 1] - ax[:, 1]) - d[:, 1] * (sf[:, 2, 0] - ax[:, 0]))
        keep &= area != 0
        mn, mx = sf.min(1), sf.max(1)
        with np.errstate(invalid="ignore"):
            x0 = np.maximum(np.floor(mn[:, 0] - 0.5), 0)
            y0 = np.maximum(np.floor(mn[:, 1] - 0.5), 0)
            x1 = np.minimum(np.ceil(mx[:, 0] - 0.5), W - 1)
            y1 = np.minimum(np.ceil(mx[:, 1] - 0.5), H - 1)
        keep &= (x0 <= x1) & (y0 <= y1)
        ids = np.nonzero(keep)[0]
        if ids.size == 0:
            continue
        bw = (x1[ids] - x0[ids] + 1).astype(np.int64)
        bh = (y1[ids] - y0[ids] + 1).astype(np.int64)
        cnt = bw * bh
        f = np.repeat(ids, cnt)
        start = np.repeat(np.cumsum(cnt) - cnt, cnt)
        loc = np.arange(cnt.sum()) - start
        bwr = np.repeat(bw, cnt)
        px = x0[f].astype(np.int64) + loc % bwr
        py = y0[f].astype(np.int64) + loc // bwr
        cxp, cyp = px + 0.5, py + 0.5
        orient = np.sign(area[f])
        inside = np.ones(f.size, bool)
        w = np.empty((3, f.size))
        near = np.zeros(f.size, bool)          # some edge value within its error bound of zero
        maybe = np.ones(f.size, bool)          # no edge value clearly outside
        for k, (axk, dk, sgk) in enumerate(E_at):
            a, dd, sgn = axk[f], dk[f], sgk[f]
            e = orient * sgn * (dd[:, 0] * (cyp - a[:, 1]) - dd[:, 1] * (cxp - a[:, 0]))
            ddx, ddy = orient * sgn * dd[:, 0], orient * sgn * dd[:, 1]
            tl = (ddy < 0) | ((ddy == 0) & (ddx > 0))
            inside &= (e > 0) | ((e == 0) & tl)
            w[k] = e / np.abs(area[f])
            if es is not None:
                lo_v, hi_v = edges[k][0][f], edges[k][1][f]
                da, db = es[m][lo_v], es[m][hi_v]
                dE = (da + db) * (np.abs(cyp - a[:, 1]) + np.abs(cxp - a[:, 0])) + da * (np.abs(dd[:, 0]) + np.abs(dd[:, 1]))
                dE += 2 * (da + db) * da + 1e-12 * (np.abs(dd).sum(1) * (np.abs(cyp - a[:, 1]) + np.abs(cxp - a[:, 0])))
                near |= np.abs(e) <= dE
                maybe &= e > -dE
        pix = mesh_image[m] * H * W + py * W + px
        if es is not None:   # the kernel's rounding may or may not put this pixel inside this face
            ambiguous[pix[near & maybe]] = True
        iz = (w / zf[f].T).sum(0)
        zc = 1.0 / iz
        dz = np.zeros(f.size)
        dw = np.zeros((3, f.size))
        if ez is not None:
            A = np.abs(area[f])
            dA = sum(_edge_bound(es[m], E_at, edges, k, f, sf[f, k]) for k in range(3)) / 3
            dw = np.stack([(_edge_bound(es[m], E_at, edges, k, f, np.stack([cxp, cyp], 1)) + np.abs(w[k]) * dA) / A
                           for k in range(3)])
            # the barycentrics sum to one before and after the perturbation, so they move 1/z only by the spread of
            # the vertices' 1/z; the vertices' own z errors and the fp32 reciprocals add their relative errors
            izv = 1.0 / zf[f].T
            diz = dw.sum(0) * (izv.max(0) - izv.min(0)) + (w * izv * (ez[m][faces[f]].T / zf[f].T + U32)).sum(0)
            dz = 2 * zc * (diz / iz + U32)
        sel = inside
        cand.append((pix[sel], zc[sel], m * F + f[sel], dz[sel], w[:, sel], dw[:, sel]))
    if not cand:
        return {"face_id": best_fid.reshape(n_images, H, W), "depth": np.zeros((n_images, H, W)),
                "ambiguous": ambiguous.reshape(n_images, H, W), "pix": np.zeros(0, np.int64)}
    pix = np.concatenate([c[0] for c in cand])
    zc = np.concatenate([c[1] for c in cand])
    fid = np.concatenate([c[2] for c in cand])
    dz = np.concatenate([c[3] for c in cand])
    w = np.concatenate([c[4] for c in cand], 1)
    dw = np.concatenate([c[5] for c in cand], 1)
    order = np.lexsort((fid, zc, pix))
    pix, zc, fid, dz, w, dw = pix[order], zc[order], fid[order], dz[order], w[:, order], dw[:, order]
    first = np.ones(pix.size, bool)
    first[1:] = pix[1:] != pix[:-1]
    second = np.zeros(pix.size, bool)
    second[1:] = first[:-1] & ~first[1:]
    win = np.nonzero(first)[0]
    best_fid[pix[win]] = fid[win]
    depth = np.zeros(n_images * H * W)
    depth[pix[win]] = zc[win]
    sec = np.nonzero(second)[0]
    close = zc[sec] - zc[sec - 1] <= dz[sec] + dz[sec - 1]
    ambiguous[pix[sec[close]]] = True
    return {"face_id": best_fid.reshape(n_images, H, W), "depth": depth.reshape(n_images, H, W),
            "depth_bound": _scatter(pix[win], dz[win], n_images * H * W).reshape(n_images, H, W),
            "ambiguous": ambiguous.reshape(n_images, H, W), "pix": pix[win], "w": w[:, win], "dw": dw[:, win],
            "fid": fid[win]}


def _edge_bound(es_m, E_at, edges, k, f, p):
    axk, dk, _ = E_at[k]
    a, dd = axk[f], dk[f]
    da, db = es_m[edges[k][0][f]], es_m[edges[k][1][f]]
    return (da + db) * (np.abs(p[:, 1] - a[:, 1]) + np.abs(p[:, 0] - a[:, 0])) + da * (np.abs(dd[:, 0]) + np.abs(dd[:, 1]))


def _scatter(idx, val, size):
    out = np.zeros(size)
    out[idx] = val
    return out


# ---------------------------------------------------------------------------------------------- shading
def vertex_normals(q, faces):
    """Area-weighted smooth normals: sum over a vertex's faces of (q1 - q0) x (q2 - q0), normalised."""
    q = np.asarray(q, float)
    faces = np.asarray(faces, np.int64)
    c = np.cross(q[faces[:, 1]] - q[faces[:, 0]], q[faces[:, 2]] - q[faces[:, 0]])
    n = np.zeros_like(q)
    for k in range(3):
        np.add.at(n, faces[:, k], c)
    ln = np.linalg.norm(n, axis=1, keepdims=True)
    return np.where(ln > 0, n / np.where(ln > 0, ln, 1), 0), c


def shade(r, q_all, faces, lights, base, ambient=0.3, perspective=True):
    """Pre-quantisation colour of every covered pixel of raster() result r (rows of r['pix']).  perspective=False
    interpolates with the screen-space barycentrics instead (what a renderer without perspective correction shows;
    the tests use it to show that their scenes tell the two apart)."""
    faces = np.asarray(faces, np.int64)
    F = faces.shape[0]
    m, f = r["fid"] // F, r["fid"] % F
    q_all = np.asarray(q_all, float)
    nrm = np.stack([vertex_normals(q, faces)[0] for q in q_all])    # (n, V, 3)
    w = r["w"]
    vi = faces[f]                                                  # (P, 3)
    qv = np.stack([q_all[m, vi[:, k]] for k in range(3)])          # (3, P, 3)
    b = w / qv[..., 2] if perspective else w.copy()
    b = b / b.sum(0)
    nv = np.stack([nrm[m, vi[:, k]] for k in range(3)])
    n = (b[..., None] * nv).sum(0)
    n = n / np.maximum(np.linalg.norm(n, axis=1, keepdims=True), 1e-300)
    p = (b[..., None] * qv).sum(0)
    light = np.full(n.shape[0], ambient)
    for kind, vec, inten in lights:
        vec = np.asarray(vec, float)
        if kind == 0:
            light += inten * np.maximum(0, n @ vec)
        else:
            dv = vec - p
            d2 = (dv * dv).sum(1)
            light += inten * np.maximum(0, (n * dv).sum(1) / np.sqrt(d2)) / d2
    light = np.clip(light, 0, 1)
    return np.asarray(base, float)[None, :] * light[:, None]


def quantise(c):
    return np.rint(np.asarray(c) * 255.0) / 255.0


# ---------------------------------------------------------------------------------------------- reference lights
def lights_from_reference() -> Dict[str, np.ndarray]:
    """Node matrices of the reference's light rig, recorded from the LIVE renderer.py (needs TOKENHMR_REFERENCE):
    'raymond' [3,4,4] (create_raymond_lights), 'directional' [6,4,4] (add_lighting), 'point' [6,4,4]
    (add_point_lighting), the camera at the identity pose as render_rgba_multiple places it."""
    from . import ref_import
    ns = ref_import.load_eval_modules()
    R = ns.renderer

    class _Light:
        def __init__(self, kind, **kw):
            self.kind, self.kw = kind, kw

    class _Node:
        def __init__(self, name=None, light=None, matrix=None, **kw):
            self.name, self.light, self.matrix = name, light, np.asarray(matrix, float)

    rec = types.SimpleNamespace(Node=_Node, DirectionalLight=lambda **kw: _Light("directional", **kw),
                                PointLight=lambda **kw: _Light("point", **kw))

    class _Scene:
        def __init__(self):
            self.nodes = []

        def get_pose(self, node):
            return np.eye(4)

        def has_node(self, node):
            return False

        def add_node(self, node):
            self.nodes.append(node)

    saved = R.pyrender
    R.pyrender = rec
    try:
        raymond = [nd.matrix for nd in R.create_raymond_lights()]
        scene = _Scene()
        R.Renderer.add_point_lighting(None, scene, None)
        R.Renderer.add_lighting(None, scene, None)
    finally:
        R.pyrender = saved
    point = [nd.matrix for nd in scene.nodes if nd.light.kind == "point"]
    directional = [nd.matrix for nd in scene.nodes if nd.light.kind == "directional"]
    assert all(nd.light.kw.get("intensity", 1.0) == 1.0 for nd in scene.nodes)
    return {"raymond": np.array(raymond), "directional": np.array(directional), "point": np.array(point)}


def write_golden(path) -> None:
    """tests/golden/render_reference.npz: the recorded light matrices and the live perspective_projection of a seeded
    point set (python -m oracle.render_oracle)."""
    import torch
    from . import ref_import
    ns = ref_import.load_modules()
    rng = np.random.default_rng(7)
    pts = rng.normal(size=(2, 50, 3)).astype(np.float32)
    trans = np.array([[0.1, -0.2, 20.0], [-0.3, 0.4, 45.0]], np.float32)
    focal = np.array([[5000.0, 5000.0], [1200.0, 1200.0]], np.float32)
    center = np.array([[128.0, 128.0], [960.0, 540.0]], np.float32)
    proj = ns.geometry.perspective_projection(torch.from_numpy(pts), torch.from_numpy(trans), torch.from_numpy(focal),
                                              camera_center=torch.from_numpy(center)).numpy()
    np.savez(path, pts=pts, trans=trans, focal=focal, center=center, proj=proj, **lights_from_reference())


if __name__ == "__main__":
    from pathlib import Path
    out = Path(__file__).resolve().parent.parent / "tests" / "golden" / "render_reference.npz"
    write_golden(out)
    print(out)

"""numpy restatement of the reference's MeshRenderer grid (tokenhmr/lib/utils/mesh_renderer.py:70-107) and of the
OpenPose overlay it draws (lib/utils/render_openpose.py).  TEST INFRASTRUCTURE.  Contract: DESIGN.md §2 "Rendering".

* `cv_line` / `cv_circle` restate the three OpenCV 4.x drawing primitives render_openpose reaches, as the scanline
  spans they paint: cv2.line with thickness 2 and LINE_8 (ThickLine: a convex quad in 16-bit fixed point, filled by
  FillConvexPoly over its Line2 outline, plus a filled radius-1 Circle at each end), cv2.circle with radius 1 and
  thickness 2 (EllipseEx: a 5-point polyline of thickness-2 segments) and cv2.circle with radius 1 and thickness 1
  (the midpoint Circle, unfilled).  Every one clips at the image border.
* `render_openpose` restates render_openpose.py with `int` for the removed `np.int`, in the reference's float32 types.
* `prepare_keypoints` / `visualize_tensorboard` restate the scaling, the keypoint_matches substitution and the
  make_grid layout; the mesh tiles are inputs.
* `load_live` imports the live mesh_renderer.py through oracle/ref_import.py with pyrender / trimesh stand-ins that
  record every scene and return a caller-given image, and with the `np.int = int` shim its render_openpose needs.
"""
from __future__ import annotations

import math
import types

import numpy as np

XY_SHIFT = 16
XY_ONE = 1 << XY_SHIFT

PAIRS = np.array([1, 8, 1, 2, 1, 5, 2, 3, 3, 4, 5, 6, 6, 7, 8, 9, 9, 10, 10, 11, 8, 12, 12, 13, 13, 14, 1, 0, 0, 15,
                  15, 17, 0, 16, 16, 18, 14, 19, 19, 20, 14, 21, 11, 22, 22, 23, 11, 24]).reshape(-1, 2)
COLORS = np.array([255, 0, 85, 255, 0, 0, 255, 85, 0, 255, 170, 0, 255, 255, 0, 170, 255, 0, 85, 255, 0, 0, 255, 0,
                   255, 0, 0, 0, 255, 85, 0, 255, 170, 0, 255, 255, 0, 170, 255, 0, 85, 255, 0, 0, 255, 255, 0, 170,
                   170, 0, 255, 255, 0, 255, 85, 0, 255, 0, 0, 255, 0, 0, 255, 0, 0, 255, 0, 255, 255, 0, 255, 255,
                   0, 255, 255], np.float64).reshape(-1, 3)
KEYPOINT_MATCHES = [(1, 12), (2, 8), (3, 7), (4, 6), (5, 9), (6, 10), (7, 11), (8, 14), (9, 2), (10, 1), (11, 0),
                    (12, 3), (13, 4), (14, 5)]
MAX_WIDTH = 11718   # largest image width whose thickness formula still gives line 2 / circle radius 1


def _cv_round(x: float) -> int:
    return int(np.rint(x))          # cvRound: round half to even


def _tdiv(a: int, b: int) -> int:
    """C integer division (truncates toward zero)."""
    q = abs(a) // abs(b)
    return q if (a >= 0) == (b >= 0) else -q


# ---------------------------------------------------------------------------------------------- OpenCV primitives
def _clip_line(W: int, H: int, p1, p2):
    """clipLine(Size2l, Point2l&, Point2l&) on the scaled image size; returns the clipped points or None."""
    right, bottom = W - 1, H - 1
    x1, y1 = p1
    x2, y2 = p2
    c1 = (x1 < 0) + (x1 > right) * 2 + (y1 < 0) * 4 + (y1 > bottom) * 8
    c2 = (x2 < 0) + (x2 > right) * 2 + (y2 < 0) * 4 + (y2 > bottom) * 8
    if (c1 & c2) == 0 and (c1 | c2) != 0:
        if c1 & 12:
            a = 0 if c1 < 8 else bottom
            x1 += int(float(a - y1) * (x2 - x1) / (y2 - y1))
            y1 = a
            c1 = (x1 < 0) + (x1 > right) * 2
        if c2 & 12:
            a = 0 if c2 < 8 else bottom
            x2 += int(float(a - y2) * (x2 - x1) / (y2 - y1))
            y2 = a
            c2 = (x2 < 0) + (x2 > right) * 2
        if (c1 & c2) == 0 and (c1 | c2) != 0:
            if c1:
                a = 0 if c1 == 1 else right
                y1 += int(float(a - x1) * (y2 - y1) / (x2 - x1))
                x1 = a
                c1 = 0
            if c2:
                a = 0 if c2 == 1 else right
                y2 += int(float(a - x2) * (y2 - y1) / (x2 - x1))
                x2 = a
                c2 = 0
    if (c1 | c2) != 0:
        return None
    return (x1, y1), (x2, y2)


def _line2(emit, W: int, H: int, p1, p2):
    """Line2: the 8-connected outline segment of a fixed-point edge (both ends included)."""
    c = _clip_line(W << XY_SHIFT, H << XY_SHIFT, p1, p2)
    if c is None:
        return
    (x1, y1), (x2, y2) = c
    dx, dy = x2 - x1, y2 - y1
    ax, ay = abs(dx), abs(dy)
    if ax > ay:
        if dx < 0:
            x1, x2, y1, y2 = x2, x1, y2, y1
            dy = -dy
        y_step = _tdiv(dy * XY_ONE, ax | 1)
        ecount = (x2 - x1) >> XY_SHIFT
    else:
        if dy < 0:
            x1, x2, y1, y2 = x2, x1, y2, y1
            dx = -dx
        x_step = _tdiv(dx * XY_ONE, ay | 1)
        ecount = (y2 - y1) >> XY_SHIFT
    x1 += XY_ONE >> 1
    y1 += XY_ONE >> 1

    def put(x, y):
        if 0 <= x < W and 0 <= y < H:
            emit(y, x, x)

    put((x2 + (XY_ONE >> 1)) >> XY_SHIFT, (y2 + (XY_ONE >> 1)) >> XY_SHIFT)
    if ax > ay:
        x1 >>= XY_SHIFT
        while ecount >= 0:
            put(x1, y1 >> XY_SHIFT)
            x1 += 1
            y1 += y_step
            ecount -= 1
    else:
        y1 >>= XY_SHIFT
        while ecount >= 0:
            put(x1 >> XY_SHIFT, y1)
            x1 += x_step
            y1 += 1
            ecount -= 1


def _fill_convex_poly(emit, W: int, H: int, v):
    """FillConvexPoly(..., LINE_8, XY_SHIFT) of fixed-point points v: the outline, then one span per scanline."""
    n = len(v)
    delta = XY_ONE >> 1
    p0 = v[n - 1]
    xmin = xmax = v[0][0]
    ymin = ymax = v[0][1]
    imin = 0
    for i in range(n):
        p = v[i]
        if p[1] < ymin:
            ymin, imin = p[1], i
        ymax = max(ymax, p[1])
        xmax = max(xmax, p[0])
        xmin = min(xmin, p[0])
        _line2(emit, W, H, p0, p)
        p0 = p
    xmin, xmax = (xmin + delta) >> XY_SHIFT, (xmax + delta) >> XY_SHIFT
    ymin, ymax = (ymin + delta) >> XY_SHIFT, (ymax + delta) >> XY_SHIFT
    if n < 3 or xmax < 0 or ymax < 0 or xmin >= W or ymin >= H:
        return
    ymax = min(ymax, H - 1)
    edge = [{"idx": imin, "di": 1, "x": -XY_ONE, "dx": 0, "ye": ymin},
            {"idx": imin, "di": n - 1, "x": -XY_ONE, "dx": 0, "ye": ymin}]
    edges = n
    y = ymin
    while True:
        for e in edge:
            if y >= e["ye"]:
                idx0 = e["idx"]
                idx = idx0 + e["di"]
                if idx >= n:
                    idx -= n
                while edges > 0:
                    edges -= 1
                    ty = (v[idx][1] + delta) >> XY_SHIFT
                    if ty > y:
                        xs, xe = v[idx0][0], v[idx][0]
                        e["ye"] = ty
                        e["dx"] = _tdiv((xe - xs) * 2 + (ty - y), 2 * (ty - y))
                        e["x"] = xs
                        e["idx"] = idx
                        break
                    idx0 = idx
                    idx += e["di"]
                    if idx >= n:
                        idx -= n
                else:
                    edges -= 1
        if edges < 0:
            break
        if y >= 0:
            left, right = (1, 0) if edge[0]["x"] > edge[1]["x"] else (0, 1)
            xx1 = (edge[left]["x"] + delta) >> XY_SHIFT
            xx2 = (edge[right]["x"] + delta) >> XY_SHIFT
            if xx2 >= 0 and xx1 < W:
                emit(y, max(xx1, 0), min(xx2, W - 1))
        edge[0]["x"] += edge[0]["dx"]
        edge[1]["x"] += edge[1]["dx"]
        y += 1
        if y > ymax:
            break


def _circle_r1(emit, W: int, H: int, cx: int, cy: int, fill: bool):
    """Circle(img, center, 1, color, fill): the plus sign (filled) or its four arms (unfilled)."""
    for yy, x0, x1 in ((cy, cx - 1, cx + 1), (cy - 1, cx, cx), (cy + 1, cx, cx)):
        if not 0 <= yy < H:
            continue
        if fill or x0 == x1:
            a, b = max(x0, 0), min(x1, W - 1)
            if a <= b:
                emit(yy, a, b)
        else:
            for x in (x0, x1):
                if 0 <= x < W:
                    emit(yy, x, x)


def _thick_line(emit, W: int, H: int, p0, p1, flags: int):
    """ThickLine(..., thickness 2, LINE_8, flags, XY_SHIFT) of fixed-point points."""
    dx = (p0[0] - p1[0]) / XY_ONE
    dy = (p1[1] - p0[1]) / XY_ONE
    r = dx * dx + dy * dy
    thickness = 2 << (XY_SHIFT - 1)
    if abs(r) > np.finfo(np.float64).eps:
        r = thickness / math.sqrt(r)
        dpx, dpy = _cv_round(dy * r), _cv_round(dx * r)
        pt = [(p0[0] + dpx, p0[1] + dpy), (p0[0] - dpx, p0[1] - dpy),
              (p1[0] - dpx, p1[1] - dpy), (p1[0] + dpx, p1[1] + dpy)]
        _fill_convex_poly(emit, W, H, pt)
    for i, p in enumerate((p0, p1)):
        if flags & (i + 1):
            _circle_r1(emit, W, H, (p[0] + (XY_ONE >> 1)) >> XY_SHIFT, (p[1] + (XY_ONE >> 1)) >> XY_SHIFT, True)


def cv_line(emit, W: int, H: int, p0, p1):
    """cv2.line(img, p0, p1, color, 2, LINE_8, 0): calls emit(y, x0, x1) for every span it paints.  cv2.line first
    clips the segment, in whole pixels, to the image grown by the thickness on every side (clipLine on
    Rect(-2, -2, W + 4, H + 4)), and draws nothing when it misses that rectangle."""
    c = _clip_line(W + 4, H + 4, (p0[0] + 2, p0[1] + 2), (p1[0] + 2, p1[1] + 2))
    if c is None:
        return
    (x0, y0), (x1, y1) = c
    _thick_line(emit, W, H, ((x0 - 2) << XY_SHIFT, (y0 - 2) << XY_SHIFT), ((x1 - 2) << XY_SHIFT, (y1 - 2) << XY_SHIFT),
                3)


def cv_circle(emit, W: int, H: int, c, thickness: int):
    """cv2.circle(img, c, 1, color, thickness, LINE_8, 0) for thickness 1 or 2."""
    if thickness == 1:
        _circle_r1(emit, W, H, c[0], c[1], False)
        return
    cx, cy = c[0] << XY_SHIFT, c[1] << XY_SHIFT
    # ellipse2Poly at 0, 90, 180, 270, 360 degrees with both axes XY_ONE: exact, no repeated points
    v = [(cx + XY_ONE, cy), (cx, cy + XY_ONE), (cx - XY_ONE, cy), (cx, cy - XY_ONE), (cx + XY_ONE, cy)]
    flags = 3
    for k in range(1, 5):
        _thick_line(emit, W, H, v[k - 1], v[k], flags)
        flags = 2


def paint(img: np.ndarray, color):
    """An emit that writes color into img[y, x0:x1 + 1] (img (H, W, C))."""
    def emit(y, x0, x1):
        img[y, x0:x1 + 1] = color
    return emit


# ---------------------------------------------------------------------------------------------- render_openpose
def overlay_params(kp: np.ndarray, W: int):
    """render_keypoints' setup for body keypoints kp (25, 3) float32 on an image of width W (shape[1]; the
    reference's `height` is shape[2] == 3): (draw at all, circle thickness), with line thickness 2 and radius 1."""
    kp = np.asarray(kp, np.float32)
    valid = kp[:, -1] > 0.1
    if valid.sum() == 0:
        return False, 0
    v = kp[valid][:, :-1]
    pw = v[:, 0].max() - v[:, 0].min()
    ph = v[:, 1].max() - v[:, 1].min()
    if not pw * ph > 0:
        return False, 0
    ratio = min(1, max(pw / W, ph / 3))
    thick_ratio = max(np.round(math.sqrt(W * 3) * (1.0 / 75.0) * ratio), 2)
    assert thick_ratio == 2, "image too wide for the overlay's fixed thicknesses"
    return True, 2 if ratio > 0.05 else 1


def render_openpose(img: np.ndarray, kp: np.ndarray, mutation: str | None = None) -> np.ndarray:
    """render_openpose(img, body_keypoints) for img (H, W, 3) float32 and kp (25, 3) float32.  `mutation` draws a
    deliberately wrong variant ("joints_first", "round" coordinates, a ">=" confidence test) so that the tests can show
    the golden tells it apart."""
    img = np.ascontiguousarray(img.copy())
    H, W = img.shape[:2]
    draw, thick_circle = overlay_params(kp, W)
    if not draw:
        return img
    ok = (lambda c: c >= np.float32(0.1)) if mutation == "ge" else (lambda c: c > 0.1)
    to_int = (lambda v: np.rint(v).astype(int)) if mutation == "round" else (lambda v: v.astype(int))

    def limbs():
        for i1, i2 in PAIRS:
            if ok(kp[i1, -1]) and ok(kp[i2, -1]):
                a = tuple(int(c) for c in to_int(kp[i1, :-1]))
                b = tuple(int(c) for c in to_int(kp[i2, :-1]))
                cv_line(paint(img, COLORS[i2 % len(COLORS)]), W, H, a, b)

    def joints():
        for part in range(len(kp)):
            if ok(kp[part, -1]):
                c = tuple(int(x) for x in to_int(kp[part, :-1]))
                cv_circle(paint(img, COLORS[part % len(COLORS)]), W, H, c, thick_circle)

    if mutation == "joints_first":
        joints()
        limbs()
    else:
        limbs()
        joints()
    return img


# ---------------------------------------------------------------------------------------------- the grid
def prepare_keypoints(kp: np.ndarray, img_res: int, gt: bool) -> np.ndarray:
    """visualize_tensorboard's keypoint handling (:75-97): (B, 44, 2) predictions or (B, 44, 3) GT -> (B, 25, 3)
    float32 body keypoints in pixels.  The caller's array is not modified."""
    kp = np.array(kp, np.float32)
    if gt:
        kp[:, :, :-1] = img_res * (kp[:, :, :-1] + 0.5)
    else:
        kp = np.concatenate((kp, np.ones_like(kp)[:, :, [0]]), axis=-1)
        kp = img_res * (kp + 0.5)
    body = kp[:, :25].copy()
    extra = kp[:, -19:]
    for b in range(kp.shape[0]):
        for i, j in KEYPOINT_MATCHES:
            if not gt or (extra[b, j, -1] > 0 and body[b, i, -1] == 0):
                body[b, i] = extra[b, j]
    return body


def skeleton_tile(image_chw: np.ndarray, body: np.ndarray, mutation: str | None = None) -> np.ndarray:
    """render_openpose(255 * crop, body) / 255 as a (3, H, W) float32 tile ("background_x": undrawn pixels keep the
    crop's x instead of fl32(fl32(255 x) / 255), a deliberately wrong variant)."""
    hwc = np.transpose(image_chw, (1, 2, 0))
    tile = np.transpose(render_openpose(255 * hwc.copy(), body, mutation) / 255, (2, 0, 1))
    if mutation == "background_x":
        bg = (np.float32(255) * image_chw) / np.float32(255)
        tile = np.where((tile == bg).all(0)[None], image_chw, tile)
    return tile


def make_grid(tiles, nrow: int, padding: int = 2) -> np.ndarray:
    """torchvision.utils.make_grid(tiles, nrow, padding, pad_value=0) for (3, H, W) tiles."""
    n = len(tiles)
    C, H, W = tiles[0].shape
    xmaps = min(nrow, n)
    ymaps = int(math.ceil(n / xmaps))
    h, w = H + padding, W + padding
    grid = np.zeros((C, h * ymaps + padding, w * xmaps + padding), np.float32)
    for k, t in enumerate(tiles):
        y, x = divmod(k, xmaps)
        grid[:, y * h + padding:y * h + padding + H, x * w + padding:x * w + padding + W] = t
    return grid


def visualize_tensorboard(images, front, side, pred_keypoints, gt_keypoints, img_res: int, nrow: int = 5,
                          padding: int = 2) -> np.ndarray:
    """The grid of visualize_tensorboard from the crops (B, 3, H, W) float32 and the mesh tiles front / side
    (B, 3, H, W)."""
    nrow = nrow - 1 if gt_keypoints is None else nrow
    nrow = nrow - 1 if pred_keypoints is None else nrow
    pred = None if pred_keypoints is None else prepare_keypoints(pred_keypoints, img_res, gt=False)
    gt = None if gt_keypoints is None else prepare_keypoints(gt_keypoints, img_res, gt=True)
    tiles = []
    for i in range(images.shape[0]):
        tiles += [images[i], front[i], side[i]]
        if pred is not None:
            tiles.append(skeleton_tile(images[i], pred[i]))
        if gt is not None:
            tiles.append(skeleton_tile(images[i], gt[i]))
    return make_grid(tiles, nrow, padding)


# ---------------------------------------------------------------------------------------------- the live reference
def _ref_file(rel: str):
    from . import ref_import
    if not ref_import.available():
        raise FileNotFoundError(f"reference tree not found at {ref_import.REF_ROOT}")
    return ref_import.REF_ROOT / "tokenhmr" / "lib" / "utils" / rel


def live_render_openpose():
    """The live render_openpose.py (cv2 + numpy only), imported from its file with `np.int = int`: NumPy 1.24 removed
    np.int, which render_openpose.py:79, 89 still use."""
    import importlib.util
    np.int = int
    spec = importlib.util.spec_from_file_location("_ref_render_openpose", _ref_file("render_openpose.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod.render_openpose


class _Trimesh:
    def __init__(self, vertices, faces):
        self.vertices, self.faces = np.asarray(vertices, np.float64), faces
        self.transform = np.eye(4)

    def apply_transform(self, m):
        self.transform = np.asarray(m, np.float64) @ self.transform


def _rotation_matrix(angle, direction):
    from . import render_oracle
    m = np.eye(4)
    m[:3, :3] = render_oracle.rot_axis(angle, direction)
    return m


class _Mesh:
    def __init__(self, tm, material):
        self.tm, self.material = tm, material


class _Camera:
    def __init__(self, fx, fy, cx, cy):
        self.fx, self.fy, self.cx, self.cy = fx, fy, cx, cy


class _Scene:
    def __init__(self, bg_color=None, ambient_light=None):
        self.rec = {"bg_color": bg_color, "ambient": ambient_light, "lights": []}

    def add(self, obj, name=None, pose=None):
        if isinstance(obj, _Mesh):
            self.rec.update(mesh_transform=obj.tm.transform, vertices=obj.tm.vertices, material=obj.material)
        else:
            self.rec.update(camera_pose=np.array(pose, np.float64), focal=(obj.fx, obj.fy), center=(obj.cx, obj.cy))

    def add_node(self, node):
        self.rec["lights"].append(node)


def load_live(mesh_image):
    """The live mesh_renderer.py (needs TOKENHMR_REFERENCE, cv2 and torchvision) with recording pyrender / trimesh
    stand-ins.  Each OffscreenRenderer.render appends the scene's record {'camera_pose', 'mesh_transform',
    'vertices', 'width', 'height', 'focal', 'center', 'bg_color', 'ambient', 'lights', 'material'} to `records` and
    returns mesh_image(record), an (H, W, 4) uint8 RGBA image, as pyrender's colour buffer.  Returns
    (MeshRenderer class, records); call it only inside `with live_modules():`."""
    import importlib
    import os
    import sys
    from . import ref_import
    _ref_file("mesh_renderer.py")
    ref_import.load_modules()
    records = []

    class _Renderer:
        def __init__(self, viewport_width, viewport_height, point_size=1.0):
            self.w, self.h = viewport_width, viewport_height

        def render(self, scene, flags=None):
            rec = dict(scene.rec, width=self.w, height=self.h)
            records.append(rec)
            return mesh_image(rec), None

        def delete(self):
            pass

    pyrender = types.ModuleType("pyrender")
    pyrender.OffscreenRenderer, pyrender.Scene, pyrender.IntrinsicsCamera = _Renderer, _Scene, _Camera
    pyrender.Mesh = types.SimpleNamespace(from_trimesh=lambda tm, material=None: _Mesh(tm, material))
    pyrender.MetallicRoughnessMaterial = lambda **kw: kw
    pyrender.Node = lambda **kw: kw
    pyrender.DirectionalLight = lambda **kw: kw
    pyrender.RenderFlags = types.SimpleNamespace(RGBA=1)
    trimesh = types.ModuleType("trimesh")
    trimesh.Trimesh = _Trimesh
    trimesh.transformations = types.SimpleNamespace(rotation_matrix=_rotation_matrix)
    np.int = int
    saved = {k: sys.modules.get(k) for k in ("pyrender", "trimesh")}
    prev = os.environ.get("PYOPENGL_PLATFORM")
    sys.modules.update(pyrender=pyrender, trimesh=trimesh)
    try:
        sys.modules.pop("lib.utils.mesh_renderer", None)
        sys.modules.pop("lib.utils.render_openpose", None)
        mod = importlib.import_module("lib.utils.mesh_renderer")   # sets PYOPENGL_PLATFORM at import
    finally:
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v
        if prev is None:
            os.environ.pop("PYOPENGL_PLATFORM", None)
        else:
            os.environ["PYOPENGL_PLATFORM"] = prev
    mod.pyrender, mod.trimesh = pyrender, trimesh
    raymond = mod.create_raymond_lights

    def create_raymond_lights():   # it does its own `import pyrender`: hand it the stand-in for the call
        before = sys.modules.get("pyrender")
        sys.modules["pyrender"] = pyrender
        try:
            return raymond()
        finally:
            if before is None:
                sys.modules.pop("pyrender", None)
            else:
                sys.modules["pyrender"] = before

    mod.create_raymond_lights = create_raymond_lights
    return mod.MeshRenderer, records


# ---------------------------------------------------------------------------------------------- the golden
def oracle_mesh_image(faces):
    """A stand-in renderer image: the float64 render oracle (oracle/render_oracle.py) of the recorded scene, quantised
    to uint8 RGBA as pyrender's colour buffer is (alpha 255 where covered)."""
    from . import render_oracle as RO

    def image(rec):
        W, H = int(rec["width"]), int(rec["height"])
        v = np.asarray(rec["vertices"], np.float64)
        M = rec["mesh_transform"]
        world = v @ M[:3, :3].T + M[:3, 3]
        cam_t = rec["camera_pose"][:3, 3]
        col, row, depth = RO._pyrender_project(world, cam_t, float(rec["focal"][0]), W, H)
        r = RO.raster(np.stack([col, row], -1)[None], depth[None], faces, W, H)
        q = (world - cam_t) * np.array([1.0, -1.0, -1.0])
        lights = [(0, np.asarray(nd["matrix"], float)[:3, 2] * np.array([1.0, -1.0, -1.0]), 1.0) for nd in rec["lights"]]
        out = np.zeros((H * W, 4), np.uint8)
        if r["pix"].size:
            c = RO.shade(r, q[None], faces, lights, rec["material"]["baseColorFactor"][:3], ambient=rec["ambient"][0])
            out[r["pix"], :3] = np.rint(c * 255)
            out[r["pix"], 3] = 255
        return out.reshape(H, W, 4)
    return image


def golden_inputs(B: int, seed: int, H: int = 256, W: int = 256):
    """Seeded inputs of one golden case: crops in [0, 1], a coarse mesh per sample, pred_cam_t, and keypoints that
    reach off the image and onto its border, with GT confidences of 0, float32(0.1) (not drawn), 0.3 and 1."""
    import sys
    from pathlib import Path
    sys.path.insert(0, str(Path(__file__).resolve().parent.parent / "tests"))
    from render_mesh import ellipsoid
    rng = np.random.default_rng(seed)
    v0, faces = ellipsoid((0.3, 0.8, 0.2))
    ang = rng.uniform(-np.pi, np.pi, B)
    Rs = np.stack([np.array([[np.cos(a), 0, np.sin(a)], [0, 1, 0], [-np.sin(a), 0, np.cos(a)]]) for a in ang])
    verts = np.einsum("bij,vj->bvi", Rs, v0.astype(np.float64)).astype(np.float32)
    cam_t = np.stack([rng.uniform(-0.2, 0.2, B), rng.uniform(-0.2, 0.2, B), rng.uniform(25, 45, B)], 1).astype(np.float32)
    images = rng.random((B, 3, H, W), dtype=np.float32)
    pred = rng.uniform(-0.45, 0.45, (B, 44, 2)).astype(np.float32)
    pred[:, rng.integers(0, 44, 4)] = rng.uniform(-0.7, 0.7, (B, 4, 2)).astype(np.float32)   # off the image
    gt = np.concatenate([rng.uniform(-0.55, 0.55, (B, 44, 2)),
                         rng.choice(np.array([0, np.float32(0.1), 0.3, 1.0], np.float32), (B, 44, 1))], -1)
    gt = gt.astype(np.float32)
    gt[:, 3, :2] = np.float32(-0.5)                       # exactly on the top-left border: pixel 0
    gt[:, 5, :2] = np.float32(0.5 - 1.0 / W)              # last pixel
    return verts, faces, cam_t, images, pred, gt


def tile_slices(b: int, slot: int, H: int, W: int, tiles: int, padding: int = 2):
    """Rows and columns of sample b's tile `slot` in a make_grid with one sample per grid row."""
    y0, x0 = b * (H + padding) + padding, slot * (W + padding) + padding
    return slice(y0, y0 + H), slice(x0, x0 + W)


def encode_skeleton(tile: np.ndarray, image: np.ndarray) -> np.ndarray:
    """Lossless code of a skeleton tile (3, H, W) over its crop: 0 where it is the background fl32(fl32(255 x) / 255)
    on every channel, j + 1 where it is joint j's colour / 255 (float32).  Raises if a pixel is neither."""
    bg = (np.float32(255) * image) / np.float32(255)
    code = np.where((tile == bg).all(0), 0, 255).astype(np.uint8)
    for j in range(COLORS.shape[0] - 1, -1, -1):
        col = (COLORS[j].astype(np.float32) / np.float32(255))[:, None, None]
        code[(code == 255) & (tile == col).all(0)] = j + 1
    assert not (code == 255).any(), "a skeleton pixel is neither background nor a joint colour"
    return code


def decode_skeleton(code: np.ndarray, image: np.ndarray) -> np.ndarray:
    bg = (np.float32(255) * image) / np.float32(255)
    cols = np.concatenate([np.zeros((1, 3), np.float32), COLORS.astype(np.float32) / np.float32(255)])
    return np.where(code[None] == 0, bg, np.transpose(cols[code], (2, 0, 1))).astype(np.float32)


GOLDEN_CASES = ((1, 11), (8, 12), (64, 13))
GOLDEN_VARIANTS = {"both": (True, True), "pred": (True, False), "gt": (False, True), "none": (False, False)}


def write_golden(path) -> None:
    """tests/golden/mesh_renderer_reference.npz from the LIVE mesh_renderer.py, render_openpose.py, cv2 and
    torchvision make_grid (python -m oracle.openpose_oracle; needs TOKENHMR_REFERENCE).  Per case and keypoint
    variant it keeps the grid's shape, every skeleton tile as encode_skeleton's lossless code, and the recorded
    camera x of every scene; the crops and pads are checked here to be the crop and 0.  The crops are regenerated
    from the seed (golden_inputs; their SHA-256 is stored)."""
    import hashlib
    import torch
    from . import ref_import
    out = {}
    for B, seed in GOLDEN_CASES:
        verts, faces, cam_t, images, pred, gt = golden_inputs(B, seed)
        H, W = images.shape[2:]
        MR, records = load_live(oracle_mesh_image(faces))
        mr = MR(ref_import._Cfg({"EXTRA": {"FOCAL_LENGTH": 5000.0}, "MODEL": {"IMAGE_SIZE": 256}}), faces)
        for name, (use_p, use_g) in GOLDEN_VARIANTS.items():
            if B != 8 and name != "both":
                continue
            records.clear()
            grid = mr.visualize_tensorboard(verts.copy(), cam_t.copy(), images.copy(),
                                            pred.copy() if use_p else None, gt.copy() if use_g else None,
                                            focal_length=np.full((B, 2), 123.0, np.float32))
            assert isinstance(grid, torch.Tensor) and grid.dtype == torch.float32
            grid = grid.numpy()
            tiles = 3 + use_p + use_g
            assert grid.shape == (3, B * (H + 2) + 2, tiles * (W + 2) + 2)
            covered = np.zeros(grid.shape[1:], bool)
            codes = []
            for b in range(B):
                for slot in range(tiles):
                    ys, xs = tile_slices(b, slot, H, W, tiles)
                    covered[ys, xs] = True
                    if slot == 0:
                        assert np.array_equal(grid[:, ys, xs], images[b])
                    elif slot >= 3:
                        codes.append(encode_skeleton(grid[:, ys, xs], images[b]))
            assert (grid[:, ~covered] == 0).all()
            key = f"b{B}_{name}"
            out[f"shape_{key}"] = np.array(grid.shape)
            if codes:
                out[f"codes_{key}"] = np.stack(codes).reshape(B, tiles - 3, H, W)
            out[f"cam_x_{key}"] = np.array([r["camera_pose"][0, 3] for r in records])
            out[f"focal_{key}"] = np.array([r["focal"][0] for r in records])
        out.update({f"cam_t_b{B}": cam_t, f"pred_b{B}": pred, f"gt_b{B}": gt,
                    f"images_sha_b{B}": np.frombuffer(hashlib.sha256(images.tobytes()).digest(), np.uint8)})
    np.savez_compressed(path, **out)


if __name__ == "__main__":
    from pathlib import Path
    dst = Path(__file__).resolve().parent.parent / "tests" / "golden" / "mesh_renderer_reference.npz"
    write_golden(dst)
    print(dst)

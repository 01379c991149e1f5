"""GPU mesh rendering behind the reference's `Renderer` (tokenhmr/lib/utils/renderer.py:137-359).

`Renderer(cfg, faces)` has the reference's `__call__` and `render_rgba_multiple` signatures and return types
(HWC float32 numpy arrays), so that demo.py swaps only its import; `render_crops` renders every person of a batch in
one call and returns CUDA tensors.  The rasterizer, shading and compositing run in libtokenhmr_b200.so
(`thmr_render_meshes`, csrc/render.cuh); Python only builds the descriptor and allocates tensors.  There is no
pyrender / OpenGL path and no CPU fallback.

Geometry follows the reference's camera chain exactly (DESIGN.md §2 "Rendering"): it reduces to the model's own
`perspective_projection` of v + t with the principal point at (W/2, H/2).  Shading is a stated model, not pyrender's
metallic-roughness shader:  base * clamp(ambient + sum_dir I max(0, n.l) + sum_point I max(0, n.l) / d^2, 0, 1),
quantised to k/255, with the reference's own light rig.  How close that is to pyrender's tone is NOT verified.
Edges are not anti-aliased (one sample per pixel centre).

    renderer = Renderer(model_cfg, faces=model.smpl.faces)
    img = renderer(verts, cam_t, batch['img'][n], mesh_base_color=LIGHT_BLUE, scene_bg_color=(1, 1, 1))
    crops = renderer.render_crops(out['pred_vertices'], out['pred_cam_t'], batch['img'])      # (B, 256, 256, 3) CUDA
"""
from __future__ import annotations

import ctypes
from typing import Dict, List, Optional, Sequence

import numpy as np
import torch

from . import _lib
from ._lib import ThmrError, check, lib

ZNEAR = 0.05            # pyrender.IntrinsicsCamera default (renderer.py:208-209 leaves it unset)
AMBIENT = 0.3           # renderer.py:202, 286, 334
DEFAULT_MEAN = (0.485, 0.456, 0.406)
DEFAULT_STD = (0.229, 0.224, 0.225)


def rotation_matrix(angle_rad: float, axis: Sequence[float]) -> np.ndarray:
    """trimesh.transformations.rotation_matrix(angle, axis)[:3, :3] (rotation about an axis through the origin)."""
    a = np.asarray(axis, dtype=np.float64)
    n = np.linalg.norm(a)
    if not n > 0:
        raise ThmrError(f"rotation axis {axis} has no direction")
    a = a / n
    c, s = np.cos(angle_rad), np.sin(angle_rad)
    K = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
    return c * np.eye(3) + s * K + (1 - c) * np.outer(a, a)


# ---- the reference's light rig, in pyrender's scene frame (x right, y up, z towards the viewer) --------------------
def raymond_directions() -> np.ndarray:
    """Direction towards each of the three create_raymond_lights (renderer.py:106-135): the +z column of each node."""
    thetas = np.pi * np.array([1.0 / 6.0] * 3)
    phis = np.pi * np.array([0.0, 2.0 / 3.0, 4.0 / 3.0])
    z = np.stack([np.sin(thetas) * np.cos(phis), np.sin(thetas) * np.sin(phis), np.cos(thetas)], axis=1)
    return z / np.linalg.norm(z, axis=1, keepdims=True)


def light_pose_columns(dist: float, n_lights: int = 5, elevation: float = np.pi / 3) -> np.ndarray:
    """get_light_poses (renderer.py:25-35) + the appended identity (:364, :380): per light, the pose's +z column and
    its position, [n + 1, 2, 3].  R = Ry(phi) Rx(-elevation), so +z = (sin phi cos e, sin e, cos phi cos e)."""
    out = []
    for k in range(n_lights):
        phi = 2 * np.pi * k / n_lights
        z = np.array([np.sin(phi) * np.cos(elevation), np.sin(elevation), np.cos(phi) * np.cos(elevation)])
        out.append((z, dist * z))
    out.append((np.array([0.0, 0.0, 1.0]), np.zeros(3)))
    return np.array(out)


def scene_to_camera(v: np.ndarray) -> np.ndarray:
    """pyrender's scene frame -> the model's camera frame (x right, y down, z forward): the 180° turn about x
    (renderer.py:196-198, 248-250) with an identity camera rotation."""
    return np.asarray(v, dtype=np.float64) * np.array([1.0, -1.0, -1.0])


def crop_lights() -> List[tuple]:
    """Renderer.__call__: ambient 0.3 + the three Raymond directionals (intensity 1)."""
    return [(_lib.LIGHT_DIRECTIONAL, scene_to_camera(d), 1.0) for d in raymond_directions()]


def multiple_lights() -> List[tuple]:
    """render_rgba_multiple: add_point_lighting (dist 0.5), add_lighting (dist 12) and the Raymond directionals,
    with the camera at the scene origin (renderer.py:338-353)."""
    lights = [(_lib.LIGHT_POINT, scene_to_camera(p), 1.0) for _, p in light_pose_columns(0.5)]
    lights += [(_lib.LIGHT_DIRECTIONAL, scene_to_camera(z), 1.0) for z, _ in light_pose_columns(12.0)]
    return lights + crop_lights()


def _cfg_get(cfg, path: str, default):
    node = cfg
    for k in path.split("."):
        if node is None:
            return default
        node = node.get(k) if isinstance(node, dict) else getattr(node, k, None)
    return default if node is None else node


class Renderer:
    """Drop-in for the reference's `Renderer(cfg, faces)` (renderer.py:137-151)."""

    def __init__(self, cfg, faces, device: str | torch.device = "cuda:0"):
        self.cfg = cfg
        # the reference's CfgNode (EXTRA.FOCAL_LENGTH, MODEL.IMAGE_SIZE / IMAGE_MEAN / IMAGE_STD) or a TokenHMRConfig
        self.focal_length = float(_cfg_get(cfg, "EXTRA.FOCAL_LENGTH", getattr(cfg, "focal_length", 5000.0)))
        self.img_res = int(_cfg_get(cfg, "MODEL.IMAGE_SIZE", getattr(cfg, "image_size", 256)))
        self.mean = tuple(float(x) for x in _cfg_get(cfg, "MODEL.IMAGE_MEAN", DEFAULT_MEAN))
        self.std = tuple(float(x) for x in _cfg_get(cfg, "MODEL.IMAGE_STD", DEFAULT_STD))
        self.camera_center = [self.img_res // 2, self.img_res // 2]
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise ThmrError("Renderer needs a CUDA device (there is no CPU fallback)")
        faces_np = faces.detach().cpu().numpy() if torch.is_tensor(faces) else np.asarray(faces)
        if faces_np.ndim != 2 or faces_np.shape[1] != 3 or faces_np.shape[0] == 0:
            raise ThmrError(f"faces must be (F, 3), got {faces_np.shape}")
        self.faces = faces_np
        self.num_verts = int(faces_np.max()) + 1
        f32 = np.ascontiguousarray(faces_np, dtype=np.int32)
        h = ctypes.c_void_p()
        check(lib().thmr_render_topology_create(f32.ctypes.data, f32.shape[0], self.num_verts, ctypes.byref(h)))
        self._topo = h
        self._ws: Optional[torch.Tensor] = None

    def __del__(self):
        h = getattr(self, "_topo", None)
        if h is not None and h.value and _lib._lib is not None:
            _lib._lib.thmr_render_topology_destroy(h)
            self._topo = None

    # ---------------------------------------------------------------------------------------- the one GPU call
    def raster(self, vertices: torch.Tensor, translations: torch.Tensor, width: int, height: int, focal: float, *,
               rotation=None, rotate_translation: bool = False, mesh_image: Optional[Sequence[int]] = None,
               n_images: Optional[int] = None, lights=(), ambient: float = AMBIENT, base_color=(1.0, 1.0, 0.9),
               bg_color=(0.0, 0.0, 0.0), bg_image: Optional[torch.Tensor] = None, bg_layout: int = _lib.BG_NONE,
               outputs: Sequence[str] = ("rgba",), out: Optional[Dict[str, torch.Tensor]] = None,
               znear: float = ZNEAR, workspace: Optional[torch.Tensor] = None) -> Dict[str, torch.Tensor]:
        """thmr_render_meshes on CUDA tensors: vertices (n, V, 3), translations (n, 3) in the model's camera frame.
        Returns the requested outputs among rgba (n_images, H, W, 4), composite (.., 3), face_id (.., int32), depth.
        `out` may hold preallocated output tensors and `workspace` a uint8 CUDA tensor of at least
        workspace_bytes(...) bytes.  Without `workspace` the call uses this Renderer's own workspace, which a larger
        call replaces and which is shared by every call: a call captured in a CUDA graph, or calls running at the same
        time on different streams, must each pass a workspace of their own that lives as long as the graph."""
        dev = self.device
        v = vertices.to(dev, torch.float32).contiguous()
        t = translations.to(dev, torch.float32).contiguous()
        if v.dim() != 3 or v.shape[2] != 3 or v.shape[1] != self.num_verts:
            raise ThmrError(f"vertices must be (n, {self.num_verts}, 3), got {tuple(v.shape)}")
        n = v.shape[0]
        if t.shape != (n, 3):
            raise ThmrError(f"translations must be ({n}, 3), got {tuple(t.shape)}")
        if len(lights) > _lib.RENDER_MAX_LIGHTS:
            raise ThmrError(f"at most {_lib.RENDER_MAX_LIGHTS} lights")
        n_images = n if n_images is None else int(n_images)
        d = _lib.RenderDesc()
        d.topology = self._topo.value
        d.n_meshes, d.n_images = n, n_images
        mi = None
        if mesh_image is not None:
            mi = np.ascontiguousarray(mesh_image, dtype=np.int32)
            if mi.shape != (n,):
                raise ThmrError(f"mesh_image must have {n} entries")
            d.mesh_image_host = mi.ctypes.data_as(ctypes.POINTER(ctypes.c_int32))
        d.vertices, d.translations = v.data_ptr(), t.data_ptr()
        R = np.eye(3) if rotation is None else np.asarray(rotation, dtype=np.float64)
        d.rotation[:] = [float(x) for x in R.reshape(9)]
        d.rotate_translation = int(bool(rotate_translation))
        d.width, d.height, d.focal, d.znear = int(width), int(height), float(focal), float(znear)
        d.base_color[:] = [float(x) for x in base_color[:3]]
        d.bg_color[:] = [float(x) for x in bg_color[:3]]
        d.ambient = float(ambient)
        d.n_lights = len(lights)
        for i, (kind, vec, intensity) in enumerate(lights):
            d.lights[i].type = int(kind)
            d.lights[i].vec[:] = [float(x) for x in vec]
            d.lights[i].intensity = float(intensity)
        bg = None
        if bg_image is not None:
            bg = bg_image.to(dev, torch.float32).contiguous()
            d.bg_layout, d.bg_image = int(bg_layout), bg.data_ptr()
        d.mean[:], d.std[:] = list(self.mean), list(self.std)
        H, W = int(height), int(width)
        shapes = {"rgba": ((n_images, H, W, 4), torch.float32), "composite": ((n_images, H, W, 3), torch.float32),
                  "face_id": ((n_images, H, W), torch.int32), "depth": ((n_images, H, W), torch.float32)}
        res = {}
        with torch.cuda.device(dev):
            for k in outputs:
                shape, dt = shapes[k]
                o = out.get(k) if out else None
                if o is None:
                    o = torch.empty(shape, dtype=dt, device=dev)
                elif tuple(o.shape) != shape or o.dtype != dt or not o.is_contiguous():
                    raise ThmrError(f"out[{k!r}] must be a contiguous {dt} tensor of shape {shape}")
                res[k] = o
                setattr(d, k, o.data_ptr())
            need = self.workspace_bytes(n, n_images, W, H)
            if workspace is not None:
                if workspace.device != dev or workspace.dtype != torch.uint8 or workspace.numel() < need:
                    raise ThmrError(f"workspace must be a uint8 tensor of at least {need} bytes on {dev}")
                ws = workspace
            else:
                if self._ws is None or self._ws.numel() < need:
                    self._ws = torch.empty(need, dtype=torch.uint8, device=dev)
                ws = self._ws
            check(lib().thmr_render_meshes(ctypes.byref(d), ws.data_ptr(), torch.cuda.current_stream().cuda_stream))
        return res

    def workspace_bytes(self, n_meshes: int, n_images: int, width: int, height: int) -> int:
        """Bytes of workspace one raster() call of these sizes needs."""
        need = lib().thmr_render_workspace_bytes(self._topo.value, int(n_meshes), int(n_images), int(width),
                                                 int(height))
        if need == 0:
            raise ThmrError(f"bad render size: {n_meshes} meshes, {n_images} images of {width}x{height}")
        return need

    # ---------------------------------------------------------------------------------------- reference surface
    def render_crops(self, vertices, cam_t, imgs, side_view: bool = False, rot_angle: float = 90,
                     mesh_base_color=(1.0, 1.0, 0.9), scene_bg_color=(0, 0, 0),
                     return_rgba: bool = False) -> torch.Tensor:
        """Renderer.__call__ for every person of a batch in one call: vertices (B, V, 3), cam_t (B, 3) (the model's
        pred_cam_t, not x-flipped), imgs (B, 3, H, W) normalised crops.  Returns (B, H, W, 3) CUDA tensors: the
        composite over the un-normalised crop, the mesh colour alone with side_view, or (B, H, W, 4) RGBA."""
        imgs = torch.as_tensor(imgs)
        if imgs.dim() != 4 or imgs.shape[1] != 3:
            raise ThmrError(f"imgs must be (B, 3, H, W), got {tuple(imgs.shape)}")
        B, _, H, W = imgs.shape
        R = rotation_matrix(np.radians(rot_angle), [0, 1, 0]) if side_view else None
        want = "rgba" if (return_rgba or side_view) else "composite"
        res = self.raster(torch.as_tensor(vertices), torch.as_tensor(cam_t), W, H, self.focal_length, rotation=R,
                          lights=crop_lights(), base_color=mesh_base_color, bg_color=scene_bg_color,
                          bg_image=None if want == "rgba" else imgs, bg_layout=_lib.BG_CHW_NORMALIZED,
                          outputs=(want,))
        if return_rgba:
            return res["rgba"]
        return res["rgba"][..., :3] if side_view else res["composite"]

    def __call__(self, vertices, camera_translation, image, full_frame: bool = False, imgname: Optional[str] = None,
                 side_view=False, rot_angle=90, mesh_base_color=(1.0, 1.0, 0.9), scene_bg_color=(0, 0, 0),
                 return_rgba=False) -> np.ndarray:
        """Renderer.__call__ (renderer.py:153-231): vertices (V, 3), camera_translation (3,), image (3, H, W)
        normalised crop; returns (H, W, 3) float32 (or (H, W, 4) with return_rgba).  Unlike the reference, the
        caller's camera_translation is not modified."""
        v = torch.as_tensor(np.asarray(vertices) if not torch.is_tensor(vertices) else vertices)[None]
        t = torch.as_tensor(np.asarray(camera_translation) if not torch.is_tensor(camera_translation)
                            else camera_translation).reshape(1, 3)
        if not full_frame:
            out = self.render_crops(v, t, torch.as_tensor(image)[None], side_view=side_view, rot_angle=rot_angle,
                                    mesh_base_color=mesh_base_color, scene_bg_color=scene_bg_color,
                                    return_rgba=return_rgba)
            return out[0].cpu().numpy()
        import cv2
        frame = cv2.imread(str(imgname))
        if frame is None:
            raise ThmrError(f"cannot read {imgname}")
        bg = torch.from_numpy(np.ascontiguousarray(frame.astype(np.float32)[:, :, ::-1] / 255.))[None]
        H, W = frame.shape[:2]
        R = rotation_matrix(np.radians(rot_angle), [0, 1, 0]) if side_view else None
        res = self.raster(v, t, W, H, self.focal_length, rotation=R, lights=crop_lights(),
                          base_color=mesh_base_color, bg_color=scene_bg_color, bg_image=bg, bg_layout=_lib.BG_HWC,
                          outputs=("rgba", "composite"))
        if return_rgba:
            return res["rgba"][0].cpu().numpy()
        return (res["rgba"][0, ..., :3] if side_view else res["composite"][0]).cpu().numpy()

    def render_rgba_multiple(self, vertices: List, cam_t: List, rot_axis=(1, 0, 0), rot_angle=0,
                             mesh_base_color=(1.0, 1.0, 0.9), scene_bg_color=(0, 0, 0), render_res=(256, 256),
                             focal_length=None) -> np.ndarray:
        """render_rgba_multiple (renderer.py:311-359): all meshes in one (H, W, 4) float32 image, render_res = (W, H),
        camera at the origin, each mesh at v + cam_t (not x-flipped), rotated by rot_angle degrees about rot_axis."""
        if len(vertices) == 0 or len(vertices) != len(cam_t):
            raise ThmrError("render_rgba_multiple needs one cam_t per mesh and at least one mesh")
        v = torch.stack([torch.as_tensor(np.asarray(x) if not torch.is_tensor(x) else x).float() for x in vertices])
        t = torch.stack([torch.as_tensor(np.asarray(x) if not torch.is_tensor(x) else x).float().reshape(3)
                         for x in cam_t])
        W, H = (int(round(float(x))) for x in render_res)
        focal = float(focal_length) if focal_length is not None else self.focal_length
        R = rotation_matrix(np.radians(float(rot_angle)), rot_axis)
        res = self.raster(v, t, W, H, focal, rotation=R, rotate_translation=True, mesh_image=[0] * v.shape[0],
                          n_images=1, lights=multiple_lights(), base_color=mesh_base_color, bg_color=scene_bg_color)
        return res["rgba"][0].cpu().numpy()


def _cuda_f32(x, dev: torch.device, name: str, shape_tail: Sequence[Optional[int]]) -> torch.Tensor:
    """numpy array or tensor -> contiguous float32 tensor on dev, with its trailing dimensions checked."""
    t = torch.as_tensor(np.asarray(x) if not torch.is_tensor(x) else x)
    if t.dim() != len(shape_tail) or any(w is not None and s != w for s, w in zip(t.shape, shape_tail)):
        want = ", ".join("*" if w is None else str(w) for w in shape_tail)
        raise ThmrError(f"{name} must be ({want}), got {tuple(t.shape)}")
    return t.to(dev, torch.float32).contiguous()


class MeshRenderer:
    """Drop-in for the reference's `MeshRenderer(cfg, faces)` (tokenhmr/lib/utils/mesh_renderer.py:44-157), the
    renderer eval.py --render uses.  `visualize_tensorboard` returns the reference's grid -- per sample the crop, the
    front mesh view, the side mesh view and the OpenPose skeletons of the predicted and GT keypoints -- as a CUDA
    float32 (3, H', W') tensor, so eval.py's `.cpu().numpy()` keeps working.  The mesh tiles come from
    `Renderer.raster`; the skeletons and the grid from `thmr_pose_grid` (csrc/keypoints.cuh), which draws them bit
    for bit as the reference's render_openpose draws them with OpenCV.  Inputs may be numpy arrays (what eval.py
    passes) or CUDA tensors (then nothing waits for the host); they are taken as float32, eval.py's dtype.

    Reference behaviour kept on purpose (DESIGN.md §2 "Rendering"):
      * the focal length is always cfg.EXTRA.FOCAL_LENGTH; visualize*'s `focal_length` argument is ignored (:82);
      * `__call__` flips camera_translation[0] in place (:118), so visualize*'s side view gets the row its front view
        already flipped and flips it back: the side view is rendered as if pred_cam_t had x negated.  This class
        renders that side view without touching the caller's arrays;
      * predicted keypoints get a confidence of img_res * 1.5 (the ones column is scaled too, :76-77) and always
        take the 14 extra-joint substitutions; GT keypoints take one only where the extra joint's confidence is > 0
        and the body joint's == 0 (:84-96).
    Unlike the reference, no argument is modified (the reference scales gt_keypoints in place)."""

    def __init__(self, cfg, faces=None, device: str | torch.device = "cuda:0"):
        if faces is None:
            raise ThmrError("MeshRenderer needs the mesh faces")
        self.cfg = cfg
        self.focal_length = float(_cfg_get(cfg, "EXTRA.FOCAL_LENGTH", getattr(cfg, "focal_length", 5000.0)))
        self.img_res = int(_cfg_get(cfg, "MODEL.IMAGE_SIZE", getattr(cfg, "image_size", 256)))
        self.camera_center = [self.img_res // 2, self.img_res // 2]
        # the mesh tiles composite over the already un-normalised crop: mean 0 and std 1 make img * std + mean exact
        self.renderer = Renderer({"EXTRA": {"FOCAL_LENGTH": self.focal_length},
                                  "MODEL": {"IMAGE_SIZE": self.img_res, "IMAGE_MEAN": [0.0, 0.0, 0.0],
                                            "IMAGE_STD": [1.0, 1.0, 1.0]}}, faces, device)
        self.faces = self.renderer.faces
        self.device = self.renderer.device

    # ---------------------------------------------------------------------------------------------- mesh tiles
    def _front(self, v, t, imgs, focal, base, ws=None):
        """(B, H, W, 3): the mesh over the crop, color * (alpha > 0.8) + (1 - mask) * crop (:146-151)."""
        H, W = imgs.shape[2:]
        return self.renderer.raster(v, t, W, H, focal, lights=crop_lights(), base_color=base, bg_image=imgs,
                                    bg_layout=_lib.BG_CHW_NORMALIZED, outputs=("composite",),
                                    workspace=ws)["composite"]

    def _side(self, v, t, H, W, focal, base, rot_angle=90.0, ws=None):
        """(B, H, W, 4): the mesh turned rot_angle degrees about y over white; rgb is the tile."""
        Ry = rotation_matrix(np.radians(rot_angle), [0, 1, 0])
        return self.renderer.raster(v, t, W, H, focal, rotation=Ry, lights=crop_lights(), base_color=base,
                                    bg_color=(1.0, 1.0, 1.0), outputs=("rgba",), workspace=ws)["rgba"]

    def __call__(self, vertices, camera_translation, image, focal_length=5000, text=None, resize=None,
                 side_view=False, baseColorFactor=(1.0, 1.0, 0.9, 1.0), rot_angle=90) -> np.ndarray:
        """MeshRenderer.__call__ (:109-157): vertices (V, 3), camera_translation (3,) (pred_cam_t), image (H, W, 3)
        in [0, 1]; returns (H, W, 3) float32.  `text` is unused, as in the reference; `resize` is not supported.
        Unlike the reference, camera_translation is not flipped in place, so every call renders it unflipped."""
        if resize is not None:
            raise ThmrError("MeshRenderer.__call__: resize is not supported")
        dev = self.device
        v = _cuda_f32(vertices, dev, "vertices", (self.renderer.num_verts, 3))[None]
        t = _cuda_f32(camera_translation, dev, "camera_translation", (3,))[None]
        img = _cuda_f32(image, dev, "image", (None, None, 3))
        H, W = img.shape[:2]
        base = tuple(float(c) for c in baseColorFactor[:3])
        if side_view:
            out = self._side(v, t, H, W, float(focal_length), base, float(rot_angle))[0, ..., :3]
        else:
            out = self._front(v, t, img.permute(2, 0, 1)[None].contiguous(), float(focal_length), base)[0]
        return out.cpu().numpy()

    # ---------------------------------------------------------------------------------------------- grids
    def visualize(self, vertices, camera_translation, images, focal_length=None, nrow=3, padding=2) -> torch.Tensor:
        """MeshRenderer.visualize (:57-68): per sample the crop, the front and the side view."""
        return self._grid(vertices, camera_translation, images, None, None, int(nrow), int(padding))

    def visualize_tensorboard(self, vertices, camera_translation, images, pred_keypoints, gt_keypoints,
                              focal_length=None, nrow=5, padding=2) -> torch.Tensor:
        """MeshRenderer.visualize_tensorboard (:70-107): vertices (B, V, 3), camera_translation (B, 3) (pred_cam_t),
        images (B, 3, H, W) crops in [0, 1], pred_keypoints (B, 44, 2) normalised or None, gt_keypoints (B, 44, 3) or
        None.  Returns the make_grid(nrow, padding) grid, (3, B (H + 2) + 2, 5 (W + 2) + 2) with both keypoint sets
        and the default nrow, padding."""
        nrow = int(nrow) - (gt_keypoints is None) - (pred_keypoints is None)
        return self._grid(vertices, camera_translation, images, pred_keypoints, gt_keypoints, nrow, int(padding))

    def _grid(self, vertices, camera_translation, images, pred_keypoints, gt_keypoints, nrow: int,
              padding: int) -> torch.Tensor:
        dev = self.device
        imgs = _cuda_f32(images, dev, "images", (None, 3, None, None))
        B, _, H, W = imgs.shape
        v = _cuda_f32(vertices, dev, "vertices", (B, self.renderer.num_verts, 3))
        t = _cuda_f32(camera_translation, dev, "camera_translation", (B, 3))
        kp = [None if k is None else _cuda_f32(k, dev, name, (B, _lib.POSE_KEYPOINTS, d))
              for k, name, d in ((pred_keypoints, "pred_keypoints", 2), (gt_keypoints, "gt_keypoints", 3))]
        n_sets = sum(k is not None for k in kp)
        gh, gw = ctypes.c_int(), ctypes.c_int()
        check(lib().thmr_pose_grid_size(B, W, H, n_sets, nrow, padding, ctypes.byref(gh), ctypes.byref(gw)))
        with torch.cuda.device(dev):
            base = (1.0, 1.0, 0.9)
            front = self._front(v, t, imgs, self.focal_length, base)
            # the double x flip of :118 (front view flips the row in place, the side view flips it back)
            t_side = t.clone()
            t_side[:, 0].neg_()
            side = self._side(v, t_side, H, W, self.focal_length, base)
            out = torch.empty(3, gh.value, gw.value, dtype=torch.float32, device=dev)
            ws = torch.empty(lib().thmr_pose_grid_workspace_bytes(B, W, H, n_sets), dtype=torch.uint8, device=dev)
            d = _lib.PoseGridDesc()
            d.n, d.width, d.height = B, W, H
            d.images, d.front, d.side = imgs.data_ptr(), front.data_ptr(), side.data_ptr()
            d.pred_keypoints = kp[0].data_ptr() if kp[0] is not None else None
            d.gt_keypoints = kp[1].data_ptr() if kp[1] is not None else None
            d.img_res = float(self.img_res)
            d.nrow, d.padding = nrow, padding
            d.out, d.out_stride_c, d.out_stride_y = out.data_ptr(), out.stride(0), out.stride(1)
            check(lib().thmr_pose_grid(ctypes.byref(d), ws.data_ptr(), torch.cuda.current_stream().cuda_stream))
        return out

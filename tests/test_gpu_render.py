"""The CUDA rasterizer (csrc/render.cuh, thmr_render_meshes) against the float64 oracle (oracle/render_oracle.py) on
the same fp32 inputs, on a closed synthetic mesh of SMPL's size (tests/render_mesh.py).

Geometry: face id and alpha must be equal on every pixel except those the oracle marks ambiguous -- a candidate face
whose edge value lies within the bound the kernel's fp32 vertex stage allows (render_oracle.vertex_error_bounds, then
the first-order edge-function perturbation), or a winning depth within the two faces' depth bounds of the runner-up.
Each case reports how many pixels it excluded and fails if that is more than 1 % of the covered pixels.  Depth must lie
within its bound; the quantised colour within one level of the oracle's (each case prints the worst error against the
oracle's value before quantisation); the composite exactly equal to the kernel's own colour and alpha over the image.
Scenes whose fp32 vertex stage is exact (test_fill_rule_exact_on_pixel_centres) are compared without any exclusion, and
a close, steeply tilted surface (test_close_tilted_surface_vs_oracle) makes perspective correction visible."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import render_oracle as RO
from render_mesh import ellipsoid, posed, synthetic_body
from tokenhmr_b200 import _lib
from tokenhmr_b200 import render as R

pytestmark = pytest.mark.gpu
MEAN = np.array([0.485, 0.456, 0.406], np.float32)
STD = np.array([0.229, 0.224, 0.225], np.float32)
BASE = (0.65, 0.74, 0.86)
MAX_EXCLUDED = 0.01


@pytest.fixture(scope="module")
def mesh():
    return synthetic_body()


@pytest.fixture(scope="module")
def renderer(cuda_dev, mesh):
    return R.Renderer({"EXTRA": {"FOCAL_LENGTH": 5000.0}, "MODEL": {"IMAGE_SIZE": 256, "IMAGE_MEAN": MEAN.tolist(),
                                                                      "IMAGE_STD": STD.tolist()}}, mesh[1], cuda_dev)


def _crop_cams(B, seed):
    rng = np.random.default_rng(seed)
    tz = 2 * 5000.0 / (256 * rng.uniform(0.6, 1.0, B))
    return np.stack([rng.uniform(-0.15, 0.15, B), rng.uniform(-0.15, 0.15, B), tz], 1).astype(np.float32)


def _check(name, gpu, v, t, faces, Rm, rot_t, W, H, focal, lights, mesh_image=None, n_images=None, bg=None):
    """Compares one raster() result with the oracle; returns the oracle result."""
    R32 = np.asarray(Rm if Rm is not None else np.eye(3), np.float32).astype(np.float64)
    v64, t64 = v.astype(np.float64), t.astype(np.float64)
    q = RO.camera_q(v64, t64, R32, rot_t)
    scr = RO.project(q, float(np.float32(focal)), W, H)
    es, ez, eq = RO.vertex_error_bounds(v64, t64, R32, rot_t, float(np.float32(focal)), W, H)
    r = RO.raster(scr, q[..., 2], faces, W, H, mesh_image, n_images, es=es, ez=ez)
    fid = gpu["face_id"].cpu().numpy()
    alpha = gpu["rgba"][..., 3].cpu().numpy()
    amb = r["ambiguous"]
    covered = r["face_id"] >= 0
    excluded = int(amb.sum())
    frac = excluded / max(int(covered.sum()), 1)
    print(f"{name}: {int(covered.sum())} covered pixels, {excluded} excluded ({100 * frac:.4f} %)")
    assert frac <= MAX_EXCLUDED, f"{name}: {excluded} ambiguous pixels exceed {MAX_EXCLUDED:.0%} of the covered ones"
    ok = ~amb
    bad = (fid != r["face_id"]) & ok
    assert not bad.any(), f"{name}: face id differs on {int(bad.sum())} unambiguous pixels, first {np.argwhere(bad)[:5]}"
    assert np.array_equal(alpha[ok], covered[ok].astype(np.float32)), f"{name}: alpha differs"
    # depth
    depth = gpu["depth"].cpu().numpy().reshape(-1)
    pix = r["pix"]
    keep = ok.reshape(-1)[pix]
    dz = np.abs(depth[pix] - r["depth"].reshape(-1)[pix])[keep]
    dzb = r["depth_bound"].reshape(-1)[pix][keep]
    assert (dz <= dzb).all(), f"{name}: depth err/bound {np.max(dz / dzb):.3g}"
    assert (depth[~covered.reshape(-1) & ok.reshape(-1)] == 0).all()
    # shading: the quantised colour within one level of the oracle's quantised colour
    pre = RO.shade(r, q, faces, lights, BASE)
    rgb = gpu["rgba"][..., :3].cpu().numpy().reshape(-1, 3)[pix]
    lv = np.abs(np.rint(rgb * 255) - np.rint(pre * 255))[keep]
    assert lv.max(initial=0) <= 1, f"{name}: colour {lv.max():.0f} levels from the oracle"
    err = np.abs(rgb - pre)[keep] * 255
    print(f"{name}: worst depth err/bound {np.max(dz / dzb, initial=0):.3g}, worst colour error before quantisation "
          f"{np.max(err, initial=0):.3f} levels, {int((lv == 1).sum())} pixels one level apart")
    # background pixels: the quantised background colour with alpha 0
    bgpx = gpu["rgba"].cpu().numpy()[~covered & ok]
    assert (bgpx[:, 3] == 0).all()
    return r


def _composite_exact(gpu, imgs):
    rgba = gpu["rgba"]
    bg = (imgs.cuda() * torch.tensor(STD, device="cuda").view(1, 3, 1, 1)
          + torch.tensor(MEAN, device="cuda").view(1, 3, 1, 1)).permute(0, 2, 3, 1)
    a = rgba[..., 3:]
    want = rgba[..., :3] * a + (1 - a) * bg
    assert torch.equal(gpu["composite"], want)


@pytest.mark.parametrize("B", [1, 7, 64])
def test_crops_vs_oracle(renderer, mesh, B):
    v0, faces = mesh
    v = posed(v0, B, seed=B)
    t = _crop_cams(B, seed=B + 1)
    imgs = torch.randn(B, 3, 256, 256, generator=torch.Generator().manual_seed(B))
    lights = R.crop_lights()
    gpu = renderer.raster(torch.from_numpy(v), torch.from_numpy(t), 256, 256, 5000.0, lights=lights, base_color=BASE,
                          bg_color=(1, 1, 1), bg_image=imgs, bg_layout=_lib.BG_CHW_NORMALIZED,
                          outputs=("rgba", "composite", "face_id", "depth"))
    _check(f"crops B={B}", gpu, v, t, faces, None, False, 256, 256, 5000.0, lights)
    _composite_exact(gpu, imgs)


def test_side_view_vs_oracle(renderer, mesh):
    v0, faces = mesh
    v, t = posed(v0, 7, seed=11), _crop_cams(7, seed=12)
    Ry = R.rotation_matrix(np.radians(90), [0, 1, 0])
    lights = R.crop_lights()
    gpu = renderer.raster(torch.from_numpy(v), torch.from_numpy(t), 256, 256, 5000.0, rotation=Ry, lights=lights,
                          base_color=BASE, outputs=("rgba", "face_id", "depth"))
    _check("side view", gpu, v, t, faces, Ry, False, 256, 256, 5000.0, lights)
    out = renderer.render_crops(torch.from_numpy(v), torch.from_numpy(t), torch.zeros(7, 3, 256, 256),
                                side_view=True, mesh_base_color=BASE)
    assert torch.equal(out, gpu["rgba"][..., :3])


def test_degenerate_faces(cuda_dev, mesh):
    v0, faces = mesh
    f2 = faces.copy()
    f2[::97, 1] = f2[::97, 0]          # zero-area faces (a repeated vertex) all over the mesh
    f2[5::101, 2] = f2[5::101, 1]
    ren = R.Renderer({"EXTRA": {"FOCAL_LENGTH": 5000.0}}, f2, cuda_dev)
    v, t = posed(v0, 7, seed=21), _crop_cams(7, seed=22)
    lights = R.crop_lights()
    gpu = ren.raster(torch.from_numpy(v), torch.from_numpy(t), 256, 256, 5000.0, lights=lights, base_color=BASE,
                     outputs=("rgba", "face_id", "depth"))
    _check("degenerate faces", gpu, v, t, f2, None, False, 256, 256, 5000.0, lights)
    fid = gpu["face_id"].cpu().numpy()
    degenerate = np.nonzero((f2[:, 0] == f2[:, 1]) | (f2[:, 1] == f2[:, 2]))[0]
    assert not np.isin(fid % faces.shape[0], degenerate).any()


def _frame_people():
    """10 people in a 1920 x 1080 frame (focal 5000 / 256 * 1920): overlapping pairs, one partly off the left edge,
    one fully off-screen to the right, one behind the camera."""
    v0, _ = synthetic_body()
    v = posed(v0, 10, seed=31)
    f = 5000.0 / 256 * 1920
    z = [120., 150., 125., 200., 90., 300., 160., 140., 150., -60.]
    sx = [700., 760., 1100., 1150., 30., 1500., 400., 1300., 5000., 960.]
    sy = [540., 560., 500., 600., 540., 300., 700., 420., 540., 540.]
    t = np.array([[(x - 960.) * zz / f, (y - 540.) * zz / f, zz] for x, y, zz in zip(sx, sy, z)], np.float32)
    return v, t, f


def test_full_frame_ten_people_vs_oracle(renderer, mesh):
    _, faces = mesh
    v, t, f = _frame_people()
    lights = R.multiple_lights()
    gpu = renderer.raster(torch.from_numpy(v), torch.from_numpy(t), 1920, 1080, f, rotate_translation=True,
                          mesh_image=[0] * 10, n_images=1, lights=lights, base_color=BASE,
                          outputs=("rgba", "face_id", "depth"))
    r = _check("1080p, 10 people", gpu, v, t, faces, None, True, 1920, 1080, f, lights, mesh_image=np.zeros(10, int),
               n_images=1)
    fid = gpu["face_id"].cpu().numpy()
    meshes = set(np.unique(fid[fid >= 0] // faces.shape[0]).tolist())
    assert 8 not in meshes and 9 not in meshes       # off-screen and behind the camera: background only
    assert {0, 1, 4}.issubset(meshes)
    # the reference surface on the same scene
    rgba = renderer.render_rgba_multiple(list(v), list(t), render_res=[1920, 1080], focal_length=f,
                                         mesh_base_color=BASE)
    assert np.array_equal(rgba, gpu["rgba"][0].cpu().numpy())


def test_deterministic_and_graph_replay(renderer, mesh):
    v0, _ = mesh
    v = torch.from_numpy(posed(v0, 64, seed=41)).cuda()
    t = torch.from_numpy(_crop_cams(64, seed=42)).cuda()
    imgs = torch.randn(64, 3, 256, 256, device="cuda")
    kw = dict(lights=R.crop_lights(), base_color=BASE, bg_image=imgs, bg_layout=_lib.BG_CHW_NORMALIZED,
              outputs=("rgba", "composite", "face_id", "depth"))
    a = renderer.raster(v, t, 256, 256, 5000.0, **kw)
    b = renderer.raster(v, t, 256, 256, 5000.0, **kw)
    out = {k: torch.empty_like(x) for k, x in a.items()}
    kw["workspace"] = torch.empty(renderer.workspace_bytes(64, 64, 256, 256), dtype=torch.uint8, device="cuda")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        renderer.raster(v, t, 256, 256, 5000.0, out=out, **kw)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    for x in out.values():
        x.zero_()
    with torch.cuda.graph(g):
        renderer.raster(v, t, 256, 256, 5000.0, out=out, **kw)
    for x in out.values():
        x.zero_()
    renderer.raster(v[:1], t[:1], 1024, 1024, 5000.0)     # a larger eager call replaces the Renderer's own workspace
    g.replay()
    torch.cuda.synchronize()
    for k in a:
        assert torch.equal(a[k], b[k]), k
        assert torch.equal(a[k], out[k]), k


def test_render_crops_on_engine_outputs_equals_per_person_call(cuda_dev, mesh):
    from tokenhmr_b200 import synth
    from tokenhmr_b200.config import tiny_config
    from tokenhmr_b200.engine import TokenHMREngine
    _, faces = mesh
    cfg = tiny_config(vit_depth=2, num_verts=6890)
    model = TokenHMREngine(cfg, synth.make_state_dict(cfg), synth.make_smpl(cfg), device=cuda_dev,
                           use_cuda_graph=False)
    img = synth.make_images(5, cfg)
    out = model({"img": img})
    ren = R.Renderer(cfg, faces, cuda_dev)
    crops = ren.render_crops(out["pred_vertices"], out["pred_cam_t"], img.cuda(), mesh_base_color=BASE,
                             scene_bg_color=(1, 1, 1))
    side = ren.render_crops(out["pred_vertices"], out["pred_cam_t"], img.cuda(), side_view=True, mesh_base_color=BASE)
    for n in range(5):
        cam = out["pred_cam_t"][n].cpu().numpy()
        one = ren(out["pred_vertices"][n].cpu().numpy(), cam, img[n], mesh_base_color=BASE, scene_bg_color=(1, 1, 1))
        assert np.array_equal(one, crops[n].cpu().numpy())
        assert np.array_equal(cam, out["pred_cam_t"][n].cpu().numpy())       # the caller's array is not modified
        one_side = ren(out["pred_vertices"][n].cpu().numpy(), cam, img[n], side_view=True, mesh_base_color=BASE)
        assert np.array_equal(one_side, side[n].cpu().numpy())
        assert one.dtype == np.float32 and one.shape == (256, 256, 3)


def test_rejects_bad_descs(renderer, mesh):
    L = _lib.lib()
    v = torch.zeros(2, 6890, 3, device="cuda")
    t = torch.zeros(2, 3, device="cuda")
    ws = torch.empty(L.thmr_render_workspace_bytes(renderer._topo.value, 2, 2, 64, 64), dtype=torch.uint8,
                     device="cuda")
    out = torch.empty(2, 64, 64, 3, device="cuda")

    def desc(**kw):
        d = _lib.RenderDesc()
        d.topology, d.n_meshes, d.n_images = renderer._topo.value, 2, 2
        d.vertices, d.translations = v.data_ptr(), t.data_ptr()
        d.rotation[:] = [1, 0, 0, 0, 1, 0, 0, 0, 1]
        d.width = d.height = 64
        d.focal, d.znear = 100.0, 0.05
        for k, val in kw.items():
            setattr(d, k, val)
        return d

    def status(d):
        return L.thmr_render_meshes(ctypes.byref(d), ws.data_ptr(), None)

    assert status(desc()) == 0
    bad_img = (ctypes.c_int32 * 2)(0, 2)
    neg_img = (ctypes.c_int32 * 2)(-1, 0)
    cases = {"no topology": desc(topology=None), "no vertices": desc(vertices=None), "n_meshes 0": desc(n_meshes=0),
             "too many meshes": desc(n_meshes=_lib.RENDER_MAX_MESHES + 1), "n_images 0": desc(n_images=0),
             "width 0": desc(width=0), "height -3": desc(height=-3), "focal 0": desc(focal=0.0),
             "image index 2 of 2": desc(mesh_image_host=ctypes.cast(bad_img, ctypes.POINTER(ctypes.c_int32))),
             "image index -1": desc(mesh_image_host=ctypes.cast(neg_img, ctypes.POINTER(ctypes.c_int32))),
             "17 lights": desc(n_lights=17), "composite without image": desc(composite=out.data_ptr()),
             "bg layout 7": desc(bg_layout=7, bg_image=out.data_ptr()),
             "rgba not 16-byte aligned": desc(rgba=out.data_ptr() + 4)}
    bad_light = desc(n_lights=1)
    bad_light.lights[0].type = 5
    cases["light type 5"] = bad_light
    for name, d in cases.items():
        assert status(d) == -1, name
    assert L.thmr_render_meshes(ctypes.byref(desc()), None, None) == -1
    torch.cuda.synchronize()
    _lib.check(L.thmr_check_device_flags())



def test_fill_rule_exact_on_pixel_centres(cuda_dev):
    """Focal 4 and z = 4 make the fp32 vertex stage exact (x / 4 and 4 * (x / 4) + 8 are exact for these x), and
    every vertex sits on a pixel centre: a 2 x 2 grid of squares over pixel centres, split by diagonals in both
    directions, wound both ways, with shared vertical, horizontal and diagonal edges through pixel centres.  Face id
    must equal the exact oracle on every pixel, with no exclusion: each centre on a shared edge has exactly one owner,
    the square's top and left borders are in and its bottom and right borders out."""
    xs = np.array([2.5, 7.5, 12.5]) - 8.0
    verts = np.array([[x, y, 0.0] for y in xs for x in xs], np.float32)
    faces = []
    for r in range(2):
        for c in range(2):
            a, b, d, e = 3 * r + c, 3 * r + c + 1, 3 * (r + 1) + c, 3 * (r + 1) + c + 1
            tris = [(a, b, e), (a, e, d)] if (r + c) % 2 == 0 else [(a, b, d), (b, e, d)]
            faces += [tris[0], tris[1][::-1]]                 # one of each pair wound the other way
    faces = np.array(faces, np.int32)
    ren = R.Renderer({"EXTRA": {"FOCAL_LENGTH": 4.0}}, faces, cuda_dev)
    t = np.array([[0, 0, 4.0]], np.float32)
    gpu = ren.raster(torch.from_numpy(verts[None]), torch.from_numpy(t), 16, 16, 4.0, outputs=("rgba", "face_id"))
    q = RO.camera_q(verts[None].astype(float), t.astype(float))
    scr = RO.project(q, 4.0, 16, 16)
    assert set(np.unique(scr % 1.0)) == {0.5}
    r = RO.raster(scr, q[..., 2], faces, 16, 16)
    fid = gpu["face_id"][0].cpu().numpy()
    assert np.array_equal(fid, r["face_id"][0])
    want = np.zeros((16, 16), bool)
    want[2:12, 2:12] = True                                   # centres 2.5 .. 11.5 in both directions
    assert np.array_equal(fid >= 0, want)
    assert np.array_equal(gpu["rgba"][0, ..., 3].cpu().numpy(), want.astype(np.float32))
    # every face owns some of the centres on its shared edges: the owner is decided by the fill rule alone
    on_edge = want & ((np.arange(16)[None, :] == 7) | (np.arange(16)[:, None] == 7))
    assert len(np.unique(fid[on_edge])) >= 4


def test_close_tilted_surface_vs_oracle(cuda_dev):
    """A coarse ellipsoid (320 large faces) tilted 40 degrees and spanning z = 1.6 .. 4.8 m in front of the camera:
    here perspective-correct and screen-space interpolation differ by many colour levels and depth far beyond its
    bound, so the comparison with the oracle fails for a kernel without perspective correction."""
    v0, faces = ellipsoid((0.8, 0.8, 2.0))
    Ry = RO.rot_axis(np.radians(40), [0, 1, 0])
    v = (v0.astype(float) @ Ry.T)[None].astype(np.float32)
    t = np.array([[0.1, -0.05, 3.2]], np.float32)
    d = np.array([0.5, -0.4, -1.0]) / np.linalg.norm([0.5, -0.4, -1.0])
    lights = [(_lib.LIGHT_DIRECTIONAL, d, 0.6), (_lib.LIGHT_POINT, [1.0, -1.0, 0.5], 1.5)]   # unsaturated: 0.2 .. 0.9
    ren = R.Renderer({"EXTRA": {"FOCAL_LENGTH": 128.0}}, faces, cuda_dev)
    gpu = ren.raster(torch.from_numpy(v), torch.from_numpy(t), 256, 256, 128.0, lights=lights, base_color=BASE,
                     outputs=("rgba", "face_id", "depth"))
    r = _check("close tilted surface", gpu, v, t, faces, None, False, 256, 256, 128.0, lights)
    # the scene tells the two interpolations apart
    q = RO.camera_q(v.astype(float), t.astype(float))
    flat = RO.shade(r, q, faces, lights, BASE, perspective=False)
    persp = RO.shade(r, q, faces, lights, BASE)
    assert np.abs(np.rint(flat * 255) - np.rint(persp * 255)).max() >= 3
    F = faces.shape[0]
    zv = np.stack([q[0, faces[r["fid"] % F, k], 2] for k in range(3)])
    z_linear = (r["w"] * zv).sum(0)
    assert (np.abs(z_linear - r["depth"].reshape(-1)[r["pix"]]) > 10 * r["depth_bound"].reshape(-1)[r["pix"]]).mean() > 0.5


def test_full_frame_call_composites_over_the_image_file(renderer, mesh, tmp_path):
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(5)
    frame = rng.integers(0, 256, (96, 128, 3), dtype=np.uint8)
    path = str(tmp_path / "frame.png")
    assert cv2.imwrite(path, frame)
    v = posed(mesh[0], 1, seed=51)[0]
    cam = np.array([0.05, 0.02, 160.0], np.float32)
    out = renderer(v, cam.copy(), None, full_frame=True, imgname=path, mesh_base_color=BASE, scene_bg_color=(1, 1, 1))
    bg = torch.from_numpy(np.ascontiguousarray(cv2.imread(path).astype(np.float32)[:, :, ::-1] / 255.))[None]
    want = renderer.raster(torch.from_numpy(v[None]), torch.from_numpy(cam[None]), 128, 96, 5000.0,
                           lights=R.crop_lights(), base_color=BASE, bg_color=(1, 1, 1), bg_image=bg,
                           bg_layout=_lib.BG_HWC, outputs=("rgba", "composite"))
    assert out.shape == (96, 128, 3) and out.dtype == np.float32
    assert np.array_equal(out, want["composite"][0].cpu().numpy())
    alpha = want["rgba"][0, ..., 3].cpu().numpy()
    assert 0 < alpha.sum() < alpha.size                       # the person is in the frame, and so is the image
    assert np.array_equal(out[alpha == 0], bg[0].numpy()[alpha == 0])

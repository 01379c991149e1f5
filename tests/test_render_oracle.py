"""The renderer's float64 oracle (oracle/render_oracle.py): known answers for the rasterizer, the reference's camera
chain reduced to perspective_projection, and the light rig pinned to the reference's own renderer.py."""
import numpy as np
import pytest

from oracle import render_oracle as RO
from render_mesh import synthetic_body
from tokenhmr_b200 import render as R

GOLD = "render_reference.npz"


def _raster1(scr, faces, W, H, z=None):
    scr = np.asarray(scr, float)[None]
    z = np.full(scr.shape[:2], 10.0) if z is None else np.asarray(z, float)[None]
    return RO.raster(scr, z, np.asarray(faces), W, H)


def test_single_triangle_covers_hand_counted_pixels():
    # (1,1) (5,1) (1,5): the centres (c + .5, r + .5) with c, r >= 1 and c + r + 1 <= 6 minus those on the
    # hypotenuse x + y = 6 (a bottom-right edge): c + r <= 4
    r = _raster1([[1, 1], [5, 1], [1, 5]], [[0, 1, 2]], 8, 8)
    got = {(int(c), int(rr)) for rr, c in zip(*np.nonzero(r["face_id"][0] == 0))}
    want = {(c, rr) for c in range(8) for rr in range(8) if c >= 1 and rr >= 1 and c + rr <= 4}
    assert got == want and len(want) == 6
    # the same triangle wound the other way covers the same pixels (no back-face culling)
    r2 = _raster1([[1, 1], [1, 5], [5, 1]], [[0, 1, 2]], 8, 8)
    assert np.array_equal(r2["face_id"] == 0, r["face_id"] == 0)


def test_pixel_centre_on_shared_edge_belongs_to_exactly_one_triangle():
    # a square split along its diagonal and along a vertical line through pixel centres (x = 2.5)
    pts = [[0.5, 0.5], [2.5, 0.5], [2.5, 6.5], [0.5, 6.5], [4.5, 0.5], [4.5, 6.5]]
    faces = [[0, 1, 2], [0, 2, 3], [1, 4, 5], [1, 5, 2]]
    cover = np.zeros((8, 8), int)
    for f in range(4):
        r = _raster1(pts, [faces[f]], 8, 8)
        cover += r["face_id"][0] == 0
    r = _raster1(pts, faces, 8, 8)
    inside = np.zeros((8, 8), bool)
    inside[0:7, 0:5] = True          # centres with 0.5 <= x <= 4.5, 0.5 <= y <= 6.5 lie in the closed square
    # every centre strictly inside the union, including those on the shared edges x = 2.5 and the diagonals, is
    # covered exactly once; the fill rule leaves the square's bottom and right borders out
    interior = np.zeros((8, 8), bool)
    interior[0:6, 0:4] = True
    assert cover[interior].min() == 1 and cover[interior].max() == 1
    assert (cover <= 1).all()
    assert ((r["face_id"][0] >= 0) == (cover == 1)).all()
    assert (cover[~inside] == 0).all()


def test_cube_silhouette_and_depth():
    # axis-aligned unit cube centred at (0, 0, 10) seen head on with f = 100 on 64 x 64: front face z = 9.5
    c = np.array([[x, y, z] for x in (-.5, .5) for y in (-.5, .5) for z in (-.5, .5)])
    quads = [(0, 1, 3, 2), (4, 6, 7, 5), (0, 4, 5, 1), (2, 3, 7, 6), (0, 2, 6, 4), (1, 5, 7, 3)]
    faces = np.array([t for a, b, cc, d in quads for t in ((a, b, cc), (a, cc, d))])
    q = RO.camera_q(c, np.array([0, 0, 10.0]))
    scr = RO.project(q, 100.0, 64, 64)
    r = RO.raster(scr[None], q[None, :, 2], faces, 64, 64)
    # front face spans 32 +- 50/9.5 = [26.737, 37.263]: centres 27.5 .. 36.5 -> columns 27..36
    covered = r["face_id"][0] >= 0
    rows, cols = np.nonzero(covered)
    assert (rows.min(), rows.max(), cols.min(), cols.max()) == (27, 36, 27, 36)
    assert covered.sum() == 100
    assert np.allclose(r["depth"][0][covered], 9.5, rtol=0, atol=1e-12)
    assert set(np.unique(r["face_id"][0][covered] // 2)) == {4}      # the z = -0.5 quad (0, 2, 6, 4) only


def test_side_view_matches_hand_rotated_mesh():
    v, f = synthetic_body()
    t = np.array([0.05, 0.1, 30.0])
    Ry = np.array([[0, 0, 1.0], [0, 1, 0], [-1.0, 0, 0]])            # 90 degrees about y, written out
    assert np.allclose(RO.rot_axis(np.radians(90), [0, 1, 0]), Ry, atol=1e-15)
    assert np.allclose(R.rotation_matrix(np.radians(90), [0, 1, 0]), Ry, atol=1e-15)
    col, row, depth = RO.crop_chain(v, t, 5000., 256, 256, side_view=True, rot_angle=90)
    vr = v.astype(float) @ Ry.T
    col2, row2, depth2 = RO.crop_chain(vr, t, 5000., 256, 256)
    assert np.allclose(col, col2, atol=1e-9) and np.allclose(row, row2, atol=1e-9) and np.allclose(depth, depth2)
    s = RO.project(RO.camera_q(v, t, Ry), 5000., 256, 256)
    assert np.allclose(np.stack([col, row], -1), s, atol=1e-9)


def test_rotation_known_answers():
    assert np.allclose(RO.rot_axis(np.pi, [1, 0, 0]), np.diag([1, -1, -1]), atol=1e-15)
    c, s = np.cos(0.3), np.sin(0.3)
    assert np.allclose(RO.rot_axis(0.3, [0, 0, 2]), [[c, -s, 0], [s, c, 0], [0, 0, 1]], atol=1e-15)
    for ang, ax in ((0.7, [1, 2, 3]), (-2.0, [0, 1, 0]), (0.0, [1, 0, 0])):
        assert np.allclose(R.rotation_matrix(ang, ax), RO.rot_axis(ang, ax), atol=1e-15)


@pytest.mark.parametrize("side", [False, True])
def test_crop_chain_is_perspective_projection_of_v_plus_t(golden_dir, side):
    """Renderer.__call__'s chain == perspective_projection(v + t, focal, (W/2, H/2)), evaluated by the live reference
    function in the stored golden (same formula, fresh points)."""
    g = np.load(golden_dir / GOLD)
    for b in range(2):
        v, t, f, c = g["pts"][b].astype(float), g["trans"][b].astype(float), float(g["focal"][b, 0]), g["center"][b]
        W, H = int(2 * c[0]), int(2 * c[1])
        col, row, depth = RO.crop_chain(v, t, f, W, H, side_view=side, rot_angle=90)
        Rm = RO.rot_axis(np.radians(90), [0, 1, 0]) if side else np.eye(3)
        q = RO.camera_q(v, t, Rm)
        assert np.allclose(np.stack([col, row], -1), RO.project(q, f, W, H), rtol=0, atol=1e-8)
        assert np.allclose(depth, q[:, 2], rtol=1e-12)
        if not side:   # the live reference's perspective_projection of the same points (fp32)
            assert np.allclose(RO.project(q, f, W, H), g["proj"][b], rtol=0, atol=2e-3)


def test_multiple_chain_is_perspective_projection(golden_dir):
    g = np.load(golden_dir / GOLD)
    v, t = g["pts"][1].astype(float), g["trans"][1].astype(float)
    col, row, depth = RO.multiple_chain(v, t, 1200., 1920, 1080)
    assert np.allclose(np.stack([col, row], -1), g["proj"][1], atol=2e-3)
    for axis, ang in (([1, 0, 0], 20.0), ([0, 1, 1], -35.0)):
        col, row, depth = RO.multiple_chain(v, t, 1200., 1920, 1080, axis=axis, angle=ang)
        q = RO.camera_q(v, t, RO.rot_axis(np.radians(ang), axis), rotate_translation=True)
        assert np.allclose(np.stack([col, row], -1), RO.project(q, 1200., 1920, 1080), atol=1e-8)
        assert np.allclose(depth, q[:, 2])


def test_live_reference_projection_when_available():
    from oracle import ref_import
    if not ref_import.available():
        pytest.skip("reference checkout not configured (TOKENHMR_REFERENCE)")
    import torch
    ns = ref_import.load_modules()
    v, _ = synthetic_body()
    t = np.array([0.2, -0.1, 25.0])
    pp = ns.geometry.perspective_projection(torch.tensor(v[None] + t, dtype=torch.float64),
                                            torch.zeros(1, 3, dtype=torch.float64),
                                            torch.full((1, 2), 5000.0, dtype=torch.float64),
                                            camera_center=torch.full((1, 2), 128.0, dtype=torch.float64))[0].numpy()
    col, row, _ = RO.crop_chain(v, t, 5000., 256, 256)
    assert np.allclose(np.stack([col, row], -1), pp, atol=1e-8)


def _check_lights(rec):
    # the oracle's reading of the rig == the product's restatement
    ray = rec["raymond"][:, :3, 2]
    assert np.allclose(ray, R.raymond_directions(), atol=1e-12)
    cols12 = R.light_pose_columns(12.0)
    cols05 = R.light_pose_columns(0.5)
    assert np.allclose(rec["directional"][:, :3, 2], cols12[:, 0], atol=1e-6)
    assert np.allclose(rec["point"][:, :3, 3], cols05[:, 1], atol=1e-6)
    lights = R.multiple_lights()
    kinds = [k for k, _, _ in lights]
    assert kinds.count(1) == 6 and kinds.count(0) == 9 and len(R.crop_lights()) == 3
    assert np.allclose([v for k, v, _ in lights if k == 1], RO.camera_q(rec["point"][:, :3, 3], np.zeros(3),
                                                                          np.diag([1, -1, -1])), atol=1e-6)


def test_light_rig_matches_recorded_reference(golden_dir):
    _check_lights(np.load(golden_dir / GOLD))


def test_light_rig_matches_live_reference_when_available():
    from oracle import ref_import
    if not ref_import.available():
        pytest.skip("reference checkout not configured (TOKENHMR_REFERENCE)")
    _check_lights(RO.lights_from_reference())


def test_synthetic_body_is_closed_and_outward():
    v, f = synthetic_body()
    e = np.sort(np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]]), 1)
    _, cnt = np.unique(e, axis=0, return_counts=True)
    assert (cnt == 2).all()                      # every edge shared by exactly two faces: closed
    n, _ = RO.vertex_normals(v.astype(float), f)
    assert (np.einsum("ij,ij->i", n, v - v.mean(0)) > 0).mean() > 0.95


def test_shading_known_answer():
    # a camera-facing quad lit by one directional light along the view axis: ambient + 1 -> clamp to 1
    q = np.array([[-1, -1, 5.0], [1, -1, 5.0], [1, 1, 5.0], [-1, 1, 5.0]])
    faces = np.array([[0, 2, 1], [0, 3, 2]])     # normal -z (towards the camera)
    scr = RO.project(q, 10.0, 16, 16)
    r = RO.raster(scr[None], q[None, :, 2], faces, 16, 16)
    col = RO.shade(r, q[None], faces, [(0, [0, 0, -1.0], 0.5)], (1.0, 0.5, 0.2), ambient=0.3)
    assert np.allclose(col, np.array([0.8, 0.4, 0.16])[None], atol=1e-12)
    assert np.allclose(RO.quantise(col)[0], np.rint(np.array([0.8, 0.4, 0.16]) * 255) / 255)


def test_topology_rejects_out_of_range_faces(built_lib):
    """Face indices are checked once per topology, before anything touches the GPU."""
    import ctypes
    h = ctypes.c_void_p()
    for bad in ([[0, 1, 3]], [[0, -1, 2]]):
        f = np.ascontiguousarray(bad, dtype=np.int32)
        assert built_lib.thmr_render_topology_create(f.ctypes.data, 1, 3, ctypes.byref(h)) == -1
        assert b"outside [0, 3)" in built_lib.thmr_last_error()
    assert built_lib.thmr_render_topology_create(None, 1, 3, ctypes.byref(h)) == -1
    assert built_lib.thmr_render_workspace_bytes(None, 1, 1, 8, 8) == 0
    assert built_lib.thmr_abi_version() == 7

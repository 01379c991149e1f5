"""The prediction grid's oracle (oracle/openpose_oracle.py) and the overlay's span generator (csrc/keypoints.cuh, run on
the host through tests/libthmr_probe.so) against live OpenCV, and the grid golden (written from the live
mesh_renderer.py, render_openpose.py, cv2 and make_grid) against the oracle.  No GPU."""
import hashlib

import numpy as np
import pytest

import probe
from oracle import openpose_oracle as O

GOLD = "mesh_renderer_reference.npz"


def _random_primitives(n, seed):
    """(kind, p0, p1, W, H): kind 0 = cv2.line thickness 2, 1 / 2 = cv2.circle radius 1 of that thickness.  Endpoints
    range from inside the image to far outside it (up to 2^30 px), so clipping is exercised at every scale."""
    rng = np.random.default_rng(seed)
    for _ in range(n):
        W, H = int(rng.integers(1, 120)), int(rng.integers(1, 120))
        scale = [2, 60, 3000, 2 ** 20, 2 ** 30][rng.integers(0, 5)]
        pts = [(int(rng.integers(-scale, W + scale)), int(rng.integers(-scale, H + scale))) for _ in range(2)]
        yield int(rng.integers(0, 3)), pts[0], pts[1], W, H


def _cv2_mask(cv2, kind, p0, p1, W, H):
    m = np.zeros((H, W), np.uint8)
    if kind == 0:
        cv2.line(m, p0, p1, 1, 2, cv2.LINE_8, 0)
    else:
        cv2.circle(m, p0, 1, 1, kind, cv2.LINE_8, 0)
    return m


def test_primitive_restatement_matches_live_cv2():
    cv2 = pytest.importorskip("cv2")
    bad = []
    for k, (kind, p0, p1, W, H) in enumerate(_random_primitives(10000, seed=1)):
        m = np.zeros((H, W, 1), np.uint8)
        if kind == 0:
            O.cv_line(O.paint(m, 1), W, H, p0, p1)
        else:
            O.cv_circle(O.paint(m, 1), W, H, p0, kind)
        if not np.array_equal(m[..., 0], _cv2_mask(cv2, kind, p0, p1, W, H)):
            bad.append((kind, p0, p1, W, H))
    assert not bad, f"{len(bad)} of 10000 primitives differ from cv2, first {bad[:3]}"


def test_span_generator_matches_live_cv2(built_lib):
    """The __host__ __device__ span generator the raster kernel runs, on the host."""
    cv2 = pytest.importorskip("cv2")
    bad = []
    cases = list(_random_primitives(20000, seed=2))
    # the extremes of int32 and primitives hugging every border
    cases += [(0, (-2 ** 31, -2 ** 31), (2 ** 31 - 1, 2 ** 31 - 1), 50, 40), (0, (2 ** 31 - 1, 5), (-2 ** 31, 7), 50, 40),
              (1, (-1, -1), (0, 0), 5, 5), (2, (5, 5), (0, 0), 5, 5), (2, (-2, 2), (0, 0), 5, 5),
              (0, (0, 0), (0, 0), 1, 1), (0, (-2, 3), (-2, 300), 4, 9), (0, (3, 3), (4, 3), 8, 8)]
    for kind, p0, p1, W, H in cases:
        m = np.zeros((H, W), np.uint8)
        assert probe.lib().probe_pose_draw(kind, p0[0], p0[1], p1[0], p1[1], W, H, m.ctypes.data) == 0
        if not np.array_equal(m, _cv2_mask(cv2, kind, p0, p1, W, H)):
            bad.append((kind, p0, p1, W, H))
    assert not bad, f"{len(bad)} of {len(cases)} primitives differ from cv2, first {bad[:3]}"


# ---------------------------------------------------------------------------------------------- the overlay
def _overlay_cases():
    rng = np.random.default_rng(5)
    f01 = np.float32(0.1)
    for k in range(40):
        kp = np.concatenate([rng.uniform(-20, 84, (25, 2)), rng.choice(np.array([0, f01, 0.3, 1], np.float32),
                                                                        (25, 1))], 1).astype(np.float32)
        yield f"random{k}", kp
    kp = np.zeros((25, 3), np.float32)
    kp[:, :2] = rng.uniform(-1e4, 1e4, (25, 2))
    kp[:, 2] = 1
    yield "far off the image", kp
    kp = np.zeros((25, 3), np.float32)
    kp[:, 0] = np.float32([-1, 0, 63, 64, -0.5, 63.9] * 4 + [0])
    kp[:, 1] = np.float32([0, -1, 64, 63, 63.5, -0.9] * 4 + [10])
    kp[:, 2] = 1
    yield "negative and on the border", kp
    kp[:, 2] = f01
    kp[::3, 2] = 0.2
    yield "confidence exactly float32(0.1)", kp
    kp = np.zeros((25, 3), np.float32)
    kp[:, 0] = 30 + rng.uniform(0, 0.1, 25)
    kp[:, 1] = 20 + rng.uniform(0, 0.1, 25)
    kp[:, 2] = 1
    yield "coincident keypoints: circle thickness 1", kp
    kp = np.zeros((25, 3), np.float32)
    kp[:, :2] = rng.uniform(0, 64, (25, 2))
    kp[1, :2] = [10.2, 10.9]
    kp[8, :2] = [10.8, 10.1]
    kp[:, 2] = 1
    yield "a limb whose endpoints truncate to one pixel", kp


def test_coincident_keypoints_take_circle_thickness_1():
    _, kp = [c for c in _overlay_cases() if c[0].startswith("coincident")][0]
    assert O.overlay_params(kp, 64) == (True, 1)
    kp2 = kp.copy()
    kp2[0, 0] += 4                       # pw / W = 4 / 64 > 0.05
    assert O.overlay_params(kp2, 64) == (True, 2)
    kp3 = kp.copy()
    kp3[:, 1] = 20                       # zero area: nothing is drawn
    assert O.overlay_params(kp3, 64)[0] is False


def test_overlay_restatement_matches_live_render_openpose():
    pytest.importorskip("cv2")
    from oracle import ref_import
    if not ref_import.available():
        pytest.skip("reference checkout not configured (TOKENHMR_REFERENCE)")
    live = O.live_render_openpose()
    rng = np.random.default_rng(6)
    for name, kp in _overlay_cases():
        img = (255 * rng.random((64, 64, 3), dtype=np.float32)).astype(np.float32)
        want = live(img.copy(), kp.copy())
        got = O.render_openpose(img, kp)
        assert got.dtype == want.dtype and np.array_equal(got, want), name


# ---------------------------------------------------------------------------------------------- the grid golden
@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(golden_dir / GOLD)


def _inputs(g, B, seed):
    verts, faces, cam_t, images, pred, gt = O.golden_inputs(B, seed)
    assert hashlib.sha256(images.tobytes()).digest() == g[f"images_sha_b{B}"].tobytes(), "crop generator drifted"
    assert np.array_equal(cam_t, g[f"cam_t_b{B}"]) and np.array_equal(pred, g[f"pred_b{B}"])
    assert np.array_equal(gt, g[f"gt_b{B}"])
    return verts, faces, cam_t, images, pred, gt


def _variants(B):
    return O.GOLDEN_VARIANTS if B == 8 else {"both": O.GOLDEN_VARIANTS["both"]}


@pytest.mark.parametrize("B,seed", O.GOLDEN_CASES)
def test_golden_skeletons_match_restatement(golden, B, seed):
    _, _, _, images, pred, gt = _inputs(golden, B, seed)
    H, W = images.shape[2:]
    for name, (use_p, use_g) in _variants(B).items():
        key = f"b{B}_{name}"
        tiles = 3 + use_p + use_g
        # make_grid's layout: nrow drops by one per missing keypoint set, one sample per grid row
        assert tuple(golden[f"shape_{key}"]) == (3, B * (H + 2) + 2, tiles * (W + 2) + 2)
        sets = [O.prepare_keypoints(pred, 256, gt=False)] * use_p + [O.prepare_keypoints(gt, 256, gt=True)] * use_g
        for s, body in enumerate(sets):
            for b in range(B):
                want = O.decode_skeleton(golden[f"codes_{key}"][b, s], images[b])
                assert np.array_equal(O.skeleton_tile(images[b], body[b]), want), (key, s, b)


def test_golden_records_the_double_flip_and_the_config_focal(golden):
    """The front view of sample i sees camera x = -t_x (the flip of :118), the side view +t_x (flipped back); the
    focal length is cfg.EXTRA.FOCAL_LENGTH whatever visualize_tensorboard's focal_length argument says."""
    for B, _ in O.GOLDEN_CASES:
        t = golden[f"cam_t_b{B}"].astype(np.float64)
        for name in _variants(B):
            cx = golden[f"cam_x_b{B}_{name}"]
            assert np.array_equal(cx[0::2], -t[:, 0]) and np.array_equal(cx[1::2], t[:, 0])
            assert (golden[f"focal_b{B}_{name}"] == 5000.0).all()


def test_prepare_keypoints_rules():
    rng = np.random.default_rng(9)
    pred = rng.uniform(-0.5, 0.5, (2, 44, 2)).astype(np.float32)
    body = O.prepare_keypoints(pred, 256, gt=False)
    assert (body[..., 2] == np.float32(384)).all()            # 256 * (1 + 0.5): always drawn
    for i, j in O.KEYPOINT_MATCHES:                           # unconditional for predictions
        assert np.array_equal(body[:, i, :2], np.float32(256) * (pred[:, 25 + j] + np.float32(0.5)))
    gt = np.concatenate([pred, np.zeros((2, 44, 1), np.float32)], -1)
    gt[:, 25 + 12, 2] = 1           # extra joint 12 visible, body joint 1 invisible: substituted
    gt[:, 25 + 8, 2] = 1
    gt[:, 2, 2] = 0.5               # body joint 2 visible: kept
    before = gt.copy()
    b = O.prepare_keypoints(gt, 256, gt=True)
    assert np.array_equal(gt, before)                         # the caller's array is left alone
    assert np.array_equal(b[:, 1, :2], np.float32(256) * (pred[:, 25 + 12] + np.float32(0.5)))
    assert (b[:, 1, 2] == 1).all() and (b[:, 2, 2] == np.float32(0.5)).all()
    assert np.array_equal(b[:, 2, :2], np.float32(256) * (pred[:, 2] + np.float32(0.5)))


@pytest.mark.parametrize("mutation", ["joints_first", "round", "ge", "background_x"])
def test_golden_tells_mutations_apart(golden, mutation):
    """Each deliberately wrong overlay differs from the golden somewhere (the GPU test uses the same golden)."""
    B, seed = 8, 12
    _, _, _, images, pred, gt = _inputs(golden, B, seed)
    sets = (O.prepare_keypoints(pred, 256, gt=False), O.prepare_keypoints(gt, 256, gt=True))
    for s, body in enumerate(sets):
        for b in range(B):
            want = O.decode_skeleton(golden[f"codes_b{B}_both"][b, s], images[b])
            if not np.array_equal(O.skeleton_tile(images[b], body[b], mutation), want):
                return
    pytest.fail(f"the golden does not tell '{mutation}' apart")


def test_grid_matches_live_visualize_tensorboard():
    """The oracle's whole grid, mesh tiles from the stand-in renderer included, against the live reference."""
    pytest.importorskip("cv2")
    pytest.importorskip("torchvision")
    from oracle import ref_import
    if not ref_import.available():
        pytest.skip("reference checkout not configured (TOKENHMR_REFERENCE)")
    B = 3
    verts, faces, cam_t, images, pred, gt = O.golden_inputs(B, 21, H=64, W=48)
    image_of = O.oracle_mesh_image(faces)
    MR, records = O.load_live(image_of)
    mr = MR(ref_import._Cfg({"EXTRA": {"FOCAL_LENGTH": 5000.0}, "MODEL": {"IMAGE_SIZE": 48}}), faces)
    for use_p, use_g in ((True, True), (False, True), (True, False), (False, False)):
        records.clear()
        args = [verts.copy(), cam_t.copy(), images.copy(), pred.copy() if use_p else None,
                gt.copy() if use_g else None]
        live = mr.visualize_tensorboard(*args).numpy()
        front, side = [], []
        for b in range(B):   # the reference's composite (:147-155) of the stand-in's image
            for k, tiles in ((0, front), (1, side)):
                rgba = image_of(records[2 * b + k]).astype(np.float32) / 255.0
                mask = (rgba[..., -1] > 0.8)[..., None]
                bg = np.transpose(images[b], (1, 2, 0)) if k == 0 else np.ones_like(rgba[..., :3])
                tiles.append(np.transpose((rgba[..., :3] * mask + (1 - mask) * bg).astype(np.float32), (2, 0, 1)))
        got = O.visualize_tensorboard(images, front, side, pred if use_p else None, gt if use_g else None, 48)
        assert got.shape == live.shape and np.array_equal(got, live), (use_p, use_g)

"""MeshRenderer (tokenhmr_b200.render) on the GPU: the grid's crop, pad and skeleton parts against the golden written
from the live reference (tests/golden/mesh_renderer_reference.npz, see tests/test_mesh_renderer_oracle.py), bit for
bit; its mesh tiles against Renderer.render_crops on the equivalent inputs, bit for bit."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import openpose_oracle as O
from tokenhmr_b200 import _lib
from tokenhmr_b200 import render as R
from tokenhmr_b200._lib import ThmrError

pytestmark = pytest.mark.gpu
GOLD = "mesh_renderer_reference.npz"
CFG = {"EXTRA": {"FOCAL_LENGTH": 5000.0}, "MODEL": {"IMAGE_SIZE": 256}}


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(golden_dir / GOLD)


@pytest.fixture(scope="module")
def case_inputs():
    return {B: O.golden_inputs(B, seed) for B, seed in O.GOLDEN_CASES}


@pytest.fixture(scope="module")
def mesh_renderer(cuda_dev, case_inputs):
    faces = case_inputs[1][1]
    return R.MeshRenderer(CFG, faces, cuda_dev)


def _variants(B):
    return O.GOLDEN_VARIANTS if B == 8 else {"both": O.GOLDEN_VARIANTS["both"]}


def _call(mr, inputs, use_p, use_g, cuda=False):
    verts, _, cam_t, images, pred, gt = inputs
    args = [verts, cam_t, images, pred if use_p else None, gt if use_g else None]
    if cuda:
        args = [None if a is None else torch.from_numpy(a).cuda() for a in args]
    return mr.visualize_tensorboard(*args, focal_length=np.full((verts.shape[0], 2), 123.0, np.float32))


@pytest.mark.parametrize("B", [B for B, _ in O.GOLDEN_CASES])
def test_grid_matches_golden(mesh_renderer, golden, case_inputs, B):
    """Crop, pad and skeleton tiles bit for bit; the skeleton tiles are decoded from the golden's lossless codes."""
    inputs = case_inputs[B]
    images = inputs[3]
    H, W = images.shape[2:]
    for name, (use_p, use_g) in _variants(B).items():
        key = f"b{B}_{name}"
        grid = _call(mesh_renderer, inputs, use_p, use_g)
        assert grid.is_cuda and grid.dtype == torch.float32
        grid = grid.cpu().numpy()
        assert grid.shape == tuple(golden[f"shape_{key}"]), key
        tiles = 3 + use_p + use_g
        covered = np.zeros(grid.shape[1:], bool)
        for b in range(B):
            for slot in range(tiles):
                ys, xs = O.tile_slices(b, slot, H, W, tiles)
                covered[ys, xs] = True
                if slot == 0:
                    assert np.array_equal(grid[:, ys, xs], images[b]), (key, b)
                elif slot >= 3:
                    want = O.decode_skeleton(golden[f"codes_{key}"][b, slot - 3], images[b])
                    bad = grid[:, ys, xs] != want
                    assert not bad.any(), f"{key} sample {b} skeleton {slot - 3}: {int(bad.any(0).sum())} pixels differ"
        assert (grid[:, ~covered] == 0).all(), f"{key}: padding is not 0"


@pytest.mark.parametrize("B", [1, 8])
def test_mesh_tiles_match_render_crops(mesh_renderer, case_inputs, B):
    """Front tile == render_crops(t) over the crop; side tile == render_crops(side_view, x-negated t) over white (the
    reference's double x flip)."""
    verts, faces, cam_t, images, pred, gt = case_inputs[B]
    H, W = images.shape[2:]
    grid = _call(mesh_renderer, case_inputs[B], True, True).cpu()
    plain = R.Renderer({"EXTRA": {"FOCAL_LENGTH": 5000.0},
                        "MODEL": {"IMAGE_SIZE": 256, "IMAGE_MEAN": [0, 0, 0], "IMAGE_STD": [1, 1, 1]}}, faces)
    v, t, im = torch.from_numpy(verts), torch.from_numpy(cam_t), torch.from_numpy(images)
    front = plain.render_crops(v, t, im).cpu()
    side = plain.render_crops(v, t * torch.tensor([-1.0, 1.0, 1.0]), im, side_view=True,
                              scene_bg_color=(1, 1, 1)).cpu()
    unflipped = plain.render_crops(v, t, im, side_view=True, scene_bg_color=(1, 1, 1)).cpu()
    differs = False
    for b in range(B):
        ys, xs = O.tile_slices(b, 1, H, W, 5)
        assert torch.equal(grid[:, ys, xs], front[b].permute(2, 0, 1)), b
        ys, xs = O.tile_slices(b, 2, H, W, 5)
        assert torch.equal(grid[:, ys, xs], side[b].permute(2, 0, 1)), b
        differs |= not torch.equal(grid[:, ys, xs], unflipped[b].permute(2, 0, 1))
    assert differs, "the side view without the double flip renders the same: the test cannot tell them apart"


def test_numpy_and_cuda_inputs_agree_and_graph_replay_is_stable(mesh_renderer, case_inputs):
    inputs = case_inputs[8]
    a = _call(mesh_renderer, inputs, True, True)
    b = _call(mesh_renderer, inputs, True, True, cuda=True)
    assert torch.equal(a, b)
    # the caller's arrays are not modified (the reference flips camera rows and scales gt_keypoints in place)
    fresh = O.golden_inputs(8, 12)
    for x, y in zip(inputs, fresh):
        assert np.array_equal(x, y)
    cuda_args = [torch.from_numpy(x).cuda() for x in (inputs[0], inputs[2], inputs[3], inputs[4], inputs[5])]
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        mesh_renderer.visualize_tensorboard(*cuda_args)          # warm-up: the renderer's workspace exists
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = mesh_renderer.visualize_tensorboard(*cuda_args)
    g.replay()
    torch.cuda.synchronize()
    first = out.clone()
    assert torch.equal(first, a)
    for _ in range(3):
        g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, first)


def test_visualize_and_call(mesh_renderer, case_inputs):
    verts, faces, cam_t, images, pred, gt = case_inputs[8]
    grid = mesh_renderer.visualize(verts, cam_t, images).cpu()
    full = _call(mesh_renderer, case_inputs[8], True, True).cpu()
    H, W = images.shape[2:]
    assert grid.shape == (3, 8 * (H + 2) + 2, 3 * (W + 2) + 2)       # nrow 3: one sample per grid row
    for b in range(8):
        for slot in range(3):
            ys, xs = O.tile_slices(b, slot, H, W, 5)
            assert torch.equal(grid[:, ys, xs], full[:, ys, xs]), (b, slot)
    front = mesh_renderer(verts[0], cam_t[0], np.transpose(images[0], (1, 2, 0)))
    assert front.dtype == np.float32 and front.shape == (H, W, 3)
    assert np.array_equal(front, np.transpose(full[:, 2:2 + H, W + 4:2 * W + 4].numpy(), (1, 2, 0)))
    with pytest.raises(ThmrError):
        mesh_renderer(verts[0], cam_t[0], np.transpose(images[0], (1, 2, 0)), resize=(128, 128))


def test_bad_inputs_raise(mesh_renderer, case_inputs):
    verts, faces, cam_t, images, pred, gt = case_inputs[1]
    with pytest.raises(ThmrError):
        mesh_renderer.visualize_tensorboard(verts, cam_t, images, pred[:, :25], gt)        # 25 keypoints, not 44
    with pytest.raises(ThmrError):
        mesh_renderer.visualize_tensorboard(verts, cam_t, images, gt, gt)                  # 3 columns for predictions
    with pytest.raises(ThmrError):
        mesh_renderer.visualize_tensorboard(verts, cam_t[:, :2], images, pred, gt)
    with pytest.raises(ThmrError):
        mesh_renderer.visualize_tensorboard(verts, cam_t, images[:, :2], pred, gt)
    with pytest.raises(ThmrError):                                                         # wider than the overlay's
        mesh_renderer.visualize_tensorboard(verts, cam_t, np.zeros((1, 3, 4, _lib.POSE_MAX_WIDTH + 1), np.float32),
                                            pred, gt)
    L = _lib.lib()
    d = _lib.PoseGridDesc()
    assert L.thmr_pose_grid(ctypes.byref(d), None, None) == -1
    assert L.thmr_pose_grid_workspace_bytes(0, 8, 8, 2) == 0
    x = torch.zeros(64, device="cuda")
    d.n, d.width, d.height, d.nrow, d.padding, d.img_res = 1, 2, 2, 5, 2, 256.0
    d.images = d.front = d.side = d.out = x.data_ptr()
    d.out_stride_c, d.out_stride_y = 100, 3          # a grid row is 3 * (2 + 2) + 2 = 14 wide
    assert L.thmr_pose_grid(ctypes.byref(d), x.data_ptr(), None) == -1
    assert b"strides" in L.thmr_last_error()

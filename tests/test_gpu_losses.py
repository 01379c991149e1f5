"""The training loss on the GPU (csrc/losses.cuh behind thmr_tokenhmr_loss, thmr_camera_tail and
thmr_camera_tail_backward; tokenhmr_b200.losses): every term and gradient against the fp64 reference run stored in
tests/golden/tals_loss.npz, the camera tail against fp64 autograd and bitwise against the engine's fused tail, the whole
differentiable_tail -> loss chain against fp64 autograd through oracle.smpl_oracle, CUDA-graph capture, the rejections,
and a frozen-backbone fine-tuning run.

The loss kernel computes in double from the fp32 inputs and rounds once, so its terms and gradients sit within a few
fp32 ulps of the fp64 reference; the chain through the body model inherits that model's fp32 backward (1e-4 of the
largest gradient, tests/test_gpu_smpl_grad.py)."""
import copy

import numpy as np
import pytest
import torch

from oracle import loss_oracle as LO
from oracle import smpl_oracle as S

pytestmark = pytest.mark.gpu

REL = 1e-5          # loss terms against the golden
GRAD_REL = 1e-6     # per element: |g - g64| <= GRAD_REL * max |g64| + GRAD_REL * |g64|
CHAIN_REL = 1e-3    # gradients through the fp32 body model, per tensor: max |g - g64| <= CHAIN_REL * max |g64|


def _batch(golden, case, dev):
    t = lambda k: torch.from_numpy(golden[f"{case}_{k}"].copy()).float().to(dev)
    B = golden[f"{case}_pred_betas"].shape[0]
    batch = {"keypoints_2d": t("gt_keypoints_2d"), "keypoints_3d": t("gt_keypoints_3d"),
             "smpl_params": {"global_orient": t("gt_global_orient"), "body_pose": t("gt_body_pose"),
                             "betas": t("gt_betas")},
             "has_smpl_params": {k: t("has_" + k) for k in ("global_orient", "body_pose", "betas")},
             "smpl_params_is_axis_angle": {"global_orient": torch.ones(B, dtype=torch.bool, device=dev),
                                           "body_pose": torch.ones(B, dtype=torch.bool, device=dev),
                                           "betas": torch.zeros(B, dtype=torch.bool, device=dev)},
             "dataset": [str(n) for n in golden[f"{case}_dataset"]]}
    output = {"pred_smpl_params": {"global_orient": t("pred_global_orient"), "body_pose": t("pred_body_pose"),
                                   "betas": t("pred_betas")},
              "pred_keypoints_2d": t("pred_keypoints_2d"), "pred_keypoints_3d": t("pred_keypoints_3d")}
    return batch, output


def _leaves(output):
    ins = [output["pred_keypoints_2d"], output["pred_keypoints_3d"], *output["pred_smpl_params"].values()]
    for x in ins:
        x.requires_grad_(True)
    return ins


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(golden_dir / "tals_loss.npz")


@pytest.fixture(scope="module")
def crit():
    from tokenhmr_b200.losses import TokenHMRLoss
    return TokenHMRLoss({"MODEL": {"LOOSE_SUP": True, "LOOSE_WEIGHT": LO.LOOSE_WEIGHT},
                         "LOSS_WEIGHTS": dict(LO.LOSS_WEIGHTS, ADVERSARIAL=0.0)})


@pytest.mark.parametrize("case", list(LO.CASES))
def test_loss_and_gradients_match_golden(cuda_dev, golden, crit, case):
    """Every term of output['losses'] within REL of the fp64 reference, each gradient element within GRAD_REL, and the
    caller's batch left exactly as it was."""
    from tokenhmr_b200._lib import check, lib
    batch, output = _batch(golden, case, cuda_dev)
    before = copy.deepcopy(batch)
    ins = _leaves(output)
    loss = crit(batch, output, train=bool(golden[f"{case}_config"][1]))
    grads = torch.autograd.grad(loss, ins)
    torch.cuda.synchronize()
    check(lib().thmr_check_device_flags())
    want = golden[f"{case}_losses"]
    got = np.array([output["losses"][k].item() for k in ("loss", "loss_keypoints_2d", "loss_keypoints_3d",
                                                          "loss_global_orient", "loss_body_pose", "loss_betas")])
    np.testing.assert_allclose(got, want, rtol=REL)
    assert loss.item() == got[0]
    for k, g in zip(LO.PRED_KEYS, grads):
        ref = golden[f"{case}_grad_{k[len('pred_'):]}"]
        err = np.abs(g.double().cpu().numpy() - ref)
        assert (err <= GRAD_REL * (np.abs(ref).max() + np.abs(ref))).all(), (k, err.max())
    for k in ("keypoints_2d", "keypoints_3d"):
        assert torch.equal(batch[k], before[k]), k
    for k in ("has_smpl_params", "smpl_params", "smpl_params_is_axis_angle"):
        for n in batch[k]:
            assert torch.equal(batch[k][n], before[k][n]), (k, n)
    assert batch["dataset"] == before["dataset"]


def test_valid_3d_tensor_equals_names_and_graph_replay_equals_eager(cuda_dev, golden, crit):
    """batch['dataset'] as a precomputed (B,) tensor gives the same numbers as the names; the loss and its gradients
    captured in one CUDA graph replay to the eager values bit for bit.  The graph's leaves are made inside the capture,
    so that autograd's stream for them is the capture stream."""
    batch, output = _batch(golden, "tals", cuda_dev)
    ins = _leaves(output)
    loss = crit(batch, output)
    eager = [loss.detach().clone(), *[g.clone() for g in torch.autograd.grad(loss, ins)]]
    batch["dataset"] = torch.from_numpy(golden["tals_valid_3d"]).float().to(cuda_dev)
    raw = [x.detach() for x in ins]

    def step():
        leaves = [x.clone().requires_grad_(True) for x in raw]
        out = {"pred_keypoints_2d": leaves[0], "pred_keypoints_3d": leaves[1],
               "pred_smpl_params": dict(zip(("global_orient", "body_pose", "betas"), leaves[2:]))}
        loss = crit(batch, out)
        return [loss.detach(), *torch.autograd.grad(loss, leaves)]

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            step()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        got = step()
    g.replay()
    torch.cuda.synchronize()
    for a, b in zip(eager, got):
        assert torch.equal(a, b)


def _tail64(joints, cam, focal=5000.0, size=256.0):
    t = torch.stack([cam[:, 1], cam[:, 2], 2 * focal / (size * cam[:, 0] + 1e-9)], -1)
    p = joints + t[:, None]
    return t, (focal / size) * p[..., :2] / p[..., 2:]


@pytest.mark.parametrize("B,J", [(1, 44), (33, 44), (5, 70)])
def test_camera_tail_vs_fp64_autograd(cuda_dev, B, J):
    from tokenhmr_b200 import ops
    g = torch.Generator().manual_seed(B * 100 + J)
    joints = (0.5 * torch.randn(B, J, 3, generator=g)).to(cuda_dev).requires_grad_(True)
    cam = torch.stack([0.7 + 0.4 * torch.rand(B, generator=g), 0.1 * torch.randn(B, generator=g),
                       0.1 * torch.randn(B, generator=g)], 1).to(cuda_dev).requires_grad_(True)
    gk, gc = torch.randn(B, J, 2, generator=g).to(cuda_dev), torch.randn(B, 3, generator=g).to(cuda_dev)
    cam_t, focal, kp2d = ops.camera_tail(joints, cam)
    assert torch.equal(focal, torch.full((B, 2), 5000.0, device=cuda_dev))
    gj, gcam = torch.autograd.grad((kp2d * gk).sum() + (cam_t * gc).sum(), [joints, cam])
    j64, c64 = joints.detach().double().requires_grad_(True), cam.detach().double().requires_grad_(True)
    t64, k64 = _tail64(j64, c64)
    torch.testing.assert_close(cam_t.double(), t64, rtol=1e-6, atol=0)
    torch.testing.assert_close(kp2d.double(), k64, rtol=1e-6, atol=1e-6 * k64.abs().max().item())
    rj, rc = torch.autograd.grad((k64 * gk.double()).sum() + (t64 * gc.double()).sum(), [j64, c64])
    for got, ref in ((gj, rj), (gcam, rc)):
        assert ((got.double() - ref).abs() <= 1e-5 * ref.abs().max()).all()


def test_camera_tail_is_bitwise_the_engine_forward(cuda_dev):
    from tokenhmr_b200 import ops, synth
    from tokenhmr_b200.config import tiny_config
    from tokenhmr_b200.engine import TokenHMREngine
    cfg = tiny_config()
    model = TokenHMREngine(cfg, synth.make_state_dict(cfg), synth.make_smpl(cfg), device=cuda_dev, use_cuda_graph=False)
    out = model({"img": synth.make_images(3, cfg)})
    cam_t, focal, kp2d = ops.camera_tail(out["pred_keypoints_3d"], out["pred_cam"], cfg.focal_length, cfg.image_size)
    assert torch.equal(cam_t, out["pred_cam_t"])
    assert torch.equal(focal, out["focal_length"])
    assert torch.equal(kp2d, out["pred_keypoints_2d"])


@pytest.fixture(scope="module")
def body(cuda_dev):
    from tokenhmr_b200 import ops, synth
    from tokenhmr_b200.config import release_config
    smpl = synth.make_smpl(release_config())
    s64 = {k: (v.double() if v.is_floating_point() else v) for k, v in smpl.items()}     # the oracle runs on the CPU
    return s64, ops.SMPLModel(smpl, cuda_dev)


@pytest.mark.parametrize("case", list(LO.CASES))
def test_tail_to_loss_gradient_vs_fp64(cuda_dev, golden, crit, body, case):
    """differentiable_tail -> TokenHMRLoss -> backward reaches the rotations, betas and pred_cam; against fp64 autograd
    through oracle.smpl_oracle and oracle.loss_oracle.torch_loss."""
    from tokenhmr_b200.losses import differentiable_tail
    s64, m = body
    batch, output = _batch(golden, case, cuda_dev)
    B = batch["keypoints_2d"].shape[0]
    gen = torch.Generator().manual_seed(5)
    cam = torch.stack([0.8 + 0.3 * torch.rand(B, generator=gen), 0.1 * torch.randn(B, generator=gen),
                       0.1 * torch.randn(B, generator=gen)], 1).to(cuda_dev)
    params = {k: v.clone().requires_grad_(True) for k, v in output["pred_smpl_params"].items()}
    cam.requires_grad_(True)
    tail = differentiable_tail(m, params, cam, 5000.0, 256.0)
    tail["pred_smpl_params"] = params
    train = bool(golden[f"{case}_config"][1])
    loss = crit(batch, tail, train=train)
    grads = torch.autograd.grad(loss, [params["global_orient"], params["body_pose"], params["betas"], cam])
    p64 = {k: v.detach().cpu().double().requires_grad_(True) for k, v in params.items()}
    c64 = cam.detach().cpu().double().requires_grad_(True)
    verts, joints = S.smpl_forward(s64, p64["global_orient"], p64["body_pose"], p64["betas"], dtype=torch.float64)
    _, kp2d = _tail64(joints, c64)
    gt = {k: torch.from_numpy(golden[f"{case}_{k}"].copy())
          for k in ("gt_keypoints_2d", "gt_keypoints_3d", "gt_global_orient", "gt_body_pose", "gt_betas",
                    "has_global_orient", "has_body_pose", "has_betas")}
    pred = {"pred_keypoints_2d": kp2d, "pred_keypoints_3d": joints, "pred_global_orient": p64["global_orient"],
            "pred_body_pose": p64["body_pose"], "pred_betas": p64["betas"]}
    terms = LO.torch_loss(pred, gt, torch.from_numpy(golden[f"{case}_valid_3d"]), train)
    assert abs(loss.item() - terms[0].item()) <= 1e-4 * abs(terms[0].item())
    refs = torch.autograd.grad(terms[0], [p64["global_orient"], p64["body_pose"], p64["betas"], c64])
    for name, got, ref in zip(("global_orient", "body_pose", "betas", "pred_cam"), grads, refs):
        err = (got.cpu().double() - ref).abs().max().item()
        assert err <= CHAIN_REL * ref.abs().max().item(), (name, err, ref.abs().max().item())


def test_rejections(cuda_dev, golden, crit):
    from tokenhmr_b200._lib import ThmrError, lib
    batch, output = _batch(golden, "tals", cuda_dev)
    cut = {**output, "pred_keypoints_2d": output["pred_keypoints_2d"][:, :43].contiguous(),
           "pred_keypoints_3d": output["pred_keypoints_3d"][:, :43].contiguous()}
    cut_batch = {**batch, "keypoints_2d": batch["keypoints_2d"][:, :43].contiguous(),
                 "keypoints_3d": batch["keypoints_3d"][:, :43].contiguous()}
    with pytest.raises(ThmrError, match="44 keypoints"):
        crit(cut_batch, dict(cut), train=True)
    crit(cut_batch, dict(cut), train=False)           # the plain branch takes any J > pelvis_id
    with pytest.raises(ThmrError, match="shapes"):
        crit({**batch, "keypoints_3d": batch["keypoints_3d"][..., :3].contiguous()}, dict(output))
    with pytest.raises(ThmrError, match="names"):
        crit({**batch, "dataset": batch["dataset"][:-1]}, dict(output))
    torch.cuda.synchronize()
    assert lib().thmr_check_device_flags() == 0
    flags = dict(batch["smpl_params_is_axis_angle"])
    flags["betas"] = flags["betas"].clone()
    flags["betas"][3] = True
    crit({**batch, "smpl_params_is_axis_angle": flags}, dict(output))
    torch.cuda.synchronize()
    assert lib().thmr_check_device_flags() == -1
    assert b"smpl_params_is_axis_angle" in lib().thmr_last_error()
    assert lib().thmr_check_device_flags() == 0       # read and cleared


def _rot6d(x):
    """geometry.rot6d_to_rotmat in torch (the head under training is a plain PyTorch module)."""
    x = x.reshape(-1, 2, 3).permute(0, 2, 1)
    b1 = torch.nn.functional.normalize(x[:, :, 0])
    a2 = x[:, :, 1]
    b2 = torch.nn.functional.normalize(a2 - (b1 * a2).sum(-1, keepdim=True) * b1)
    return torch.stack((b1, b2, torch.cross(b1, b2, dim=-1)), dim=-2)


def _head_forward(lin, feats):
    B = feats.shape[0]
    y = lin(feats.mean((2, 3)))
    rot = _rot6d(y[:, :144] + torch.tensor([1, 0, 0, 0, 1, 0], dtype=y.dtype, device=y.device).repeat(24)).view(B, 24, 3, 3)
    cam = y[:, 154:157] + torch.tensor([0.9, 0.0, 0.0], dtype=y.dtype, device=y.device)
    return {"global_orient": rot[:, :1], "body_pose": rot[:, 1:], "betas": y[:, 144:154]}, cam


def test_frozen_backbone_fine_tuning(cuda_dev, crit):
    """A small PyTorch head on frozen model.backbone features of tiny_config, trained with the TALS loss through
    differentiable_tail(model.smpl, ...) for 30 Adam steps: the loss falls, and the step-0 head gradients match the
    same chain in fp64 torch (oracle body model, torch_loss)."""
    from tokenhmr_b200 import synth
    from tokenhmr_b200.config import tiny_config
    from tokenhmr_b200.losses import differentiable_tail
    cfg = tiny_config()
    smpl = synth.make_smpl(cfg)
    from tokenhmr_b200.engine import TokenHMREngine
    model = TokenHMREngine(cfg, synth.make_state_dict(cfg), smpl, device=cuda_dev, use_cuda_graph=False)
    B = 8
    feats = model.backbone(synth.make_images(B, cfg)).detach()
    g = torch.Generator().manual_seed(3)
    gt_aa = (0.3 * torch.randn(B, 24, 3, generator=g)).to(cuda_dev)
    gt_betas = torch.randn(B, 10, generator=g).to(cuda_dev)
    with torch.no_grad():
        rot = S.batch_rodrigues(gt_aa.reshape(-1, 3).cpu()).view(B, 24, 3, 3).to(cuda_dev)
        gt_cam = torch.tensor([[0.9, 0.02, -0.03]], device=cuda_dev).expand(B, 3).contiguous()
        gt_out = differentiable_tail(model.smpl, {"global_orient": rot[:, :1], "body_pose": rot[:, 1:],
                                                  "betas": gt_betas}, gt_cam, cfg.focal_length, cfg.image_size)
    ones = torch.ones(B, 44, 1, device=cuda_dev)
    batch = {"keypoints_2d": torch.cat([gt_out["pred_keypoints_2d"], ones], -1),
             "keypoints_3d": torch.cat([gt_out["pred_keypoints_3d"], ones], -1),
             "smpl_params": {"global_orient": gt_aa[:, 0], "body_pose": gt_aa[:, 1:].reshape(B, 69), "betas": gt_betas},
             "has_smpl_params": {k: torch.ones(B, device=cuda_dev) for k in ("global_orient", "body_pose", "betas")},
             "smpl_params_is_axis_angle": {"global_orient": torch.ones(B, dtype=torch.bool, device=cuda_dev),
                                           "body_pose": torch.ones(B, dtype=torch.bool, device=cuda_dev),
                                           "betas": torch.zeros(B, dtype=torch.bool, device=cuda_dev)},
             "dataset": ["BEDLAM", "COCO-TRAIN-2014"] * (B // 2)}
    torch.manual_seed(0)
    lin = torch.nn.Linear(cfg.vit_dim, 157).to(cuda_dev)
    torch.nn.init.normal_(lin.weight, std=1e-3)
    torch.nn.init.zeros_(lin.bias)
    lin64 = copy.deepcopy(lin).double()
    opt = torch.optim.Adam(lin.parameters(), lr=1e-3)
    losses = []
    for step in range(30):
        params, cam = _head_forward(lin, feats)
        out = differentiable_tail(model.smpl, params, cam, cfg.focal_length, cfg.image_size)
        out["pred_smpl_params"] = params
        loss = crit(batch, out, train=True)
        opt.zero_grad()
        loss.backward()
        if step == 0:
            g0 = [p.grad.clone() for p in lin.parameters()]
        opt.step()
        losses.append(loss.item())
    assert losses[-1] < 0.5 * losses[0], losses
    # step 0 in fp64 torch
    s64 = {k: (v.double() if v.is_floating_point() else v) for k, v in smpl.items()}
    lin64 = lin64.cpu()
    params, cam = _head_forward(lin64, feats.cpu().double())
    verts, joints = S.smpl_forward(s64, params["global_orient"], params["body_pose"], params["betas"],
                                   dtype=torch.float64)
    _, kp2d = _tail64(joints, cam, cfg.focal_length, cfg.image_size)
    c = lambda t: t.cpu().double()
    gt = {"gt_keypoints_2d": c(batch["keypoints_2d"]), "gt_keypoints_3d": c(batch["keypoints_3d"]),
          "gt_global_orient": c(gt_aa[:, 0]), "gt_body_pose": c(gt_aa[:, 1:].reshape(B, 69)),
          "gt_betas": c(gt_betas), **{"has_" + k: torch.ones(B, dtype=torch.float64)
                                      for k in ("global_orient", "body_pose", "betas")}}
    pred = {"pred_keypoints_2d": kp2d, "pred_keypoints_3d": joints, "pred_global_orient": params["global_orient"],
            "pred_body_pose": params["body_pose"], "pred_betas": params["betas"]}
    v3d = torch.tensor([1.0, 0.0] * (B // 2), dtype=torch.float64)
    terms = LO.torch_loss(pred, gt, v3d, True)
    assert abs(terms[0].item() - losses[0]) <= 1e-4 * abs(terms[0].item())
    refs = torch.autograd.grad(terms[0], list(lin64.parameters()))
    for got, ref in zip(g0, refs):
        assert (got.cpu().double() - ref).abs().max().item() <= CHAIN_REL * ref.abs().max().item()

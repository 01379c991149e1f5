"""Training HMR 2.0's regression head on the GPU (csrc/head_train.cuh behind thmr_reg_head_train_forward /
thmr_reg_head_backward; tokenhmr_b200.heads.RegressionHead), with the release decoder (depth 6, 8 heads, mlp 1024):
the forward against the fp64 restatement of SMPLTransformerDecoderHead and against a strict engine, every parameter
gradient against fp64 autograd, graph replay and determinism, batch independence, and a 30-step AdamW fine-tune with
the TALS loss whose weights a strict engine then serves.

Gradient bound per parameter tensor: max |g - g64| <= max(4 x the fp32 torch restatement's own error, 1e-5 max |g64|).
"""
import pytest
import torch

from oracle import regression_oracle as R
from oracle import smpl_oracle as S
from oracle import tokenhmr_oracle as O

pytestmark = pytest.mark.gpu

REG = "transformer_decoder"


@pytest.fixture(scope="module")
def setup(cuda_dev):
    from tokenhmr_b200 import synth
    from tokenhmr_b200.config import tiny_config
    from tokenhmr_b200.engine import TokenHMREngine
    cfg = tiny_config(vit_depth=2, head=REG)
    sd, smpl = synth.make_state_dict(cfg), synth.make_smpl(cfg)
    strict = TokenHMREngine(cfg, sd, smpl, device=cuda_dev, use_cuda_graph=False, strict=True)
    return cfg, sd, smpl, strict


def _feats(cfg, B, seed, dev):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(B, cfg.vit_dim, cfg.grid_h, cfg.grid_w, generator=g).to(dev)


def _head_sd(sd, dtype, dev):
    return {k: v.to(dev, dtype).clone().requires_grad_(k.split(".")[-1] not in ("init_body_pose", "init_betas",
                                                                                  "init_cam"))
            for k, v in sd.items() if k.startswith("smpl_head.")}


def _restated(sd, feats, cfg, dtype):
    """The restatement of SMPLTransformerDecoderHead.forward (oracle.regression_oracle) in `dtype` with autograd:
    (leaf state dict, pose6d, betas, cam, rotmats)."""
    leaves = _head_sd(sd, dtype, feats.device)
    params, cam, aux = R.regression_head_forward(leaves, feats.to(dtype).flatten(2).transpose(1, 2), cfg,
                                                 O.Numerics(False))
    rot = torch.cat([params["global_orient"], params["body_pose"]], 1)
    return leaves, aux["pred_body_pose_6d"], params["betas"], cam, rot


def _upstream(B, seed, dev):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(B, 24, 3, 3, generator=g).to(dev), torch.randn(B, 10, generator=g).to(dev),
            torch.randn(B, 3, generator=g).to(dev))


def _ref_grads(leaves, outs, up):
    rot, betas, cam = outs
    loss = (rot * up[0].to(rot.dtype)).sum() + (betas * up[1].to(rot.dtype)).sum() + (cam * up[2].to(rot.dtype)).sum()
    names = [k for k, v in leaves.items() if v.requires_grad]
    gs = torch.autograd.grad(loss, [leaves[k] for k in names], allow_unused=True)
    return {k[len("smpl_head."):]: (torch.zeros_like(leaves[k]) if g is None else g) for k, g in zip(names, gs)}


def _cuda_grads(head, feats, up):
    head.zero_grad(set_to_none=True)
    params, cam, _ = head(feats)
    rot = torch.cat([params["global_orient"], params["body_pose"]], 1)
    loss = (rot * up[0]).sum() + (params["betas"] * up[1]).sum() + (cam * up[2]).sum()
    loss.backward()
    return {k: p.grad.clone() for k, p in head.named_parameters()}, rot.detach(), params["betas"].detach(), cam.detach()


@pytest.mark.parametrize("B", [1, 5, 48])
def test_forward_matches_fp64_restatement(setup, cuda_dev, B):
    from tokenhmr_b200.heads import RegressionHead
    cfg, sd, _, _ = setup
    head = RegressionHead(cfg, sd, cuda_dev)
    feats = _feats(cfg, B, B, cuda_dev)
    with torch.no_grad():
        params, cam, lst = head(feats)
        _, p6, be, ca, rot = _restated(sd, feats, cfg, torch.float64)
    got_rot = torch.cat([params["global_orient"], params["body_pose"]], 1)
    assert tuple(got_rot.shape) == (B, 24, 3, 3) and tuple(params["betas"].shape) == (B, 10) and tuple(cam.shape) == (B, 3)
    assert torch.equal(lst["body_pose"], params["body_pose"]) and torch.equal(lst["cam"], cam)
    for name, a, b in (("rotmats", got_rot, rot), ("betas", params["betas"], be), ("cam", cam, ca)):
        err = ((a.double() - b).abs().max() / b.abs().max()).item()
        print(f"B={B} {name}: {err:.2e}")
        assert err <= 1e-5, (name, err)


def test_pose6d_output_and_no_saved_state_under_no_grad(setup, cuda_dev):
    """The 6D pose the backward differentiates is the restatement's; under no_grad the call keeps no workspace."""
    from tokenhmr_b200.heads import _RegHeadFn, RegressionHead
    cfg, sd, _, _ = setup
    head = RegressionHead(cfg, sd, cuda_dev)
    feats = _feats(cfg, 3, 1, cuda_dev)
    with torch.no_grad():
        p6, _, _, _ = _RegHeadFn.apply(head, False, feats, *head._params())
        _, p6_ref, _, _, _ = _restated(sd, feats, cfg, torch.float64)
        assert p6.grad_fn is None
    assert ((p6.double() - p6_ref).abs().max() / p6_ref.abs().max()).item() <= 1e-5


def test_forward_matches_the_strict_engine(setup):
    """head(strict.backbone(img)) against strict(batch): both see the same features."""
    from tokenhmr_b200 import synth
    from tokenhmr_b200.heads import RegressionHead
    cfg, sd, _, strict = setup
    img = synth.make_images(4, cfg, seed=7)
    head = RegressionHead(cfg, sd, strict.device)
    with torch.no_grad():
        params, cam, _ = head(strict.backbone(img))
    want = strict({"img": img})
    rel = lambda a, b: ((a - b).abs().max() / b.abs().max()).item()
    assert rel(cam, want["pred_cam"]) <= 1e-4
    for k in ("global_orient", "body_pose", "betas"):
        assert rel(params[k], want["pred_smpl_params"][k]) <= 1e-4, k


@pytest.mark.parametrize("B", [1, 5, 48])
def test_gradients_match_fp64_autograd(setup, cuda_dev, B):
    from tokenhmr_b200.heads import RegressionHead
    cfg, sd, _, _ = setup
    head = RegressionHead(cfg, sd, cuda_dev)
    feats = _feats(cfg, B, 100 + B, cuda_dev)
    up = _upstream(B, 200 + B, cuda_dev)
    got, *_ = _cuda_grads(head, feats, up)
    l64, _, be, ca, rot = _restated(sd, feats, cfg, torch.float64)
    g64 = _ref_grads(l64, (rot, be, ca), up)
    l32, _, be, ca, rot = _restated(sd, feats, cfg, torch.float32)
    g32 = _ref_grads(l32, (rot, be, ca), up)
    assert set(got) == set(g64)
    worst = 0.0
    for k, ref in g64.items():
        scale = ref.abs().max().item()
        err = (got[k].double() - ref).abs().max().item()
        own = (g32[k].double() - ref).abs().max().item()
        bound = max(4 * own, 1e-5 * scale)
        worst = max(worst, err / max(bound, 1e-300))
        assert err <= bound, (k, err, own, scale)
    print(f"B={B}: worst gradient error / bound = {worst:.2f}")
    inner = cfg.dec_inner
    for l in range(cfg.dec_depth):
        assert not got[f"transformer.transformer.layers.{l}.0.fn.to_qkv.weight"][:2 * inner].any()
    assert not got["transformer.to_token_embedding.weight"].any()


def test_graph_replay_equals_eager_bit_for_bit(setup, cuda_dev):
    from tokenhmr_b200.heads import RegressionHead
    cfg, sd, _, _ = setup
    head = RegressionHead(cfg, sd, cuda_dev)
    B = 6
    feats = _feats(cfg, B, 11, cuda_dev)
    up = _upstream(B, 12, cuda_dev)
    e1 = _cuda_grads(head, feats, up)
    e2 = _cuda_grads(head, feats, up)
    for k in e1[0]:
        assert torch.equal(e1[0][k], e2[0][k]), k
    for a, b in zip(e1[1:], e2[1:]):
        assert torch.equal(a, b)
    static_feats = feats.clone()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        _cuda_grads(head, static_feats, up)            # warm-up on the capture stream
    torch.cuda.current_stream().wait_stream(s)
    head.zero_grad(set_to_none=True)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        params, cam, _ = head(static_feats)
        rot = torch.cat([params["global_orient"], params["body_pose"]], 1)
        loss = (rot * up[0]).sum() + (params["betas"] * up[1]).sum() + (cam * up[2]).sum()
        loss.backward()
    for _ in range(2):
        g.replay()
        torch.cuda.synchronize()
        for k, p in head.named_parameters():
            assert torch.equal(p.grad, e1[0][k]), k
        assert torch.equal(rot, e1[1]) and torch.equal(cam, e1[3])


def test_batch_independence(setup, cuda_dev):
    """Row b's outputs and its own gradient (the batch of one) do not depend on the other rows."""
    from tokenhmr_b200.heads import RegressionHead
    cfg, sd, _, _ = setup
    head = RegressionHead(cfg, sd, cuda_dev)
    feats = _feats(cfg, 5, 21, cuda_dev)
    up = _upstream(5, 22, cuda_dev)
    with torch.no_grad():
        p_all, cam_all, _ = head(feats)
        p_one, cam_one, _ = head(feats[2:3].contiguous())
    torch.testing.assert_close(cam_one, cam_all[2:3], rtol=0, atol=1e-6)
    torch.testing.assert_close(p_one["body_pose"], p_all["body_pose"][2:3], rtol=0, atol=1e-6)
    other = feats.clone()
    other[[0, 1, 3, 4]] = _feats(cfg, 4, 23, cuda_dev)
    only_b = tuple(torch.zeros_like(u) for u in up)
    for z, u in zip(only_b, up):
        z[2] = u[2]
    ga, *_ = _cuda_grads(head, feats, only_b)
    gb, *_ = _cuda_grads(head, other, only_b)
    for k in ga:
        scale = ga[k].abs().max().item()
        assert (ga[k] - gb[k]).abs().max().item() <= 1e-6 * max(scale, 1e-30) + 1e-30, k


def test_rejections(setup, cuda_dev):
    from tokenhmr_b200._lib import ThmrError
    from tokenhmr_b200.heads import RegressionHead
    cfg, sd, _, _ = setup
    head = RegressionHead(cfg, sd, cuda_dev)
    f = _feats(cfg, 2, 0, cuda_dev)
    for bad, msg in ((f[:, :, :, :6], "must be"), (f.double(), "float32"), (f.cpu(), "features on"),
                     (f.transpose(2, 3).contiguous().transpose(2, 3), "contiguous"),
                     (f.clone().requires_grad_(True), "not built")):
        with pytest.raises(ThmrError, match=msg):
            head(bad)


def _fine_tune_batch(model, cfg, B, dev):
    from tokenhmr_b200.losses import differentiable_tail
    g = torch.Generator().manual_seed(3)
    gt_aa = (0.3 * torch.randn(B, 24, 3, generator=g)).to(dev)
    gt_betas = torch.randn(B, 10, generator=g).to(dev)
    with torch.no_grad():
        rot = S.batch_rodrigues(gt_aa.reshape(-1, 3).cpu()).view(B, 24, 3, 3).to(dev)
        gt_cam = torch.tensor([[0.9, 0.02, -0.03]], device=dev).expand(B, 3).contiguous()
        gt_out = differentiable_tail(model.smpl, {"global_orient": rot[:, :1], "body_pose": rot[:, 1:],
                                                  "betas": gt_betas}, gt_cam, cfg.focal_length, cfg.image_size)
    ones = torch.ones(B, 44, 1, device=dev)
    return {"keypoints_2d": torch.cat([gt_out["pred_keypoints_2d"], ones], -1),
            "keypoints_3d": torch.cat([gt_out["pred_keypoints_3d"], ones], -1),
            "smpl_params": {"global_orient": gt_aa[:, 0], "body_pose": gt_aa[:, 1:].reshape(B, 69), "betas": gt_betas},
            "has_smpl_params": {k: torch.ones(B, device=dev) for k in ("global_orient", "body_pose", "betas")},
            "smpl_params_is_axis_angle": {"global_orient": torch.ones(B, dtype=torch.bool, device=dev),
                                          "body_pose": torch.ones(B, dtype=torch.bool, device=dev),
                                          "betas": torch.zeros(B, dtype=torch.bool, device=dev)},
            "dataset": ["BEDLAM", "COCO-TRAIN-2014"] * (B // 2)}


class _TorchHead(torch.nn.Module):
    """The fp32 torch restatement as a module with the same parameter names, for the same optimiser."""

    def __init__(self, sd, cfg, dev):
        super().__init__()
        self.cfg = cfg
        self.p = torch.nn.ParameterDict({k[len("smpl_head."):].replace(".", "/"): torch.nn.Parameter(v.to(dev).clone())
                                         for k, v in sd.items() if k.startswith("smpl_head.") and "init_" not in k})
        self.init = {k: v.to(dev) for k, v in sd.items() if "init_" in k}

    def forward(self, feats):
        sd = {"smpl_head." + k.replace("/", "."): v for k, v in self.p.items()}
        sd.update(self.init)
        params, cam, _ = R.regression_head_forward(sd, feats.flatten(2).transpose(1, 2), self.cfg, O.Numerics(False))
        return params, cam


def test_fine_tune_with_adamw_and_serve_the_weights(setup, cuda_dev):
    from tokenhmr_b200.engine import TokenHMREngine
    from tokenhmr_b200.heads import RegressionHead
    from tokenhmr_b200.losses import TokenHMRLoss, differentiable_tail
    from tokenhmr_b200 import synth
    cfg, sd, smpl, strict = setup
    B = 8
    img = synth.make_images(B, cfg, seed=41)
    feats = strict.backbone(img).detach()
    batch = _fine_tune_batch(strict, cfg, B, cuda_dev)
    crit = TokenHMRLoss({"MODEL": {"LOOSE_SUP": True, "LOOSE_WEIGHT": 0.1},
                         "LOSS_WEIGHTS": {"KEYPOINTS_2D": 0.01, "KEYPOINTS_3D": 0.05, "GLOBAL_ORIENT": 0.001,
                                          "BODY_POSE": 0.001, "BETAS": 0.0005}})
    head = RegressionHead(cfg, sd, cuda_dev)
    ref = _TorchHead(sd, cfg, cuda_dev)
    kw = dict(lr=5e-5, weight_decay=1e-4)
    opt, opt_ref = torch.optim.AdamW(head.parameters(), **kw), torch.optim.AdamW(ref.parameters(), **kw)
    losses = []
    for step in range(30):
        for h, o, is_ref in ((head, opt, False), (ref, opt_ref, True)):
            if is_ref:
                params, cam = h(feats)
            else:
                params, cam, _ = h(feats)
            out = differentiable_tail(strict.smpl, params, cam, cfg.focal_length, cfg.image_size)
            out["pred_smpl_params"] = params
            loss = crit(batch, out, train=True)
            o.zero_grad()
            loss.backward()
            o.step()
            if not is_ref:
                losses.append(loss.item())
    print("loss", losses[0], "->", losses[-1])
    assert losses[-1] < 0.5 * losses[0], losses
    ours = dict(head.named_parameters())
    largest = max(p.abs().max().item() for p in ref.p.values())
    drift = {k.replace("/", "."): (ours[k.replace("/", ".")] - p).abs().max().item() for k, p in ref.p.items()}
    print("largest |param|", largest, "worst drift from the torch restatement", max(drift.items(), key=lambda kv: kv[1]))
    for name, d in drift.items():
        assert d <= 1e-4 * largest, (name, d)
    # serve the fine-tuned weights from a strict engine
    tuned = dict(sd)
    tuned.update({"smpl_head." + k: v.detach().cpu() for k, v in head.state_dict().items()})
    served = TokenHMREngine(cfg, tuned, smpl, device=cuda_dev, use_cuda_graph=False, strict=True)
    want = served({"img": img})
    with torch.no_grad():
        params, cam, _ = head(served.backbone(img))
    rel = lambda a, b: ((a - b).abs().max() / b.abs().max()).item()
    assert rel(cam, want["pred_cam"]) <= 1e-4
    for k in ("global_orient", "body_pose", "betas"):
        assert rel(params[k], want["pred_smpl_params"][k]) <= 1e-4, k

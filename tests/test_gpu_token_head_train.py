"""Training TokenHMR's token head on the GPU (csrc/token_head_train.cuh behind thmr_tok_head_train_forward /
thmr_tok_head_backward; tokenhmr_b200.heads.TokenHead), with the release decoder (depth 6, 8 heads, mlp 1024), the
release classifier and tokenizer, and class_pred_layer as made (gain 20, a peaky softmax) and scaled by 0.05: the
forward against the fp64 restatement of SMPLTokenDecoderHead (oracle.tokenhmr_oracle.head_forward) and against a strict
engine, every parameter gradient against fp64 autograd, each upstream path on its own, graph replay and determinism,
batch independence, and a 30-step AdamW fine-tune with the TALS loss whose weights a strict engine then serves.

Bound per output and per parameter gradient: max |x - x64| <= max(4 x the fp32 torch restatement's own error,
1e-5 max |x64|).
"""
import pytest
import torch

from oracle import smpl_oracle as S
from oracle import tokenhmr_oracle as O

pytestmark = pytest.mark.gpu

SCALES = (1.0, 0.05)
TOL_STRICT = 1e-4


@pytest.fixture(scope="module")
def setup(cuda_dev):
    from tokenhmr_b200 import synth
    from tokenhmr_b200.config import tiny_config
    from tokenhmr_b200.engine import TokenHMREngine
    cfg = tiny_config(vit_depth=2)
    sd, smpl = synth.make_state_dict(cfg), synth.make_smpl(cfg)
    strict = TokenHMREngine(cfg, sd, smpl, device=cuda_dev, use_cuda_graph=False, strict=True)
    return cfg, sd, smpl, strict


def _scaled(sd, scale):
    out = dict(sd)
    out["smpl_head.decpose.class_pred_layer.weight"] = sd["smpl_head.decpose.class_pred_layer.weight"] * scale
    return out


def _clear_of_kinks(sd):
    """The weights with the affine of the two LayerNorms that feed a ReLU (mixer_trans.ff.1, mixer_norm_layer.ff.1) set
    to gamma / 2 and bias +-2 by channel: a pre-activation then crosses zero only where |xhat| > ~4, so none lands
    within fp32 rounding of the kink.  At such an element fp32 and fp64 may take different ReLU branches: the
    gradient then differs by that element's whole contribution.  That is a property of fp32, not an error of the
    kernels, and it is what broke the bound at B = 129 / 130 with the weights as made (a pre-activation of 2.6e-7 in
    mixer_trans, 3.8e-7 in mixer_norm_layer).  Both signs occur in every channel, so both ReLU branches stay tested."""
    out = dict(sd)
    for ln in ("smpl_head.decpose.mixer_trans.ff.1", "smpl_head.decpose.mixer_norm_layer.ff.1"):
        g = torch.Generator().manual_seed(len(ln))
        n = sd[ln + ".bias"].numel()
        out[ln + ".weight"] = sd[ln + ".weight"] * 0.5
        out[ln + ".bias"] = torch.where(torch.rand(n, generator=g) < 0.5, -2.0, 2.0)
    return out


def _kink_margin(sd, feats, cfg):
    """min |pre-activation| / max |pre-activation| over the two classifier ReLUs, in fp64."""
    import torch.nn.functional as F
    seen = []
    real = F.relu

    def spy(x, *a, **k):
        if x.shape[-1] in (cfg.cls_hidden, cfg.token_num * cfg.cls_hidden) and x.dim() in (2, 3) and \
                x.shape[-2:] != (cfg.tok_width, cfg.token_num):
            seen.append((x.detach().abs().min() / x.detach().abs().max()).item())
        return real(x, *a, **k)

    O.F.relu = spy
    try:
        with torch.no_grad():
            O.classifier_logits_softmax({k: v.to(feats.device, torch.float64) for k, v in sd.items()
                                         if k.startswith("smpl_head.decpose.")},
                                        O.decoder_forward({k: v.to(feats.device, torch.float64) for k, v in sd.items()
                                                           if k.startswith("smpl_head.transformer.")},
                                                          feats.double().flatten(2).transpose(1, 2), cfg,
                                                          O.Numerics(False)), cfg, O.Numerics(False))
    finally:
        O.F.relu = real
    assert len(seen) == 2, seen
    return min(seen)


def _feats(cfg, B, seed, dev):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(B, cfg.vit_dim, cfg.grid_h, cfg.grid_w, generator=g).to(dev)


def _upstream(cfg, B, seed, dev):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(B, 24, 3, 3, generator=g).to(dev), torch.randn(B, 10, generator=g).to(dev),
            torch.randn(B, 3, generator=g).to(dev),
            torch.randn(B, cfg.token_num, cfg.token_class_num, generator=g).to(dev))


def _restated(sd, feats, cfg, dtype):
    """SMPLTokenDecoderHead.forward restated in `dtype` with autograd: (leaf state dict, outputs)."""
    leaves = {k: v.to(feats.device, dtype).clone().requires_grad_(k.startswith("smpl_head.") and "init_" not in k)
              for k, v in sd.items() if k.startswith(("smpl_head.", "tokenizer."))}
    params, cam, aux = O.head_forward(leaves, feats.to(dtype).flatten(2).transpose(1, 2), cfg, O.Numerics(False))
    rot = torch.cat([params["global_orient"], params["body_pose"]], 1)
    return leaves, {"rotmats": rot, "betas": params["betas"], "cam": cam, "pose6d": aux["pred_body_pose_6d"],
                    "cls": aux["cls_logits_softmax"]}


def _loss(out, up):
    return sum((out[k] * u.to(out[k].dtype)).sum() for k, u in zip(("rotmats", "betas", "cam", "cls"), up)
               if u is not None)


def _ref_grads(leaves, out, up):
    names = [k for k, v in leaves.items() if v.requires_grad]
    gs = torch.autograd.grad(_loss(out, up), [leaves[k] for k in names], allow_unused=True)
    return {k[len("smpl_head."):]: (torch.zeros_like(leaves[k]) if g is None else g) for k, g in zip(names, gs)}


def _run(head, feats, up):
    """One CUDA forward + backward: (gradients by name, outputs)."""
    head.zero_grad(set_to_none=True)
    params, cam, lst = head(feats)
    out = {"rotmats": torch.cat([params["global_orient"], params["body_pose"]], 1), "betas": params["betas"],
           "cam": cam, "cls": lst["cls_logits_softmax"]}
    _loss(out, up).backward()
    return {k: p.grad.clone() for k, p in head.named_parameters()}, {k: v.detach() for k, v in out.items()}


def _ratio(got, ref64, ref32):
    """(error / bound, error, the fp32 restatement's error, max |ref64|)"""
    scale = ref64.abs().max().item()
    err = (got.double() - ref64).abs().max().item()
    own = (ref32.double() - ref64).abs().max().item()
    return err / max(max(4 * own, 1e-5 * scale), 1e-300), err, own, scale


def _within(got, ref64, ref32, what):
    r = _ratio(got, ref64, ref32)
    assert r[0] <= 1.0, (what, *r)
    return r[0]


@pytest.mark.parametrize("scale", SCALES)
@pytest.mark.parametrize("B", [1, 5, 48, 130])
def test_forward_matches_fp64_restatement(setup, cuda_dev, B, scale):
    from tokenhmr_b200.heads import _TokHeadFn, TokenHead
    cfg, sd, _, _ = setup
    sd = _scaled(sd, scale)
    head = TokenHead(cfg, sd, cuda_dev)
    feats = _feats(cfg, B, B, cuda_dev)
    with torch.no_grad():
        params, cam, lst = head(feats)
        p6, *_ = _TokHeadFn.apply(head, False, feats, *head._params())
        _, r64 = _restated(sd, feats, cfg, torch.float64)
        _, r32 = _restated(sd, feats, cfg, torch.float32)
    got = {"rotmats": torch.cat([params["global_orient"], params["body_pose"]], 1), "betas": params["betas"],
           "cam": cam, "pose6d": p6, "cls": lst["cls_logits_softmax"]}
    assert tuple(got["cls"].shape) == (B, 160, 2048) and tuple(got["rotmats"].shape) == (B, 24, 3, 3)
    assert torch.equal(lst["body_pose"], params["body_pose"]) and torch.equal(lst["cam"], cam)
    worst = max(_within(got[k], r64[k], r32[k], k) for k in got)
    print(f"B={B} scale={scale}: worst output error / bound = {worst:.2f}")


@pytest.mark.parametrize("scale", SCALES)
def test_forward_matches_the_strict_engine(setup, scale):
    """head(strict.backbone(img)) against a strict engine's own forward: both see the same features."""
    from tokenhmr_b200 import synth
    from tokenhmr_b200.engine import TokenHMREngine
    from tokenhmr_b200.heads import TokenHead
    cfg, sd, smpl, strict = setup
    if scale != 1.0:
        strict = TokenHMREngine(cfg, _scaled(sd, scale), smpl, device=strict.device, use_cuda_graph=False, strict=True)
    img = synth.make_images(4, cfg, seed=7)
    head = TokenHead(cfg, _scaled(sd, scale), strict.device)
    with torch.no_grad():
        params, cam, lst = head(strict.backbone(img))
    want = strict({"img": img})
    rel = lambda a, b: ((a - b).abs().max() / b.abs().max()).item()
    assert rel(cam, want["pred_cam"]) <= TOL_STRICT
    assert rel(lst["cls_logits_softmax"], want["cls_logits_softmax"]) <= TOL_STRICT
    for k in ("global_orient", "body_pose", "betas"):
        assert rel(params[k], want["pred_smpl_params"][k]) <= TOL_STRICT, k


@pytest.mark.parametrize("scale", SCALES)
@pytest.mark.parametrize("B", [1, 5, 48, 130])
def test_gradients_match_fp64_autograd(setup, cuda_dev, B, scale):
    from tokenhmr_b200.heads import TokenHead
    cfg, sd, _, _ = setup
    sd = _clear_of_kinks(_scaled(sd, scale))
    head = TokenHead(cfg, sd, cuda_dev)
    feats = _feats(cfg, B, 100 + B, cuda_dev)
    assert _kink_margin(sd, feats, cfg) > 1e-6            # no ReLU input within fp32 rounding of zero
    up = _upstream(cfg, B, 200 + B, cuda_dev)
    got, _ = _run(head, feats, up)
    l64, r64 = _restated(sd, feats, cfg, torch.float64)
    g64 = _ref_grads(l64, r64, up)
    del l64, r64
    l32, r32 = _restated(sd, feats, cfg, torch.float32)
    g32 = _ref_grads(l32, r32, up)
    assert set(got) == set(g64) and set(head.state_dict()) == set(g64) | {"init_body_pose", "init_betas", "init_cam"}
    ratios = {k: _ratio(got[k], g64[k], g32[k]) for k in g64}
    over = {k: r for k, r in ratios.items() if r[0] > 1.0}
    worst = max(ratios.items(), key=lambda kv: kv[1][0])
    print(f"B={B} scale={scale}: worst gradient error / bound = {worst[1][0]:.2f} ({worst[0]}); over: {over}")
    assert not over, over
    for l in range(cfg.dec_depth):
        assert not got[f"transformer.transformer.layers.{l}.0.fn.to_qkv.weight"][:2 * cfg.dec_inner].any()
    assert not got["transformer.to_token_embedding.weight"].any()


_READOUTS = ("decpose_grot.", "decpose_hands.", "decshape.", "deccam.")


def _path(cfg, B, dev, which):
    """Upstream gradients that reach the head through one path only."""
    rot, betas, cam, cls = _upstream(cfg, B, 7, dev)
    z = torch.zeros_like
    if which == "cls":
        return None, None, None, cls
    if which == "body":
        r = z(rot)
        r[:, 1:22] = rot[:, 1:22]
        return r, None, None, None
    if which == "rot0":
        r = z(rot)
        r[:, 0] = rot[:, 0]
        return r, None, None, None
    if which == "hands":
        r = z(rot)
        r[:, 22:] = rot[:, 22:]
        return r, None, None, None
    return (None, betas, None, None) if which == "betas" else (None, None, cam, None)


@pytest.mark.parametrize("scale", SCALES)
@pytest.mark.parametrize("which", ["cls", "body", "rot0", "hands", "betas", "cam"])
def test_each_path_on_its_own(setup, cuda_dev, which, scale):
    """One upstream gradient at a time: the parameters it reaches match fp64; those it does not get exact zeros."""
    from tokenhmr_b200.heads import TokenHead
    cfg, sd, _, _ = setup
    sd = _clear_of_kinks(_scaled(sd, scale))
    B = 5
    head = TokenHead(cfg, sd, cuda_dev)
    feats = _feats(cfg, B, 31, cuda_dev)
    assert _kink_margin(sd, feats, cfg) > 1e-6
    up = _path(cfg, B, cuda_dev, which)
    got, _ = _run(head, feats, up)
    l64, r64 = _restated(sd, feats, cfg, torch.float64)
    g64 = _ref_grads(l64, r64, up)
    l32, r32 = _restated(sd, feats, cfg, torch.float32)
    g32 = _ref_grads(l32, r32, up)
    own = {"rot0": "decpose_grot.", "hands": "decpose_hands.", "betas": "decshape.", "cam": "deccam."}
    for k in got:
        if k.startswith(_READOUTS):
            reached = own.get(which) is not None and k.startswith(own[which])
        elif k.startswith("decpose."):
            reached = which in ("cls", "body")
        else:
            reached = True
        if k == "transformer.to_token_embedding.weight":   # its input is zero: never reached
            reached = False
        if reached:
            assert got[k].any(), k
            _within(got[k], g64[k], g32[k], k)
        else:
            assert not got[k].any(), k


def test_graph_replay_equals_eager_bit_for_bit(setup, cuda_dev):
    from tokenhmr_b200.heads import TokenHead
    cfg, sd, _, _ = setup
    head = TokenHead(cfg, _scaled(sd, 0.05), cuda_dev)
    B = 6
    feats = _feats(cfg, B, 11, cuda_dev)
    up = _upstream(cfg, B, 12, cuda_dev)
    e1 = _run(head, feats, up)
    e2 = _run(head, feats, up)
    for k in e1[0]:
        assert torch.equal(e1[0][k], e2[0][k]), k
    for k in e1[1]:
        assert torch.equal(e1[1][k], e2[1][k]), k
    static_feats = feats.clone()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        _run(head, static_feats, up)                     # warm-up on the capture stream
    torch.cuda.current_stream().wait_stream(s)
    head.zero_grad(set_to_none=True)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        params, cam, lst = head(static_feats)
        out = {"rotmats": torch.cat([params["global_orient"], params["body_pose"]], 1), "betas": params["betas"],
               "cam": cam, "cls": lst["cls_logits_softmax"]}
        _loss(out, up).backward()
    for _ in range(2):
        g.replay()
        torch.cuda.synchronize()
        for k, p in head.named_parameters():
            assert torch.equal(p.grad, e1[0][k]), k
        for k in out:
            assert torch.equal(out[k], e1[1][k]), k


def test_batch_independence_and_nothing_kept_under_no_grad(setup, cuda_dev):
    """Row b's outputs and its own gradient do not depend on the other rows; under no_grad the call keeps nothing."""
    from tokenhmr_b200.heads import TokenHead
    cfg, sd, _, _ = setup
    head = TokenHead(cfg, _scaled(sd, 0.05), cuda_dev)
    feats = _feats(cfg, 5, 21, cuda_dev)
    up = _upstream(cfg, 5, 22, cuda_dev)
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated()
    with torch.no_grad():
        p_all, cam_all, l_all = head(feats)
        assert cam_all.grad_fn is None and l_all["cls_logits_softmax"].grad_fn is None
        p_one, cam_one, l_one = head(feats[2:3].contiguous())
    torch.testing.assert_close(cam_one, cam_all[2:3], rtol=0, atol=1e-6)
    torch.testing.assert_close(p_one["body_pose"], p_all["body_pose"][2:3], rtol=0, atol=1e-6)
    torch.testing.assert_close(l_one["cls_logits_softmax"], l_all["cls_logits_softmax"][2:3], rtol=0, atol=1e-6)
    held = sum(t.numel() * 4 for t in (p_all["body_pose"], p_all["betas"], cam_all, l_all["cls_logits_softmax"],
                                        p_one["body_pose"], p_one["betas"], cam_one, l_one["cls_logits_softmax"]))
    assert torch.cuda.memory_allocated() - before <= held + (4 << 20)   # outputs only: no workspace was kept
    del p_all, cam_all, l_all, p_one, cam_one, l_one
    other = feats.clone()
    other[[0, 1, 3, 4]] = _feats(cfg, 4, 23, cuda_dev)
    only_b = tuple(torch.zeros_like(u) for u in up)
    for z, u in zip(only_b, up):
        z[2] = u[2]
    ga, _ = _run(head, feats, only_b)
    gb, _ = _run(head, other, only_b)
    for k in ga:
        scale = ga[k].abs().max().item()
        assert (ga[k] - gb[k]).abs().max().item() <= 1e-6 * max(scale, 1e-30) + 1e-30, k


def test_rejections(setup, cuda_dev):
    from tokenhmr_b200._lib import ThmrError
    from tokenhmr_b200.heads import TokenHead
    cfg, sd, _, _ = setup
    head = TokenHead(cfg, sd, cuda_dev)
    assert set(head.state_dict()) == {k[len("smpl_head."):] for k in sd if k.startswith("smpl_head.")}
    assert not any(n.startswith("tokenizer") or n == "_tokenizer" for n, _ in head.named_parameters())
    f = _feats(cfg, 2, 0, cuda_dev)
    for bad, msg in ((f[:, :, :, :6], "must be"), (f.double(), "float32"), (f.cpu(), "features on"),
                     (f.transpose(2, 3).contiguous().transpose(2, 3), "contiguous"),
                     (f.clone().requires_grad_(True), "not built")):
        with pytest.raises(ThmrError, match=msg):
            head(bad)
    bad_sd = dict(sd)
    del bad_sd["tokenizer.decoder.decoder.15.bias"]
    with pytest.raises(ThmrError, match="no tokenizer.decoder.decoder.15.bias"):
        TokenHead(cfg, bad_sd, cuda_dev)
    bad_sd = dict(sd)
    bad_sd["smpl_head.decpose.mixer_head.0.layernorm1.weight"] = torch.ones(32)
    with pytest.raises(ThmrError, match="mixer_head.0.layernorm1.weight has shape"):
        TokenHead(cfg, bad_sd, cuda_dev)


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
        self.fixed = {k: v.to(dev) for k, v in sd.items() if "init_" in k or k.startswith("tokenizer.")}

    def forward(self, feats):
        sd = {"smpl_head." + k.replace("/", "."): v for k, v in self.p.items()}
        sd.update(self.fixed)
        params, cam, _ = O.head_forward(sd, feats.flatten(2).transpose(1, 2), self.cfg, O.Numerics(False))
        return params, cam


def test_fine_tune_with_adamw_and_serve_the_weights(setup, cuda_dev):
    from tokenhmr_b200 import synth
    from tokenhmr_b200.engine import TokenHMREngine
    from tokenhmr_b200.heads import TokenHead
    from tokenhmr_b200.losses import TokenHMRLoss, differentiable_tail
    cfg, sd, smpl, strict = setup
    # class_pred_layer scaled so that the body pose trains through the classifier (at gain 20 its softmax starves it),
    # and no ReLU input at the kink, where fp32 and fp64 (and so the two runs) may branch differently
    sd = _clear_of_kinks(_scaled(sd, 0.05))
    B = 8
    img = synth.make_images(B, cfg, seed=41)
    feats = strict.backbone(img).detach()
    batch = _fine_tune_batch(strict, cfg, B, cuda_dev)
    crit = TokenHMRLoss({"MODEL": {"LOOSE_SUP": True, "LOOSE_WEIGHT": 0.1},
                         "LOSS_WEIGHTS": {"KEYPOINTS_2D": 0.01, "KEYPOINTS_3D": 0.05, "GLOBAL_ORIENT": 0.001,
                                          "BODY_POSE": 0.001, "BETAS": 0.0005}})
    head = TokenHead(cfg, sd, cuda_dev)
    ref = _TorchHead(sd, cfg, cuda_dev)
    kw = dict(lr=2e-5, weight_decay=1e-4)
    opt, opt_ref = torch.optim.AdamW(head.parameters(), **kw), torch.optim.AdamW(ref.parameters(), **kw)
    losses, ref_losses = [], []
    steps = 30
    for step in range(steps):
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
            (ref_losses if is_ref else losses).append(loss.item())
    print("loss", losses[0], "->", losses[-1], "; torch restatement", ref_losses[0], "->", ref_losses[-1])
    # 30 steps do not halve this loss for either implementation: the fp32 torch restatement also ends at ~0.53-0.55 of
    # its first value, and no learning rate from 1e-5 to 5e-4 reaches 0.5.  The two runs' loss values are not compared:
    # TALS gates each sample on a keypoint-error threshold, so the loss jumps where a sample crosses it.  Parity is
    # asserted on the parameters below, at the bound the regression head's fine-tune uses.
    assert losses[-1] < 0.6 * losses[0], losses
    ours = dict(head.named_parameters())
    largest = max(p.abs().max().item() for p in ref.p.values())
    drift = {k.replace("/", "."): (ours[k.replace("/", ".")] - p).abs().max().item() for k, p in ref.p.items()}
    print("largest |param|", largest, "worst drift from the torch restatement", max(drift.items(), key=lambda kv: kv[1]))
    for name, d in drift.items():
        assert d <= 1e-4 * largest, (name, d)
    tuned = dict(sd)
    tuned.update({"smpl_head." + k: v.detach().cpu() for k, v in head.state_dict().items()})
    served = TokenHMREngine(cfg, tuned, smpl, device=cuda_dev, use_cuda_graph=False, strict=True)
    want = served({"img": img})
    with torch.no_grad():
        params, cam, _ = head(served.backbone(img))
    rel = lambda a, b: ((a - b).abs().max() / b.abs().max()).item()
    assert rel(cam, want["pred_cam"]) <= TOL_STRICT
    for k in ("global_orient", "body_pose", "betas"):
        assert rel(params[k], want["pred_smpl_params"][k]) <= TOL_STRICT, k

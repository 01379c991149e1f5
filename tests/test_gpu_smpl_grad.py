"""Gradients of the SMPL stage (csrc/smpl_grad.cuh behind thmr_smpl_backward / thmr_lbs_backward): against fp64
torch.autograd through oracle.smpl_oracle on the body-model variants of test_gpu_smpl_kernels.py, bitwise
reproducibility, the autograd Functions of SMPLModel and model.smpl, and SMPLifyInv(model.smpl) against the fp64
reference run stored in tests/golden/smplify_inv.npz.

Gradient bound (per pose and per gradient tensor): max |g - g64| <= GRAD_TOL * max |g64|.  The backward is fp32
throughout except for v_posed, which it recomputes with the forward's split-fp16 blend GEMM (~2^-21 relative), and its
longest sums are the 20 670-term contraction of the v_posed cotangent with the blend basis (32 split-K partials of
<= 646 fused terms, summed in order) and the per-joint skinning sums over up to 6890 vertices (per-block lists of
<= 1024 terms, then 27 block partials).  With random unit cotangents such a sum's rounding error grows like
sqrt(n) u of the sum of |terms|, and the largest gradient entries are sums of like-signed terms, so errors of a few
1e-6 of max |g64| are expected.  Measured on an H100 80GB HBM3 (700 W) over every variant, batch and cotangent below:
at most 3.2e-6 (axis-angle lbs, both cotangents); 1e-4 leaves a factor of 30.

SMPLifyInv free-running, measured on the same card: per-iteration loss within 1.3e-7 relative of the fp64 reference in
both cases, final reprojection loss within 3.7e-7 and joints within 9.5e-7; the bounds (1e-4 on the first five losses,
1e-3 at the end) leave room for Adam's sign-like first steps to take a different branch on a near-zero gradient entry.
"""
import pytest
import torch

from oracle import smpl_oracle as S
from tokenhmr_b200.config import SMPL_TO_OPENPOSE

pytestmark = pytest.mark.gpu

J = 24
GRAD_TOL = 1e-4
VARIANTS = ["base", "w6", "w12", "nb7", "noextra", "V1003"]
BATCHES = [1, 17, 255, 256, 257, 513]
COTANGENTS = ["verts", "joints", "both"]


def _weights_with(V, k, seed):
    g = torch.Generator().manual_seed(seed)
    joints = torch.rand(V, J, generator=g).argsort(1)[:, :k]
    w = torch.zeros(V, J).scatter_(1, joints, torch.rand(V, k, generator=g) + 0.05)
    return w / w.sum(1, keepdim=True)


def _variant(name):
    from tokenhmr_b200 import synth
    from tokenhmr_b200.config import release_config, tiny_config
    if name == "V1003":
        return synth.make_smpl(tiny_config(num_verts=1003))
    smpl = synth.make_smpl(release_config())
    if name in ("w6", "w12"):
        smpl["lbs_weights"] = _weights_with(6890, int(name[1:]), 5)
    elif name == "nb7":
        smpl["shapedirs"] = smpl["shapedirs"][..., :7].contiguous()
    elif name == "noextra":
        del smpl["joint_regressor_extra"]
    return smpl


@pytest.fixture(scope="module")
def models(cuda_dev):
    from tokenhmr_b200 import ops
    cache = {}

    def get(name):
        if name not in cache:
            smpl = _variant(name)
            s64 = {k: (v.cuda().double() if v.is_floating_point() else v.cuda()) for k, v in smpl.items()}
            cache[name] = (s64, ops.SMPLModel(smpl, cuda_dev))
        return cache[name]
    return get


def _oracle_wrapper(s64, rot, betas):
    """The SMPL wrapper's forward in fp64 (25 mapped joints only without the extra regressor)."""
    if "joint_regressor_extra" in s64:
        return S.smpl_forward(s64, rot[:, :1], rot[:, 1:], betas, dtype=torch.float64)
    verts, joints = S.lbs(betas, rot, s64["v_template"], s64["shapedirs"], s64["posedirs"], s64["J_regressor"],
                          s64["parents"], s64["lbs_weights"], pose2rot=False)
    j45 = torch.cat([joints, verts[:, s64["extra_vertex_ids"]]], 1)
    return verts, j45[:, torch.tensor(SMPL_TO_OPENPOSE)]


def _inputs(B, nb, seed):
    g = torch.Generator().manual_seed(seed)
    aa = 0.6 * torch.randn(B, J, 3, generator=g)
    aa[0, :3] = 0.0                      # exactly-zero axis-angle rows (root included)
    aa[-1, 7] = 0.0
    betas = 2 * torch.randn(B, nb, generator=g)
    betas[::4] = 60 * (2 * torch.rand(betas[::4].shape, generator=g) - 1)
    betas[0, 0], betas[-1, -1] = 60.0, -60.0
    return aa.cuda(), betas.cuda()


def _cotangents(kind, B, V, nj, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    gv = torch.randn(B, V, 3, device="cuda", generator=g) if kind in ("verts", "both") else None
    gj = torch.randn(B, nj, 3, device="cuda", generator=g) if kind in ("joints", "both") else None
    return gv, gj


def _within(name, got, ref, worst):
    """Per pose: max |got - ref| <= GRAD_TOL * max |ref|."""
    B = ref.shape[0]
    err = (got.double() - ref).reshape(B, -1).abs().amax(1)
    scale = ref.reshape(B, -1).abs().amax(1)
    ratio = (err / scale.clamp_min(1e-300)).max().item()
    worst[name] = max(worst.get(name, 0.0), ratio)
    assert torch.isfinite(got).all(), name
    assert (err <= GRAD_TOL * scale).all(), f"{name}: worst err/max|g64| {ratio:.3g}"


def _vjp64(outs, ins, gv, gj):
    terms = [(o * c.double()).sum() for o, c in zip(outs, (gv, gj)) if c is not None]
    return torch.autograd.grad(sum(terms), ins, retain_graph=True, allow_unused=True)


@pytest.mark.parametrize("B", BATCHES)
@pytest.mark.parametrize("variant", VARIANTS)
def test_backward_vs_fp64_autograd(models, variant, B):
    """thmr_smpl_backward (rotation matrices, 25 + n_extra joints) and thmr_lbs_backward (pose2rot 1 and 0, the 24
    J_transformed joints) against fp64 autograd through the oracle, for vertex-only, joint-only and both cotangents."""
    s64, m = models(variant)
    nb, V = m.num_betas, m.num_verts
    nj = 25 + m.n_extra
    seed = B + 1000 * VARIANTS.index(variant)
    aa, betas = _inputs(B, nb, seed)
    worst = {}
    with torch.device("cuda"):
        rot32 = S.batch_rodrigues(aa.double().reshape(-1, 3)).view(B, J, 3, 3).float()
        # wrapper forward on rotation matrices
        r64, b64 = rot32.double().requires_grad_(), betas.double().requires_grad_()
        fwd64 = _oracle_wrapper(s64, r64, b64)
        # lbs, axis-angle and rotation matrices
        a64, bl64 = aa.double().requires_grad_(), betas.double().requires_grad_()
        lbs_aa = S.lbs(bl64, a64.reshape(B, -1), s64["v_template"], s64["shapedirs"], s64["posedirs"],
                       s64["J_regressor"], s64["parents"], s64["lbs_weights"], pose2rot=True)
        rr64, br64 = rot32.double().requires_grad_(), betas.double().requires_grad_()
        lbs_rm = S.lbs(br64, rr64, s64["v_template"], s64["shapedirs"], s64["posedirs"], s64["J_regressor"],
                       s64["parents"], s64["lbs_weights"], pose2rot=False)
        for k, kind in enumerate(COTANGENTS):
            gv, gj = _cotangents(kind, B, V, nj, seed + k)
            g_rot, g_b = m.smpl_backward(rot32, betas, gv, gj)
            want_rot, want_b = _vjp64(fwd64, (r64, b64), gv, gj)
            _within(f"smpl rot {kind}", g_rot, want_rot, worst)
            _within(f"smpl betas {kind}", g_b, want_b, worst)
            gj24 = None if gj is None else gj[:, :J].contiguous()
            for pose2rot, pose, outs, ins in ((True, aa, lbs_aa, (a64, bl64)), (False, rot32, lbs_rm, (rr64, br64))):
                g_pose, g_b = m.lbs_backward(betas, pose, pose2rot, gv, gj24)
                want_pose, want_b = _vjp64(outs, ins, gv, gj24)
                _within(f"lbs{int(pose2rot)} pose {kind}", g_pose, want_pose.view(g_pose.shape), worst)
                _within(f"lbs{int(pose2rot)} betas {kind}", g_b, want_b, worst)
    print(f"[grad] {variant} B={B} worst err/max|g64|: " + ", ".join(f"{k} {v:.2e}" for k, v in worst.items()))


def test_backward_is_bitwise_reproducible(models):
    s64, m = models("base")
    B = 300
    aa, betas = _inputs(B, m.num_betas, 7)
    rot = _rot32(aa)
    gv, gj = _cotangents("both", B, m.num_verts, 25 + m.n_extra, 8)
    a = m.smpl_backward(rot, betas, gv, gj)
    b = m.smpl_backward(rot, betas, gv, gj)
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    a = m.lbs_backward(betas, aa, True, gv, gj[:, :J].contiguous())
    b = m.lbs_backward(betas, aa, True, gv, gj[:, :J].contiguous())
    assert all(torch.equal(x, y) for x, y in zip(a, b))


def _rot32(aa):
    with torch.device("cuda"):
        return S.batch_rodrigues(aa.double().reshape(-1, 3)).view(aa.shape[0], J, 3, 3).float().contiguous()


def test_autograd_functions_equal_direct_abi(models):
    """torch.autograd.grad through SMPLModel.forward, .lbs and model.smpl(...) gives the direct ABI result bit for bit;
    without a grad-requiring input (or under no_grad) the outputs are the plain forward's, with no grad_fn."""
    from tokenhmr_b200._lib import ThmrError
    from tokenhmr_b200.engine import _SmplFacade
    s64, m = models("base")
    B = 33
    aa, betas = _inputs(B, m.num_betas, 9)
    rot = _rot32(aa)
    gv, gj = _cotangents("both", B, m.num_verts, 25 + m.n_extra, 10)
    v0, j0 = m.forward(rot[:, :1], rot[:, 1:], betas)
    assert v0.grad_fn is None and j0.grad_fn is None
    go, bp, bt = rot[:, :1].clone().requires_grad_(), rot[:, 1:].clone().requires_grad_(), betas.clone().requires_grad_()
    with torch.no_grad():
        v1, j1 = m.forward(go, bp, bt)
    assert v1.grad_fn is None and torch.equal(v1, v0) and torch.equal(j1, j0)
    facade = _SmplFacade(m)
    for call in (lambda: m.forward(go, bp, bt), lambda: tuple(facade(global_orient=go, body_pose=bp, betas=bt))):
        v, j = call()
        assert v.grad_fn is not None and torch.equal(v, v0) and torch.equal(j, j0)
        g_go, g_bp, g_bt = torch.autograd.grad((v * gv).sum() + (j * gj).sum(), (go, bp, bt))
        want_rot, want_b = m.smpl_backward(rot, betas, gv, gj)
        assert torch.equal(torch.cat([g_go, g_bp], 1), want_rot) and torch.equal(g_bt, want_b)
        # vertices unused: its cotangent reaches the kernel as a null pointer
        (g_bp2,) = torch.autograd.grad((call()[1] * gj).sum(), (bp,))
        assert torch.equal(g_bp2, m.smpl_backward(rot, betas, None, gj)[0][:, 1:])
    out = facade(global_orient=go, body_pose=bp, betas=bt, pose2rot=True)      # ignored, as in SMPLLayer
    assert out.vertices.shape == (B, m.num_verts, 3) and out.joints.shape == (B, 44, 3)
    with pytest.raises(ThmrError):
        m.forward(go, bp, bt, pred_cam=torch.ones(B, 3, device="cuda"))
    for pose2rot, pose in ((True, aa), (False, rot)):
        vl0, jl0 = m.lbs(betas, pose, pose2rot=pose2rot)
        p = pose.clone().requires_grad_()
        vl, jl = m.lbs(betas, p, pose2rot=pose2rot)
        assert vl.grad_fn is not None and torch.equal(vl, vl0) and torch.equal(jl, jl0)
        (g_p,) = torch.autograd.grad((vl * gv).sum() + (jl * gj[:, :J]).sum(), (p,))
        assert torch.equal(g_p, m.lbs_backward(betas, pose, pose2rot, gv, gj[:, :J].contiguous())[0])


# ------------------------------------------------------------------------------------------------ SMPLifyInv
@pytest.fixture(scope="module")
def golden(golden_dir):
    import numpy as np
    return np.load(golden_dir / "smplify_inv.npz")


def _g(golden, key):
    return torch.from_numpy(golden[key].copy()).float().cuda()


@pytest.fixture(scope="module")
def smpl_fn(models):
    from tokenhmr_b200.engine import _SmplFacade
    return _SmplFacade(models("base")[1])


@pytest.mark.parametrize("case", ["a", "b"])
def test_smplify_teacher_forced_gradients(golden, models, smpl_fn, case):
    """At each stored iteration's parameters, the body-model gradients of SMPLifyInv's loss through model.smpl are within
    the gradient bound of fp64 autograd through the oracle.

    Both sides get the same loss cotangent on the joints, computed in fp64 from the oracle's joints: the loss's
    sqrt(|r|^2) term has the direction r / |r| as its gradient, and at a joint whose 2D residual r is near zero that
    direction turns a 1e-7 difference in the joints (or in the fp32-stored parameters) into a gradient difference of
    1e-4 and more (measured: up to 1.5e-4 of max |g| with each side's own loss), which is the loss's conditioning, not
    the body model's.  pred_cam_t's gradient passes through no body-model backward and is left to the free-running
    test.  The golden's own gradients (taken at the unrounded fp64 parameters) are printed for comparison."""
    from tokenhmr_b200.fitting import camera_fitting_loss
    s64, _ = models("base")
    margin = float(golden[f"{case}_config"][2])
    betas, focal = _g(golden, f"{case}_betas"), _g(golden, f"{case}_focal_length").double()
    kp2, kp3 = _g(golden, f"{case}_gt_keypoints_2d")[..., :2].double(), _g(golden, f"{case}_gt_keypoints_3d").double()
    worst, vs_golden = {}, {}
    for i in range(int(golden[f"{case}_steps"])):
        go = _g(golden, f"{case}_global_orient_it")[i]
        bp = _g(golden, f"{case}_body_pose_it")[i]
        cam = _g(golden, f"{case}_pred_cam_t_it")[i].double()
        with torch.device("cuda"):
            go64, bp64 = go.double().requires_grad_(), bp.double().requires_grad_()
            _, j64 = S.smpl_forward(s64, go64, bp64, betas.double(), dtype=torch.float64)
            push = torch.sqrt(((j64 - kp3) ** 2).sum(2)).sum(1)
            loss = 4 * camera_fitting_loss(j64, cam, focal, kp2) - push.mean() / 2 + margin
            (cot,) = torch.autograd.grad(loss, j64, retain_graph=True)
            want = torch.autograd.grad(loss, (go64, bp64))
        go, bp = go.requires_grad_(), bp.requires_grad_()
        joints = smpl_fn(global_orient=go, body_pose=bp, betas=betas).joints
        got = torch.autograd.grad(joints, (go, bp), grad_outputs=cot.float())
        for name, g, w in zip(("global_orient", "body_pose"), got, want):
            _within(name, g, w, worst)
            gold = torch.from_numpy(golden[f"{case}_grad_{name}_it"][i]).double().cuda()
            vs_golden[name] = max(vs_golden.get(name, 0.0), ((w - gold).abs().max() / gold.abs().max()).item())
    print(f"[smplify {case}] teacher-forced worst err/max|g64|: " + ", ".join(f"{k} {v:.2e}" for k, v in worst.items())
          + "; fp64 at the stored parameters vs the golden's gradients: "
          + ", ".join(f"{k} {v:.2e}" for k, v in vs_golden.items()))


@pytest.mark.parametrize("case", ["a", "b"])
def test_smplify_free_running(golden, smpl_fn, case):
    """The whole fit on the GPU: the first 5 iterations' loss within 1e-4 relative of the fp64 reference's, the final
    reprojection loss and joints within 1e-3, the break at the golden's iteration, and the caller's tensors updated in
    place."""
    from tokenhmr_b200.fitting import SMPLifyInv
    step, iters, margin, f2d, f3d, _ = golden[f"{case}_config"]
    go, bp = _g(golden, f"{case}_global_orient"), _g(golden, f"{case}_body_pose")
    cam = _g(golden, f"{case}_pred_cam_t")
    fit = SMPLifyInv(smpl_fn, step_size=float(step), num_iters=int(iters), margin=float(margin),
                     loss_thresh_f2d=float(f2d), loss_thresh_f3d=float(f3d))
    out = fit(go, bp, _g(golden, f"{case}_betas"), cam, _g(golden, f"{case}_focal_length"),
              _g(golden, f"{case}_gt_keypoints_2d"), _g(golden, f"{case}_gt_keypoints_3d"))
    loss = torch.tensor([float(h[0]) for h in fit.history], dtype=torch.float64)
    want = torch.from_numpy(golden[f"{case}_loss_it"])
    assert len(loss) == len(want)
    rel = ((loss[:5] - want[:5]).abs() / want[:5].abs()).max().item()
    reproj = float(out[7])
    want_reproj = float(golden[f"{case}_reprojection_loss"])
    want_j = torch.from_numpy(golden[f"{case}_joints"])
    j_rel = ((out[1].double().cpu() - want_j).abs().max() / want_j.abs().max()).item()
    print(f"[smplify {case}] loss rel (first 5) {rel:.2e}, all {((loss - want).abs() / want.abs()).max().item():.2e}, "
          f"reprojection rel {abs(reproj - want_reproj) / want_reproj:.2e}, joints rel {j_rel:.2e}")
    assert rel <= 1e-4
    assert abs(reproj - want_reproj) <= 1e-3 * want_reproj
    assert j_rel <= 1e-3
    assert torch.equal(bp.detach(), out[4]) and torch.equal(go.detach(), out[3]) and out[6] is cam

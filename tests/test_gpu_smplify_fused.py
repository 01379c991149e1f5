"""The fused SMPLify-inverse (csrc/smplify.cuh behind thmr_smplify_inv, tokenhmr_b200.fitting.FusedSMPLifyInv): the loss
and cotangent kernel against fp64 autograd, the Adam kernel against torch.optim.Adam bit for bit, the whole fit against
the fp64 reference run in tests/golden/smplify_inv.npz and against SMPLifyInv(model.smpl), the stop semantics,
reproducibility and CUDA-graph capture, the in-place contract and the rejections.

Loss and cotangent bound (per element, U = 2^-24).  The kernel rounds each operation once: p = joint + t, q = p_xy / p_z,
u = (f / 256) q, d = kp - u, |d| through squares, a sum and a square root.  So u carries at most 4U |u| (one rounding
each in p, q, u, plus p_z's rounding entering q), and d at most 4U |u| + U |d|.  The 2D cotangent is
(4/B) (d / |d|) (f / 256) dq/dp: the direction d / |d| moves by at most 2 (4U |u| + U |d|) / |d| plus 3U from its own
roundings, and the chain to p adds at most 6 roundings.  With kp in the sum for safety,
    |err| <= 32 U (1 + (|u|_1 + |kp|_1) / |d|) (4/B) c M  +  16 U (0.5/B),
where c = max focal / 256, M = 1 / |p_z| for x and y and (|q_x| + |q_y|) / |p_z| for z; the second term is the 3D
part's (its residual joint - kp3d is rounded once and its direction has no cancellation beyond that).  pred_cam_t's
cotangent sums the J joints' 2D parts: the sum of their bounds plus J U sum |term|.  The per-sample sums carry
16 U (|u|_1 + |kp|_1 + |d|) per joint plus J U sum |d| for the summation.  Joints whose 2D residual is within
rounding of zero (|d| <= 2^-16 (|u|_1 + |kp|_1)) are excluded as in test_gpu_smpl_grad.py's teacher-forced test: the
direction d / |d| is then set by rounding, not by the loss; they are counted and printed.  A residual of exactly zero
gives NaN, as torch's sqrt backward does.

Fit against SMPLifyInv(model.smpl) (same seeded inputs, 100 iterations, no stop): both run the same body model
kernels; they differ in the loss's and the batch means' summation order (a few ulp of the loss) and in nothing else that
Adam sees, except where that difference flips the sign of a near-zero gradient entry: Adam's first steps are close to
sign steps of size lr, so such an entry can differ by about 2 lr.  Bounds: every iteration's loss within 1e-4 relative,
the final rotations and pred_cam_t within 10 lr absolute, and the final joints within 3e-2 of max |joint|: a change
of delta in every entry of a rotation matrix turns a bone by at most 3 delta of its length, and the bones of a joint's
chain add up to about max |joint|, so 10 lr in the parameters allows 3 x 10 lr = 3e-2.  Measured on one H100 80GB HBM3
(700 W): loss 3.9e-7, parameters 0.79 lr, joints 1.3e-3 at B = 64; 1.9e-7, 0.26 lr and 3.9e-4 at B = 257.
"""
import ctypes

import pytest
import torch

import probe
from oracle import smpl_oracle as S

pytestmark = pytest.mark.gpu

U = 2.0 ** -24


@pytest.fixture(scope="module")
def model(cuda_dev):
    from tokenhmr_b200 import ops, synth
    from tokenhmr_b200.config import release_config
    return ops.SMPLModel(synth.make_smpl(release_config()), cuda_dev)


@pytest.fixture(scope="module")
def facade(model):
    from tokenhmr_b200.engine import _SmplFacade
    return _SmplFacade(model)


def _fit_inputs(B, J, nb, seed):
    """Seeded inputs of the size users run: poses around rest, a camera 45 units away, focal 5000."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    with torch.device("cuda"):
        rot = S.batch_rodrigues(0.3 * torch.randn(B * 24, 3, device="cuda", generator=g)).view(B, 24, 3, 3).float()
    betas = torch.randn(B, nb, device="cuda", generator=g)
    focal = torch.full((B, 2), 5000.0, device="cuda")
    kp2 = torch.cat([0.3 * torch.randn(B, J, 2, device="cuda", generator=g), torch.ones(B, J, 1, device="cuda")], -1)
    kp3 = 0.3 * torch.randn(B, J, 3, device="cuda", generator=g)
    cam = torch.tensor([0.0, 0.0, 45.0], device="cuda").repeat(B, 1) + 0.5 * torch.randn(B, 3, device="cuda",
                                                                                         generator=g)
    return rot[:, :1].contiguous(), rot[:, 1:].contiguous(), betas, cam, focal, kp2, kp3


def _fresh(t):
    return [x.detach().clone() for x in t]


# ------------------------------------------------------------------------------------------------ loss kernel
@pytest.mark.parametrize("B", [1, 17, 64, 257])
def test_loss_kernel_vs_fp64_autograd(cuda_dev, B):
    from tokenhmr_b200.fitting import camera_fitting_loss
    J = 44
    g = torch.Generator(device="cuda").manual_seed(100 + B)
    joints = 0.4 * torch.randn(B, J, 3, device="cuda", generator=g)
    cam = torch.tensor([0.1, -0.2, 40.0], device="cuda") + torch.randn(B, 3, device="cuda", generator=g)
    focal = 5000.0 + 100 * torch.rand(B, 2, device="cuda", generator=g)
    kp3 = 0.4 * torch.randn(B, J, 3, device="cuda", generator=g)
    p = joints + cam[:, None]
    u32 = (focal / 256)[:, None] * (p[..., :2] / p[..., 2:])        # the kernel's fp32 operation sequence
    kp2 = torch.cat([u32 + 0.05 * torch.randn(B, J, 2, device="cuda", generator=g),
                     torch.rand(B, J, 1, device="cuda", generator=g)], -1)
    kp2[0, 3, :2] = u32[0, 3]                                         # a 2D residual of exactly zero
    kp2[-1, 5, :2] = u32[-1, 5] + torch.tensor([3e-7, -2e-7], device="cuda")   # within rounding of zero
    gj = torch.empty(B, J, 3, device="cuda")
    gcam = torch.empty(B, 3, device="cuda")
    part = torch.empty(2, B, device="cuda")
    probe.call("probe_smplify_loss", joints.data_ptr(), cam.data_ptr(), focal.data_ptr(), kp2.data_ptr(),
               kp3.data_ptr(), J, B, gj.data_ptr(), gcam.data_ptr(), part.data_ptr(), None, probe.stream())
    pj2d = torch.empty(B, J, 2, device="cuda")
    part_f = torch.empty(2, B, device="cuda")
    probe.call("probe_smplify_loss", joints.data_ptr(), cam.data_ptr(), focal.data_ptr(), kp2.data_ptr(),
               kp3.data_ptr(), J, B, None, None, part_f.data_ptr(), pj2d.data_ptr(), probe.stream())
    torch.cuda.synchronize()
    assert torch.equal(pj2d, u32), "projection differs from the same fp32 operations in torch"
    assert torch.equal(part_f, part)
    # fp64 autograd of the reference's loss expression on the same fp32 values
    j64, c64 = joints.double().requires_grad_(), cam.double().requires_grad_()
    f64, k2, k3 = focal.double(), kp2[..., :2].double(), kp3.double()
    fit_b = torch.sqrt(((k2 - (f64 / 256)[:, None] * ((j64 + c64[:, None])[..., :2] / (j64 + c64[:, None])[..., 2:]))
                        ** 2).sum(-1)).sum(1)
    push_b = torch.sqrt(((j64 - k3) ** 2).sum(2)).sum(1)
    loss = 4 * camera_fitting_loss(j64, c64, f64, k2) - push_b.mean() / 2 + 20.0
    want_j, want_c = torch.autograd.grad(loss, (j64, c64))
    # magnitudes
    p64 = (j64 + c64[:, None]).detach()
    u64 = (f64 / 256)[:, None] * (p64[..., :2] / p64[..., 2:])
    d64 = k2 - u64
    r2 = d64.norm(dim=-1)
    r3 = (j64.detach() - k3).norm(dim=-1)
    mag = u64.abs().sum(-1) + k2.abs().sum(-1)
    near_zero = r2 <= 2.0 ** -16 * mag
    n_excl = int(near_zero.sum())
    assert n_excl >= (2 if B > 1 else 1)
    assert torch.isnan(gj[0, 3]).all() and torch.isnan(gcam[0]).all(), "exact-zero residual must give autograd's NaN"
    c = (f64 / 256).amax(-1)[:, None]
    pz = p64[..., 2].abs()
    qsum = (p64[..., :2] / p64[..., 2:]).abs().sum(-1)
    cond = 1 + mag / r2.clamp_min(1e-300)
    b2 = 32 * U * cond * (4.0 / B) * c
    bound_j = torch.stack([b2 / pz, b2 / pz, b2 * qsum / pz], -1) + 16 * U * (0.5 / B)
    term2 = (4.0 / B) * c[..., None] * torch.stack([1 / pz, 1 / pz, qsum / pz], -1)
    bound_c = (bound_j - 16 * U * (0.5 / B)).sum(1) + J * U * term2.sum(1)
    keep = ~near_zero
    keep_s = keep.all(1)
    rep = {}
    probe.assert_within(f"grad_joints B={B}", gj[keep], want_j[keep], bound_j[keep], rep)
    if bool(keep_s.any()):
        probe.assert_within(f"grad_cam B={B}", gcam[keep_s], want_c[keep_s], bound_c[keep_s], rep)
    probe.assert_within(f"fit2D_b B={B}", part[0], fit_b.detach(), 16 * U * (mag + r2).sum(1) + J * U * r2.sum(1), rep)
    probe.assert_within(f"push3D_b B={B}", part[1], push_b.detach(),
                        16 * U * (j64.detach().abs().sum(-1) + k3.abs().sum(-1) + r3).sum(1) + J * U * r3.sum(1), rep)
    print(f"[smplify loss] B={B}: {n_excl} joints with a 2D residual within rounding of zero excluded "
          f"({int((~keep_s).sum())} samples' pred_cam_t cotangent); worst err/bound "
          + ", ".join(f"{k} {v:.3g}" for k, v in rep.items()))


# ------------------------------------------------------------------------------------------------ Adam kernel
@pytest.mark.parametrize("lr", [1e-3, 0.05])
def test_adam_kernel_equals_torch_adam_bitwise(cuda_dev, lr):
    """20 steps of identical random gradients (magnitudes 1e-6 .. 1e3, some exact zeros) on the three parameter sets:
    every parameter, after every step, bit for bit equal to torch.optim.Adam's default (foreach) CUDA step."""
    B = 64
    g = torch.Generator(device="cuda").manual_seed(7)
    go = torch.randn(B, 1, 3, 3, device="cuda", generator=g)
    bp = torch.randn(B, 23, 3, 3, device="cuda", generator=g)
    cam = torch.randn(B, 3, device="cuda", generator=g) * 10
    params = [bp.clone().requires_grad_(), go.clone().requires_grad_(), cam.clone().requires_grad_()]
    opt = torch.optim.Adam(params, lr=lr, betas=(0.9, 0.999))
    flat = torch.cat([go.flatten(), bp.flatten(), cam.flatten()])
    m, v = torch.zeros_like(flat), torch.zeros_like(flat)
    n1, n2 = go.numel(), go.numel() + bp.numel()
    for step in range(1, 21):
        grads = [torch.randn(t.shape, device="cuda", generator=g)
                 * 10 ** (9 * torch.rand(t.shape, device="cuda", generator=g) - 6) for t in (bp, go, cam)]
        grads[0].view(-1)[::97] = 0.0
        for t, gr in zip(params, grads):
            t.grad = gr.clone()
        opt.step()
        gflat = torch.cat([grads[1].flatten(), grads[0].flatten(), grads[2].flatten()])
        probe.call("probe_smplify_adam", flat.data_ptr(), m.data_ptr(), v.data_ptr(), gflat.data_ptr(), flat.numel(),
                   step, lr, probe.stream())
        torch.cuda.synchronize()
        for name, got, want in (("global_orient", flat[:n1], params[1]), ("body_pose", flat[n1:n2], params[0]),
                                ("pred_cam_t", flat[n2:], params[2])):
            diff = int((got != want.detach().flatten()).sum())
            assert diff == 0, f"step {step} {name}: {diff} elements differ from torch.optim.Adam"
    print(f"[smplify adam] lr={lr}: 20 steps bit for bit equal to torch.optim.Adam")


# ------------------------------------------------------------------------------------------------ whole fit
@pytest.fixture(scope="module")
def golden(golden_dir):
    import numpy as np
    return np.load(golden_dir / "smplify_inv.npz")


def _g(golden, key):
    return torch.from_numpy(golden[key].copy()).float().cuda()


@pytest.mark.parametrize("case", ["a", "b"])
def test_fit_vs_fp64_golden(golden, facade, case):
    """The bounds of test_gpu_smpl_grad.py::test_smplify_free_running: the first 5 losses within 1e-4 relative of the
    fp64 reference run, the final reprojection loss and joints within 1e-3, the same number of iterations (case b
    stops early)."""
    from tokenhmr_b200.fitting import FusedSMPLifyInv
    step, iters, margin, f2d, f3d, _ = golden[f"{case}_config"]
    go, bp = _g(golden, f"{case}_global_orient"), _g(golden, f"{case}_body_pose")
    cam = _g(golden, f"{case}_pred_cam_t")
    fit = FusedSMPLifyInv(facade, step_size=float(step), num_iters=int(iters), margin=float(margin),
                          loss_thresh_f2d=float(f2d), loss_thresh_f3d=float(f3d))
    out = fit(go, bp, _g(golden, f"{case}_betas"), cam, _g(golden, f"{case}_focal_length"),
              _g(golden, f"{case}_gt_keypoints_2d"), _g(golden, f"{case}_gt_keypoints_3d"))
    loss = torch.tensor([float(h[0]) for h in fit.history], dtype=torch.float64)
    want = torch.from_numpy(golden[f"{case}_loss_it"])
    assert len(loss) == len(want)
    rel = ((loss[:5] - want[:5]).abs() / want[:5].abs()).max().item()
    reproj, want_reproj = float(out[7]), float(golden[f"{case}_reprojection_loss"])
    want_j = torch.from_numpy(golden[f"{case}_joints"])
    j_rel = ((out[1].double().cpu() - want_j).abs().max() / want_j.abs().max()).item()
    print(f"[smplify fused {case}] {len(loss)} iterations; loss rel (first 5) {rel:.2e}, all "
          f"{((loss - want).abs() / want.abs()).max().item():.2e}, reprojection rel "
          f"{abs(reproj - want_reproj) / want_reproj:.2e}, joints rel {j_rel:.2e}")
    assert rel <= 1e-4
    assert abs(reproj - want_reproj) <= 1e-3 * want_reproj
    assert j_rel <= 1e-3
    assert torch.equal(bp.detach(), out[4]) and torch.equal(go.detach(), out[3]) and out[6] is cam


@pytest.mark.parametrize("B", [64, 257])
def test_fit_vs_smplifyinv(model, facade, B):
    """Against SMPLifyInv(model.smpl) on the same seeded inputs, 100 iterations, no stop (bounds: module docstring)."""
    from tokenhmr_b200.fitting import FusedSMPLifyInv, SMPLifyInv
    lr = 1e-3
    inputs = _fit_inputs(B, 25 + model.n_extra, model.num_betas, B)
    a, b = _fresh(inputs), _fresh(inputs)
    ref = SMPLifyInv(facade, step_size=lr, num_iters=100, loss_thresh_f2d=-1.0)
    want = ref(*a)
    fit = FusedSMPLifyInv(facade, step_size=lr, num_iters=100, loss_thresh_f2d=-1.0)
    got = fit(*b)
    assert len(fit.history) == len(ref.history) == 100
    loss = torch.stack([h[0] for h in fit.history]).double()
    want_loss = torch.stack([h[0] for h in ref.history]).double()
    l_rel = ((loss - want_loss).abs() / want_loss.abs()).max().item()
    p_abs = max((x - y).abs().max().item() for x, y in zip((got[3], got[4], got[6]), (want[3], want[4], want[6])))
    j_rel = ((got[1] - want[1]).abs().max() / want[1].abs().max()).item()
    r_rel = abs(float(got[7]) - float(want[7])) / abs(float(want[7]))
    print(f"[smplify fused vs SMPLifyInv] B={B}: loss rel {l_rel:.2e}, parameters abs {p_abs:.2e} "
          f"({p_abs / lr:.3g} lr), joints rel {j_rel:.2e}, reprojection rel {r_rel:.2e}")
    assert l_rel <= 1e-4
    assert p_abs <= 10 * lr
    assert j_rel <= 3 * 10 * lr


def test_stop_semantics(model, facade):
    from tokenhmr_b200.fitting import FusedSMPLifyInv
    B = 5
    inputs = _fit_inputs(B, 25 + model.n_extra, model.num_betas, 3)
    # fires at iteration 0: no step
    x = _fresh(inputs)
    fit = FusedSMPLifyInv(facade, num_iters=20, loss_thresh_f2d=1e30, loss_thresh_f3d=1e30)
    out = fit(*x)
    assert len(fit.history) == 1
    for got, init in zip((x[0], x[1], x[3]), (inputs[0], inputs[1], inputs[3])):
        assert torch.equal(got.detach(), init)
    hist = fit.run(*_fresh(inputs))[8]
    assert torch.equal(hist[1:], torch.zeros_like(hist[1:]))
    # never fires: num_iters entries
    fit = FusedSMPLifyInv(facade, num_iters=7, loss_thresh_f2d=-1.0)
    fit(*_fresh(inputs))
    assert len(fit.history) == 7
    # num_iters = 0: the final forward on the initial parameters
    x = _fresh(inputs)
    fit = FusedSMPLifyInv(facade, num_iters=0)
    out = fit(*x)
    assert fit.history == []
    v, j = model.forward(inputs[0], inputs[1], inputs[2])
    assert torch.equal(out[0], v) and torch.equal(out[1], j) and torch.equal(x[3].detach(), inputs[3])
    from tokenhmr_b200.fitting import camera_fitting_loss
    want = camera_fitting_loss(j.double(), inputs[3].double(), inputs[4].double(), inputs[5][..., :2].double())
    assert abs(float(out[7]) - float(want)) <= 1e-5 * float(want)
    print("[smplify fused] stop at iteration 0, no stop and num_iters = 0 behave as SMPLifyInv")


def test_reproducible_and_graph_capturable(model, facade):
    from tokenhmr_b200.fitting import FusedSMPLifyInv
    B = 33
    inputs = _fit_inputs(B, 25 + model.n_extra, model.num_betas, 11)
    fit = FusedSMPLifyInv(facade, num_iters=30, loss_thresh_f2d=-1.0)
    first = fit.run(*_fresh(inputs))
    second = fit.run(*_fresh(inputs))
    for x, y in zip(first, second):
        assert torch.equal(x, y)
    static = _fresh(inputs)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        fit.run(*static)                                  # warm-up on the side stream, as torch.cuda.graphs advises
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    for t, init in zip(static, inputs):
        t.data.copy_(init)
    with torch.cuda.graph(graph):
        captured = fit.run(*static)
    for t, init in zip(static, inputs):
        t.data.copy_(init)
    graph.replay()
    torch.cuda.synchronize()
    for name, x, y in zip(("vertices", "joints", "pj2ds", "global_orient", "body_pose", "betas", "pred_cam_t",
                           "reprojection_loss", "history", "iters_run"), captured, first):
        assert torch.equal(x, y), f"graph replay differs from the eager call in {name}"
    print("[smplify fused] two calls and a CUDA-graph replay bitwise equal")


def test_in_place_and_rejections(model, facade):
    from tokenhmr_b200 import _lib
    from tokenhmr_b200.fitting import FusedSMPLifyInv
    B = 4
    J = 25 + model.n_extra
    inputs = _fit_inputs(B, J, model.num_betas, 5)
    x = _fresh(inputs)
    ptrs = [t.data_ptr() for t in x]
    v0 = [t._version for t in x]
    fit = FusedSMPLifyInv(model, num_iters=3, loss_thresh_f2d=-1.0)
    out = fit(*x)
    assert [t.data_ptr() for t in x] == ptrs
    assert x[0].requires_grad and x[1].requires_grad and x[3].requires_grad and not x[2].requires_grad
    assert out[6] is x[3] and torch.equal(out[3], x[0].detach()) and torch.equal(out[4], x[1].detach())
    assert not torch.equal(x[1].detach(), inputs[1]) and not torch.equal(x[3].detach(), inputs[3])
    assert all(t._version > v for t, v in zip((x[0], x[1], x[3]), (v0[0], v0[1], v0[3])))
    bad = [
        ("body_pose shape", lambda y: (y[0], y[1][:, :22].contiguous()) + tuple(y[2:])),
        ("J mismatch", lambda y: tuple(y[:5]) + (y[5][:, :J - 1].contiguous(), y[6])),
        ("kp3d J mismatch", lambda y: tuple(y[:6]) + (y[6][:, :J - 1].contiguous(),)),
        ("CPU tensors", lambda y: tuple(t.cpu() for t in y)),
        ("CPU keypoints", lambda y: tuple(y[:5]) + (y[5].cpu(), y[6])),
    ]
    for name, make in bad:
        with pytest.raises(_lib.ThmrError):
            fit(*make(_fresh(inputs)))
    with pytest.raises(_lib.ThmrError):
        FusedSMPLifyInv(lambda **kw: None)
    # the C ABI's own checks: J must be 25 + n_extra, B >= 1, num_iters >= 0
    y = _fresh(inputs)
    outs = [torch.empty(B, model.num_verts, 3, device="cuda"), torch.empty(B, J, 3, device="cuda"),
            torch.empty(B, J, 2, device="cuda"), torch.empty((), device="cuda"), torch.empty(3, 3, device="cuda"),
            torch.empty(1, device="cuda", dtype=torch.int32)]
    ws = torch.empty(_lib.lib().thmr_smplify_workspace_bytes(model.handle, B, 3), device="cuda", dtype=torch.uint8)
    for B_, it, J_ in ((B, 3, J - 1), (0, 3, J), (B, -1, J)):
        d = _lib.SmplifyDesc(B_, it, J_, 1e-3, 20.0, 1.0, 0.0, *[t.data_ptr() for t in (y[0], y[1], y[3], y[2], y[4],
                                                                                         y[5], y[6])],
                             *[t.data_ptr() for t in outs])
        assert _lib.lib().thmr_smplify_inv(model.handle, ctypes.byref(d), ws.data_ptr(), None) == -1
    assert _lib.lib().thmr_smplify_workspace_bytes(model.handle, 0, 3) == 0
    assert _lib.lib().thmr_smplify_workspace_bytes(model.handle, B, -1) == 0

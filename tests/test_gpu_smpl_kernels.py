"""SMPL stage (csrc/smpl_lbs.cuh, driven by smpl_run in csrc/engine.cuh) one kernel at a time, through the test-only
kernel probe, against torch fp64 on the fp32 values each kernel receives: the create-time joint regression and basis
packing, the pose kernel (Rodrigues, split blend feature, kinematic chain), the split-fp16 blend GEMM, every skinning
instantiation and ELL width, and the joints / camera kernel.  Then the product ABI (ops.SMPLModel) on body-model variants
the synthetic model does not cover, against oracle.smpl_oracle in fp64, and the engine's SMPL tail against
SMPLModel.forward.  Bounds are per element and scale-free (probe.assert_within); exact stages are compared with
torch.equal, and every output starts as NaN so that an unwritten element fails."""
import math

import pytest
import torch

import probe
from oracle import smpl_oracle as S
from probe import U32, assert_within
from tokenhmr_b200.config import SMPL_EXTRA_VERTEX_IDS, SMPL_PARENTS, SMPL_TO_OPENPOSE

pytestmark = pytest.mark.gpu

J = 24
PF, PFPAD, BETA0, ONE = 207, 224, 207, 217     # kSmplPF, kSmplPFPad, kSmplFeatBeta, kSmplFeatOne
SCALE = 1024.0                                   # kSplitScale
DEPTH = [0] * J                                  # depth of each joint in the kinematic tree (root 0, deepest 8)
for _i in range(1, J):
    DEPTH[_i] = DEPTH[SMPL_PARENTS[_i]] + 1

# Blend GEMM (split fp16, K' = 3 * 224 = 672 columns: hi.hi, then lo.hi, then hi.lo), per product f.w of the unscaled
# fp32 operands: hi + lo keeps 22 significand bits of each scaled operand (|a - hi - lo| <= 2^-22 |a|) and the dropped
# lo.lo term is <= 2^-22 |f||w|: 3 * 2^-22 of sum |f||w|.  Inside one 16-product tensor-core step the products are
# aligned and truncated at 2^-23 of the largest: 3 * 2^-23 more over the three column groups.  Together
# 1.125 * 2^-20 < 2^-19.
C_SPLIT = 2.0 ** -19
# The wgmma fp32 accumulator truncates the running sum P_s at each of the 42 16-column steps by up to one ulp, 2^-23 |P_s|,
# with errors of one sign: 2^-23 sum_s |P_s| over the kernel's column order (_blend_bound).
C_TRUNC = 2.0 ** -23
# fp16-subnormal floor: an operand is split after scaling by 2^10, and a lo (or hi) below fp16's smallest normal 2^-14 is
# rounded on the subnormal grid 2^-24, i.e. off by up to 2^-25 absolute, 2^-35 in unscaled units.  Per product that is
# 2^-35 (|w| + |f|): FLOOR * (sum_k |w_k| + sum_k |f_k|) per output.  (Strict mode's 2^-29 / 2^-33 are the same rule for
# its 2^4 / 2^8 scales.)
FLOOR = 2.0 ** -35


@pytest.fixture(autouse=True)
def _flags(cuda_dev, built_lib):
    yield
    assert probe.flags() == 0, "probe device flags set"
    assert built_lib.thmr_check_device_flags() == 0, built_lib.thmr_last_error()


def _nan(*shape, dtype=torch.float32):
    return torch.full(shape, float("nan"), dtype=dtype, device="cuda")


def _wide(shape, lo_exp: float, hi_exp: float, g):
    """Random signs, magnitudes log-uniform in [2^lo_exp, 2^hi_exp)."""
    e = lo_exp + (hi_exp - lo_exp) * torch.rand(shape, device="cuda", generator=g)
    s = torch.where(torch.rand(shape, device="cuda", generator=g) < 0.5, -1.0, 1.0)
    return s * torch.exp2(e)


def _pitch(V: int) -> int:
    """3V rounded up to 4 floats: the offsets pitch and the padded blend GEMM N (smpl_carve)."""
    return (3 * V + 3) // 4 * 4


def _split16(v):
    """hi = fp16(v), lo = fp16(v - hi) of fp32 v: the kernels' __float2half_rn pair (v - hi is exact in fp32)."""
    hi = v.half()
    return hi, (v - hi.float()).half()


def _rodrigues(aa):
    """fp64 smplx batch_rodrigues of fp32 axis-angles (.., 3) -> (.., 3, 3) on the device."""
    return S.batch_rodrigues(aa.double().cpu().reshape(-1, 3)).view(*aa.shape[:-1], 3, 3).to(aa.device)


def _sparse_rows(rows: int, V: int, nnz: int, g):
    """Row-normalised sparse regressor [rows, V] (the shape of J_regressor / joint_regressor_extra)."""
    w = torch.zeros(rows, V, device="cuda")
    idx = torch.randint(0, V, (rows, nnz), device="cuda", generator=g)
    w.scatter_add_(1, idx, torch.rand(rows, nnz, device="cuda", generator=g) + 0.05)
    return w / w.sum(1, keepdim=True)


def _basis(V: int, nb: int, seed: int):
    """A body model with magnitudes spread far past SMPL's, so that the fp16 splits meet normal, subnormal-lo and
    subnormal-hi values: v_template 2^-14..1 m, shapedirs 2^-22..2^-5, posedirs 2^-26..2^-6 (below 2^-24 the scaled
    hi itself is an fp16 subnormal), J_regressor sparse and row-normalised."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    vt = _wide((V, 3), -14, 0, g)
    sd = _wide((V, 3, nb), -22, -5, g)
    pd = _wide((PF, 3 * V), -26, -6, g)
    return vt, sd, pd, _sparse_rows(J, V, 30, g)


def _pack_ref(pd, sd, vt, nb: int, V: int):
    """smpl_pack_posedirs_kernel restated: row n = (vertex, coordinate) of [posedirs^T | shapedirs | 0 | v_template | 0]
    times 2^10, stored [hi | hi | lo]; the rows past 3V (up to the 16-byte pitch) are zero."""
    basis = torch.zeros(3 * V, PFPAD, device="cuda")
    basis[:, :PF] = pd.t()
    basis[:, BETA0:BETA0 + nb] = sd.reshape(3 * V, nb)
    basis[:, ONE] = vt.reshape(-1)
    hi, lo = _split16(basis * SCALE)
    out = torch.zeros(_pitch(V), 3 * PFPAD, dtype=torch.float16, device="cuda")
    out[:3 * V] = torch.cat([hi, hi, lo], 1)
    return out, basis


def _feature(R, betas, nb: int):
    """The blend feature row [R_j - I for joints 1..23 (207) | betas | 0 | 1 | 0] in fp32 (smpl_pose_kernel)."""
    B = R.shape[0]
    f = torch.zeros(B, PFPAD, device="cuda")
    f[:, :PF] = (R[:, 1:] - torch.eye(3, device="cuda")).reshape(B, PF)
    f[:, BETA0:BETA0 + nb] = betas
    f[:, ONE] = 1.0
    return f


def _feature_ref(R, betas, nb: int):
    """smpl_pose_kernel's pf16 restated: [hi | lo | hi] of the feature times 2^10."""
    f = _feature(R, betas, nb)
    hi, lo = _split16(f * SCALE)
    return torch.cat([hi, lo, hi], 1), f


@pytest.fixture(scope="module")
def parents_dev(cuda_dev):
    return torch.tensor(SMPL_PARENTS, dtype=torch.int32, device=cuda_dev)


def _pose(pose, pose2rot: int, betas, Jt, Jsd, nb: int, parents_dev):
    B = betas.shape[0]
    A, Jp, pf = _nan(B, J, 12), _nan(B, J, 3), _nan(B, 3 * PFPAD, dtype=torch.float16)
    probe.call("probe_smpl_pose", pose.data_ptr(), pose2rot, betas.data_ptr(), Jt.data_ptr(), Jsd.data_ptr(), nb,
               parents_dev.data_ptr(), A.data_ptr(), Jp.data_ptr(), pf.data_ptr(), B, probe.stream())
    torch.cuda.synchronize()
    return A, Jp, pf


def _joint_inputs(nb: int, g):
    """J_template (24, 3) and J_shapedirs (24, 3, nb) as smpl_jreg_kernel would give them for an SMPL-sized body."""
    return torch.randn(J, 3, device="cuda", generator=g) * 0.5, torch.randn(J, 3, nb, device="cuda", generator=g) * 0.02


# ------------------------------------------------------------------------------------------------ create-time kernels
@pytest.mark.parametrize("nb", [1, 7, 10])
@pytest.mark.parametrize("V", [37, 1000, 1003, 6890])     # 3V mod 4 = 3, 0, 1, 2
def test_create_jreg_and_pack(cuda_dev, V, nb):
    """J_template / J_shapedirs against fp64 J_regressor . v_template / shapedirs; the split blend basis bit for bit,
    with zero columns 207 + nb .. 216 and 218 .. 223 and zero pad rows."""
    vt, sd, pd, jr = _basis(V, nb, 7 * V + nb)
    Jt, Jsd = _nan(J, 3), _nan(J, 3, nb)
    probe.call("probe_smpl_jreg", jr.data_ptr(), vt.data_ptr(), sd.data_ptr(), Jt.data_ptr(), Jsd.data_ptr(), V, nb,
               probe.stream())
    packed = _nan(_pitch(V), 3 * PFPAD, dtype=torch.float16)
    probe.call("probe_smpl_pack_posedirs", pd.data_ptr(), sd.data_ptr(), vt.data_ptr(), nb, packed.data_ptr(), V,
               probe.stream())
    torch.cuda.synchronize()
    # Each of the 256 threads sums ceil(V/256) products serially (one rounding each, fused or not), the 5-level warp
    # tree adds 5 roundings and thread 0's serial sum of the 8 warp partials 7 more (its first add, to 0, is exact):
    # every product passes through at most n = ceil(V/256) + 12 roundings, gamma_n <= (n + 1) u of sum |w||x|.
    c = (math.ceil(V / 256) + 13) * U32
    jr64, vt64, sd64 = jr.double(), vt.double(), sd.double().reshape(V, 3 * nb)
    assert_within(f"J_template V={V} nb={nb}", Jt, jr64 @ vt64, c * (jr64.abs() @ vt64.abs()))
    assert_within(f"J_shapedirs V={V} nb={nb}", Jsd.reshape(J, 3 * nb), jr64 @ sd64, c * (jr64.abs() @ sd64.abs()))
    want, _ = _pack_ref(pd, sd, vt, nb, V)
    assert torch.equal(packed, want)
    for seg in range(3):
        cols = packed[:, seg * PFPAD:(seg + 1) * PFPAD]
        assert (cols[:, BETA0 + nb:ONE] == 0).all() and (cols[:, ONE + 1:] == 0).all()
    assert (packed[3 * V:] == 0).all()


# ------------------------------------------------------------------------------------------------ pose kernel
@pytest.mark.parametrize("nb", [1, 7, 10])
def test_pose_feature_exact(cuda_dev, parents_dev, nb):
    """pose2rot = 0 (R is the input itself): pf16 = [hi | lo | hi] of 2^10 (R - I) for joints 1..23, of 2^10 betas and
    of the constant 2^10, bit for bit, for |beta| up to 60.  |beta| >= 63.99 overflows the fp16 hi to inf (the
    documented range limit): the restatement and the kernel agree on that too."""
    g = torch.Generator(device="cuda").manual_seed(40 + nb)
    B = 37
    R = _rodrigues(0.6 * torch.randn(B, J, 3, device="cuda", generator=g)).float()
    R[3] += 1e-3 * torch.randn(J, 3, 3, device="cuda", generator=g)        # not a rotation: the kernel does not care
    betas = 3 * torch.randn(B, nb, device="cuda", generator=g)
    betas[0], betas[1, 0], betas[2] = 60.0, -60.0, 60 * (2 * torch.rand(nb, device="cuda", generator=g) - 1)
    betas[4, 0] = 64.0
    Jt, Jsd = _joint_inputs(nb, g)
    _, _, pf = _pose(R.contiguous(), 0, betas, Jt, Jsd, nb, parents_dev)
    want, _ = _feature_ref(R, betas, nb)
    assert torch.equal(pf, want)
    assert torch.isfinite(pf[:4]).all() and float(pf[4, BETA0]) == float("inf")


def _chain64(R, Jl, absolute: bool = False):
    """fp64 batch_rigid_transform: G_0 = [R_0 | J_0], G_i = G_parent [R_i | J_i - J_parent] -> (B, 24, 3, 4).  With
    `absolute` (R, J >= 0) the translation is J_i + J_parent: the chain on absolute values that scales the bound."""
    G = [None] * J
    for i in range(J):
        p = SMPL_PARENTS[i]
        if p < 0:
            G[i] = torch.cat([R[:, i], Jl[:, i, :, None]], -1)
        else:
            t = Jl[:, i] + Jl[:, p] if absolute else Jl[:, i] - Jl[:, p]
            rot = G[p][..., :3] @ R[:, i]
            G[i] = torch.cat([rot, (G[p][..., :3] @ t[..., None]) + G[p][..., 3:]], -1)
    return torch.stack(G, 1)


@pytest.mark.parametrize("nb", [1, 10])
def test_pose_chain_vs_fp64(cuda_dev, parents_dev, nb):
    """Relative transforms A = [G_rot | G_t - G_rot J] and posed joints G_t against an fp64 kinematic chain on the
    kernel's R (pose2rot = 0) and the fp64 joint locations J_template + J_shapedirs . betas."""
    g = torch.Generator(device="cuda").manual_seed(50 + nb)
    B = 67
    R = _rodrigues(0.8 * torch.randn(B, J, 3, device="cuda", generator=g)).float().contiguous()
    betas = 3 * torch.randn(B, nb, device="cuda", generator=g)
    betas[0] = 60.0
    Jt, Jsd = _joint_inputs(nb, g)
    A, Jp, _ = _pose(R, 0, betas, Jt, Jsd, nb, parents_dev)
    J64 = Jt.double() + torch.einsum("jcl,bl->bjc", Jsd.double(), betas.double())
    Jabs = Jt.double().abs() + torch.einsum("jcl,bl->bjc", Jsd.double().abs(), betas.double().abs())
    G = _chain64(R.double(), J64)
    Gabs = _chain64(R.double().abs(), Jabs, absolute=True)
    # Error constant by depth d.  J_i = J_template + sum_l J_shapedirs * beta_l (nb fused steps): |dJ| <= cJ u Jabs with
    # cJ = nb + 1.  Root: G_0 = [R_0 | J_0] is off by cJ u.  Each level adds the parent's error carried through
    # [R_i | t_i] (c_parent u of the absolute chain), t_i = J_i - J_parent (cJ u of |J_i| + |J_parent| plus one
    # rounding) and the 3-term rotation / 4-term translation dot products (<= 4 roundings): c_i = c_parent + cJ + 5.
    # (d + 1)(cJ + 6) covers that with one spare u per level for second-order terms.  A's translation subtracts
    # G_rot J (c_d u of Gabs_rot Jabs, cJ u from J, 4 roundings): (d + 2)(cJ + 6).
    cJ = nb + 1
    d = torch.tensor(DEPTH, dtype=torch.float64, device="cuda")[None, :, None, None]
    c_g = (d + 1) * (cJ + 6) * U32
    A64 = torch.cat([G[..., :3], G[..., 3:] - G[..., :3] @ J64[..., None]], -1)
    bound = torch.cat([c_g * Gabs[..., :3], (d + 2) * (cJ + 6) * U32 * (Gabs[..., 3:] + Gabs[..., :3] @ Jabs[..., None])],
                      -1)
    assert_within(f"A nb={nb}", A.view(B, J, 3, 4), A64, bound)
    assert_within(f"posed joints nb={nb}", Jp, G[..., 3], c_g[..., 0] * Gabs[..., 3])


ANGLES = [0.0, 1e-6, 0.3, math.pi - 1e-4, math.pi, 2 * math.pi + 0.1, 40.0]


def test_pose_rodrigues_vs_fp64(cuda_dev, parents_dev):
    """pose2rot = 1: R of every joint against fp64 Rodrigues (smplx, angle = ||r + 1e-8||) of the same fp32 axis-angle,
    at angles 0 (only the 1e-8 shift keeps r / angle finite), 1e-6, 0.3, pi - 1e-4, pi, 2 pi + 0.1 and 40.  The root's R
    is A[:, 0, :, :3] exactly; joints 1..23 are read back from pf16 (hi + lo)."""
    g = torch.Generator(device="cuda").manual_seed(60)
    n_dir = 8
    d = torch.randn(len(ANGLES) * n_dir, J, 3, device="cuda", generator=g, dtype=torch.float64)
    d[:3, :] = torch.eye(3, device="cuda", dtype=torch.float64)[:, None, :]      # the axes themselves
    d = d / d.norm(dim=-1, keepdim=True)
    theta = torch.tensor(ANGLES, device="cuda", dtype=torch.float64).repeat_interleave(n_dir)
    aa = (d * theta[:, None, None]).float().contiguous()
    B, nb = aa.shape[0], 10
    betas = torch.zeros(B, nb, device="cuda")
    Jt, Jsd = _joint_inputs(nb, g)
    A, _, pf = _pose(aa, 1, betas, Jt, Jsd, nb, parents_dev)
    R64 = _rodrigues(aa)
    ang = (aa.double() + 1e-8).norm(dim=-1)[..., None, None]
    # angle = sqrtf of a 3-term sum of squares of r + 1e-8f (the shift and the squares / sums round at most 4 times
    # relative to angle^2, sqrtf once more): |d angle| <= 5 u angle.  dir = r / angle: 6 u relative.  sincosf (CUDA's
    # documented 2 ulp = 4 u relative) of the rounded angle: |ds|, |dc| <= 5 u angle + 4 u; 1 - c one more rounding
    # (<= 2 u absolute).  R = I + s K + (1 - c) K^2 with |K_ab| <= 1, |K^2_ab| <= 1: |ds| + 6 u |s| + (|dc| + 2 u) +
    # 2 (2 * 6 u + 2 u) for the K^2 products, plus the final expression's <= 3 roundings of terms <= 6: 10 u angle + 62 u.
    bound = U32 * (10 * ang + 64)
    assert_within("rodrigues root", A.view(B, J, 3, 4)[:, 0, :, :3], R64[:, 0], bound[:, 0])
    # pf16 stores 2^10 (R - I) as hi + lo: r - 1 rounds once (2^-24) and the split keeps 22 bits (2^-22), under 2^-21
    # of |R - I| together, plus the subnormal floor 2^-35 (FLOOR).
    split = pf[:, :PF].double() + pf[:, PFPAD:PFPAD + PF].double()
    eye = torch.eye(3, device="cuda", dtype=torch.float64)
    assert_within("rodrigues joints 1..23", split.view(B, J - 1, 3, 3) / SCALE + eye, R64[:, 1:],
                  bound[:, 1:] + 2.0 ** -21 * (R64[:, 1:] - eye).abs() + FLOOR)
    assert torch.isfinite(A).all()


# ------------------------------------------------------------------------------------------------ blend GEMM
def _blend(pf16, packed, V: int, p0: int, n: int):
    off = _nan(n, _pitch(V))
    probe.call("probe_smpl_blend", pf16.data_ptr(), packed.data_ptr(), V, p0, n, off.data_ptr(), probe.stream())
    torch.cuda.synchronize()
    return off


def _blend_bound(f, basis, pf16, packed, V: int):
    """C_SPLIT sum |f||w| + C_TRUNC sum_s |P_s| (P_s: the running sum after each 16-column step, in the kernel's column
    order, on the dequantised split operands) + FLOOR (sum |w| + sum |f|)."""
    f64, w64 = f.double(), basis.double()
    a3 = pf16.double() / SCALE
    b3 = packed[:3 * V].double() / SCALE
    P = torch.zeros(f.shape[0], 3 * V, dtype=torch.float64, device="cuda")
    tot = torch.zeros_like(P)
    for s in range(0, 3 * PFPAD, 16):
        P += a3[:, s:s + 16] @ b3[:, s:s + 16].t()
        tot += P.abs()
    return (C_SPLIT * (f64.abs() @ w64.abs().t()) + C_TRUNC * tot
            + FLOOR * (w64.abs().sum(1)[None, :] + f64.abs().sum(1)[:, None]))


@pytest.mark.parametrize("V,n,p0", [(6890, 1, 0), (6890, 17, 0), (6890, 256, 0), (1003, 17, 3)])
def test_blend_gemm_vs_fp64(cuda_dev, V, n, p0):
    """v_posed = feature . [posedirs ; shapedirs ; v_template] through smpl_blend_plan against fp64 on the fp32 values
    the operands were split from; the pad columns 3V .. pitch of the offsets are exactly zero."""
    g = torch.Generator(device="cuda").manual_seed(70 + n + p0)
    nb = 10
    vt, sd, pd, _ = _basis(V, nb, 80 + V)
    packed, basis = _pack_ref(pd, sd, vt, nb, V)
    B = p0 + n
    R = _rodrigues(0.8 * torch.randn(B, J, 3, device="cuda", generator=g)).float()
    betas = 3 * torch.randn(B, nb, device="cuda", generator=g)
    betas[-1] = 60 * (2 * torch.rand(nb, device="cuda", generator=g) - 1)
    pf16, f = _feature_ref(R, betas, nb)
    off = _blend(pf16, packed, V, p0, n)
    y64 = f[p0:].double() @ basis.double().t()
    bound = _blend_bound(f[p0:], basis, pf16[p0:], packed, V)
    assert_within(f"blend GEMM V={V} n={n} p0={p0}", off[:, :3 * V], y64, bound)
    assert torch.equal(off[:, 3 * V:], torch.zeros_like(off[:, 3 * V:]))


def test_blend_bound_rejects_plain_fp16_gemm(cuda_dev):
    """Self-check of the bound: the same GEMM on fp16-only operands (the lo columns zeroed, i.e. hi.hi alone) on the
    synthetic SMPL model is far outside it, so the blend tests can tell a split blend from a plain fp16 one."""
    from tokenhmr_b200 import synth
    from tokenhmr_b200.config import release_config
    smpl = {k: v.cuda() for k, v in synth.make_smpl(release_config()).items()}
    V, nb, n = 6890, 10, 64
    packed, basis = _pack_ref(smpl["posedirs"], smpl["shapedirs"], smpl["v_template"], nb, V)
    g = torch.Generator(device="cuda").manual_seed(90)
    R = _rodrigues(0.5 * torch.randn(n, J, 3, device="cuda", generator=g)).float()
    pf16, f = _feature_ref(R, 2 * torch.randn(n, nb, device="cuda", generator=g), nb)
    y64 = f.double() @ basis.double().t()
    bound = _blend_bound(f, basis, pf16, packed, V)
    assert_within("blend GEMM (self-check data)", _blend(pf16, packed, V, 0, n)[:, :3 * V], y64, bound)
    plain_a, plain_b = pf16.clone(), packed.clone()
    plain_a[:, PFPAD:2 * PFPAD] = 0          # A' = [hi | 0 | hi]
    plain_b[:, 2 * PFPAD:] = 0               # B' = [hi | hi | 0]: only hi.hi survives
    plain = _blend(plain_a, plain_b, V, 0, n)[:, :3 * V]
    ratio = (plain.double() - y64).abs() / bound
    print(f"[bound] plain fp16 blend against the split bound: median err/bound {float(ratio.median()):.3g}, "
          f"max {float(ratio.max()):.3g}")
    assert float((ratio > 1).double().mean()) > 0.5, "the blend bound does not separate fp16 operands from split ones"


# ------------------------------------------------------------------------------------------------ skinning
def _ell_layout(V: int, ell: int, g):
    """ELL skinning weights [V, ell]: every third vertex uses all ell slots, the others 1..ell; distinct joints per
    vertex, weights positive and summing to one; unused slots hold index 0 and weight 0 (thmr_smpl_create's padding)."""
    nnz = torch.randint(1, ell + 1, (V,), device="cuda", generator=g)
    nnz[::3] = ell
    joints = torch.rand(V, J, device="cuda", generator=g).argsort(1)[:, :ell]
    used = torch.arange(ell, device="cuda")[None, :] < nnz[:, None]
    w = torch.where(used, torch.rand(V, ell, device="cuda", generator=g) + 0.05, torch.zeros((), device="cuda"))
    w = w / w.sum(1, keepdim=True)
    return torch.where(used, joints, 0).int().contiguous(), w.contiguous()


@pytest.mark.parametrize("V", [37, 6890])
@pytest.mark.parametrize("ell", [1, 4, 5, 8, 9, 24])
def test_skin_kernel_vs_fp64(cuda_dev, ell, V):
    """All four instantiations <256|128, 4|8> (register weights when ell <= kEllReg, the re-read loop otherwise) at pose
    counts around kSkinPoses = 16, against fp64 (sum_k w_k A_jk) [v_posed; 1]; the two thread shapes bit-identical."""
    g = torch.Generator(device="cuda").manual_seed(100 * ell + V)
    idx, w = _ell_layout(V, ell, g)
    W = torch.zeros(V, J, dtype=torch.float64, device="cuda").scatter_add_(1, idx.long(), w.double())
    pitch = _pitch(V)
    for B in (1, 15, 16, 17):
        A = torch.cat([_rodrigues(0.8 * torch.randn(B, J, 3, device="cuda", generator=g)).float(),
                       0.5 * torch.randn(B, J, 3, 1, device="cuda", generator=g)], -1).contiguous()
        vposed = _nan(B, pitch)
        vposed[:, :3 * V] = torch.randn(B, 3 * V, device="cuda", generator=g)    # pad columns stay NaN: never read
        vh = torch.cat([vposed[:, :3 * V].view(B, V, 3).double(), torch.ones(B, V, 1, dtype=torch.float64,
                                                                              device="cuda")], -1)
        T = torch.einsum("vj,bje->bve", W, A.double().view(B, J, 12)).view(B, V, 3, 4)
        Tabs = torch.einsum("vj,bje->bve", W.abs(), A.double().abs().view(B, J, 12)).view(B, V, 3, 4)
        ref = (T @ vh[..., None])[..., 0]
        # T: ell fused multiply-adds per entry; vertex: 3 products and 3 adds of T [v; 1] (<= 4 roundings deep):
        # (ell + 4) u of sum_k |w_k| |A_k| |[v; 1]|.
        bound = (ell + 4) * U32 * (Tabs @ vh.abs()[..., None])[..., 0]
        out = {}
        for threads in (256, 128):
            for ell_reg in (4, 8):
                verts = _nan(B, V, 3)
                probe.call("probe_smpl_skin", threads, ell_reg, idx.data_ptr(), w.data_ptr(), ell, A.data_ptr(),
                           vposed.data_ptr(), pitch, verts.data_ptr(), 3 * V, V, B, probe.stream())
                torch.cuda.synchronize()
                assert_within(f"skin <{threads},{ell_reg}> ell={ell} V={V} B={B}", verts, ref, bound)
                out[threads, ell_reg] = verts
        for ell_reg in (4, 8):
            assert torch.equal(out[256, ell_reg], out[128, ell_reg])


# ------------------------------------------------------------------------------------------------ joints / camera
@pytest.mark.parametrize("cam", [False, True])
@pytest.mark.parametrize("n_extra", [19, 0])
def test_joints_kernel(cuda_dev, n_extra, cam):
    """The 25 OpenPose joints are exact gathers (posed joints or extra_vertex_ids vertices); the CSR-regressed extra
    joints against fp64; n_extra = 0 with a null CSR; with pred_cam: focal exact, cam_t to the fp32 formula, kp2d
    against fp64 on the kernel's joints and cam_t."""
    g = torch.Generator(device="cuda").manual_seed(110 + n_extra + cam)
    B, V, focal, isz = 70, 6890, 5000.0, 256.0
    Jp = torch.randn(B, J, 3, device="cuda", generator=g)
    verts = torch.randn(B, V, 3, device="cuda", generator=g)
    jmap = torch.tensor(SMPL_TO_OPENPOSE, dtype=torch.int32, device="cuda")
    evid = torch.tensor(SMPL_EXTRA_VERTEX_IDS, dtype=torch.int32, device="cuda")
    jx = _sparse_rows(19, V, 30, g)
    jx[:, ::5] *= -1                                                            # signed weights
    nz = jx.nonzero()                                                           # CSR, rows in order
    ptr = torch.cat([torch.zeros(1, dtype=torch.int64, device="cuda"), (jx != 0).sum(1).cumsum(0)]).int()
    cidx, cval = nz[:, 1].int().contiguous(), jx[nz[:, 0], nz[:, 1]].contiguous()
    if not n_extra:
        ptr = cidx = cval = None
    nj = 25 + n_extra
    joints = _nan(B, nj, 3)
    pred_cam = cam_t = focal_out = kp2d = None
    if cam:
        pred_cam = torch.stack([0.5 + torch.rand(B, device="cuda", generator=g),
                                0.3 * torch.randn(B, device="cuda", generator=g),
                                0.3 * torch.randn(B, device="cuda", generator=g)], 1)
        cam_t, focal_out, kp2d = _nan(B, 3), _nan(B, 2), _nan(B, nj, 2)
    probe.call("probe_smpl_joints", Jp.data_ptr(), verts.data_ptr(), 3 * V, jmap.data_ptr(), evid.data_ptr(),
               probe.ptr(ptr), probe.ptr(cidx), probe.ptr(cval), n_extra, joints.data_ptr(), probe.ptr(pred_cam), focal,
               isz, probe.ptr(cam_t), probe.ptr(focal_out), probe.ptr(kp2d), B, probe.stream())
    torch.cuda.synchronize()
    j45 = torch.cat([Jp, verts[:, SMPL_EXTRA_VERTEX_IDS]], 1)
    assert torch.equal(joints[:, :25], j45[:, SMPL_TO_OPENPOSE])
    if n_extra:
        jx64 = jx.double()
        ref = torch.einsum("rv,bvc->brc", jx64, verts.double())
        # serial x += w s over a row's nnz entries (one rounding each): (nnz + 1) u of sum |w||v|
        nnz = (jx != 0).sum(1).double()[None, :, None]
        bound = (nnz + 1) * U32 * torch.einsum("rv,bvc->brc", jx64.abs(), verts.double().abs())
        assert_within(f"regressed joints B={B}", joints[:, 25:], ref, bound)
    if cam:
        assert torch.equal(focal_out, torch.full((B, 2), focal, device="cuda"))
        assert torch.equal(cam_t[:, :2], pred_cam[:, 1:])
        # nvcc may contract isz * s + 1e-9 into one FMA: the denominator then differs by at most one rounding (1 ulp)
        # from torch's two-step fp32, and the quotient by at most 2 ulp = 2^-22 relative.
        t32 = 2 * focal / (isz * pred_cam[:, 0] + 1e-9)
        assert ((cam_t[:, 2] - t32).abs() <= 2.0 ** -22 * t32.abs()).all()
        x = joints.double()
        t = cam_t.double()[:, None, :]
        kp64 = (focal / isz) * (x[..., :2] + t[..., :2]) / (x[..., 2:] + t[..., 2:])
        # px = x + t and pz = z + t_z round once each (relative to themselves), f = focal / image_size, px / pz and
        # f * (px / pz) once each: 5 roundings, each relative to the result -> 6 u |kp|.
        assert_within(f"kp2d n_extra={n_extra}", kp2d, kp64, 6 * U32 * kp64.abs())


# ------------------------------------------------------------------------------------------------ product ABI
def _weights_with(V: int, k: int, seed: int):
    """lbs_weights with exactly k non-zeros per vertex (distinct joints, rows summing to one)."""
    g = torch.Generator().manual_seed(seed)
    joints = torch.rand(V, J, generator=g).argsort(1)[:, :k]
    w = torch.zeros(V, J).scatter_(1, joints, torch.rand(V, k, generator=g) + 0.05)
    return w / w.sum(1, keepdim=True)


def _variant(name: str):
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


VARIANTS = ["base", "w6", "w12", "nb7", "noextra", "V1003"]


@pytest.fixture(scope="module")
def models(cuda_dev):
    from tokenhmr_b200 import ops
    cache = {}

    def get(name):
        if name not in cache:
            smpl = _variant(name)
            cache[name] = (smpl, ops.SMPLModel(smpl, cuda_dev))
        return cache[name]
    return get


def _oracle_forward(smpl, rot, betas):
    """oracle.smpl_forward in fp64; without joint_regressor_extra only the 25 mapped joints."""
    if "joint_regressor_extra" in smpl:
        return S.smpl_forward(smpl, rot[:, :1], rot[:, 1:], betas, dtype=torch.float64)
    c = lambda t: t.double()
    verts, joints = S.lbs(c(betas), c(rot), c(smpl["v_template"]), c(smpl["shapedirs"]), c(smpl["posedirs"]),
                          c(smpl["J_regressor"]), smpl["parents"], c(smpl["lbs_weights"]), pose2rot=False)
    j45 = torch.cat([joints, verts[:, smpl["extra_vertex_ids"]]], 1)
    return verts, j45[:, torch.tensor(SMPL_TO_OPENPOSE)]


def _contract(name, got, ref):
    # DESIGN §2's SMPL contract per element: |err| <= 1e-4 |ref| + 1e-5 m.  The floor is for coordinates near zero,
    # which are sums of terms of up to ~1 m (template, shape offsets at |beta| = 60, joint translations): each such
    # term carries an fp32 rounding of 2^-24 m ~ 6e-8 m, so 1e-5 m is ~100x the rounding of one unit-size term and
    # covers the ~20 terms of the blend and the skinning with room for the blend GEMM's truncating accumulation.
    ref = ref.double()
    assert_within(name, got, ref, 1e-4 * ref.abs() + 1e-5)


@pytest.mark.parametrize("B", [1, 255, 256, 257, 513])          # around kSmplChunk = 256
@pytest.mark.parametrize("variant", VARIANTS)
def test_smpl_model_vs_oracle(cuda_dev, models, variant, B):
    """SMPLModel.lbs (axis-angle) and SMPLModel.forward (rotation matrices) against oracle.smpl_oracle in fp64 on body
    models with 6 and 12 skinning weights per vertex, 7 betas, no extra-joint regressor and V = 1003, with |beta| up to
    60 (the fp16 split of 2^10 beta overflows at 63.99)."""
    smpl, m = models(variant)
    nb = smpl["shapedirs"].shape[2]
    g = torch.Generator().manual_seed(B + 1000 * VARIANTS.index(variant))
    aa = 0.6 * torch.randn(B, J, 3, generator=g)
    betas = 2 * torch.randn(B, nb, generator=g)
    betas[::4] = 60 * (2 * torch.rand(betas[::4].shape, generator=g) - 1)
    betas[0, 0], betas[-1, -1] = 60.0, -60.0
    with torch.device("cuda"):
        s64 = {k: (v.cuda().double() if v.is_floating_point() else v.cuda()) for k, v in smpl.items()}
        vr, jr = S.lbs(betas.cuda().double(), aa.cuda().double().reshape(B, -1), s64["v_template"], s64["shapedirs"],
                       s64["posedirs"], s64["J_regressor"], s64["parents"], s64["lbs_weights"], pose2rot=True)
        rot = S.batch_rodrigues(aa.cuda().double().reshape(-1, 3)).view(B, J, 3, 3)
        rot32 = rot.float()
        fv, fj = _oracle_forward(s64, rot32.double(), betas.cuda().double())
    v, j = m.lbs(betas.cuda(), aa.cuda(), pose2rot=True)
    _contract(f"lbs verts {variant} B={B}", v, vr)
    _contract(f"lbs joints {variant} B={B}", j, jr)
    v, j = m.forward(rot32[:, :1], rot32[:, 1:], betas.cuda())
    _contract(f"forward verts {variant} B={B}", v, fv)
    _contract(f"forward joints {variant} B={B}", j, fj)
    assert j.shape[1] == (25 if variant == "noextra" else 44)


def test_engine_smpl_tail_equals_smpl_model_forward(cuda_dev):
    """The engine's SMPL tail (blend plans built once per batch shape) gives bit for bit what SMPLModel.forward (plans
    built per call) gives on the engine's own rotation matrices, betas and camera, across a pose-chunk boundary."""
    from tokenhmr_b200 import synth
    from tokenhmr_b200.config import tiny_config
    from tokenhmr_b200.engine import TokenHMREngine
    cfg = tiny_config(vit_depth=2)
    model = TokenHMREngine(cfg, synth.make_state_dict(cfg), synth.make_smpl(cfg), device=cuda_dev,
                           use_cuda_graph=False, max_batch=260)
    B = 257
    out = model({"img": synth.make_images(B, cfg, seed=4)})
    p = out["pred_smpl_params"]
    v, j, cam_t, focal, kp2d = model.smpl_model.forward(p["global_orient"], p["body_pose"], p["betas"],
                                                        pred_cam=out["pred_cam"], focal_length=cfg.focal_length,
                                                        image_size=float(cfg.image_size))
    torch.cuda.synchronize()
    assert torch.equal(v, out["pred_vertices"]) and torch.equal(j, out["pred_keypoints_3d"])
    assert torch.equal(cam_t, out["pred_cam_t"]) and torch.equal(focal, out["focal_length"])
    assert torch.equal(kp2d, out["pred_keypoints_2d"])

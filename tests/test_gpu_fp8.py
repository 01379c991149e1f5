"""FP8 mode, kernel by kernel: the LayerNorm with e4m3 output, the block-scaled e4m3 wgmma GEMM (with its promotion
and its e4m3 output epilogue), against the quantisation definition (exact) and fp64 (per-element bounds)."""
import pytest
import torch

import probe
from tokenhmr_b200 import fp8

pytestmark = pytest.mark.gpu

# Tensor-core accumulation of the 128-element k-blocks (four k32 MMAs into a fresh tile each), relative to sum |a||w|.
# The products of two e4m3 codes are exact; what the FP8 tensor core keeps of their running sum is not documented (the
# DeepSeek-V3 report says fewer bits than fp32), so this constant is measured: with 2^-9 here the worst err / bound
# over the cases below was 0.19 (0.21 through GELU) on an H100 80GB HBM3 at 400 W, i.e. the accumulation loses up to
# ~2^-11.4 of sum |a||w| -- some 2^9 times what fp32 accumulation of the same products would (DESIGN.md §2).
# Pinned at 2^-10 (a 2.3x margin); the promotion adds one fp32 rounding per k-block on top.
C_BLK = 2.0 ** -10


@pytest.fixture(autouse=True)
def _flags(cuda_dev, built_lib):
    yield
    assert probe.flags() == 0, "probe device flags set"


def _blocky(rows: int, cols: int, g, spread: int = 4) -> torch.Tensor:
    """randn with a different power-of-two magnitude per 128 x 128 block (so that every block has its own scale and a
    transposed or shifted block index shows), plus a few exact zeros and tiny values (subnormal codes)."""
    x = torch.randn(rows, cols, device="cuda", generator=g)
    e = torch.randint(-spread, spread + 1, ((rows + 127) // 128, (cols + 127) // 128), device="cuda", generator=g)
    x = x * torch.ldexp(torch.ones_like(x), e.repeat_interleave(128, 0)[:rows].repeat_interleave(128, 1)[:, :cols])
    x[:, 5] = 0.0
    x[3, :] *= 2.0 ** -12
    return x


def _pad_scales(s: torch.Tensor, rows: int) -> torch.Tensor:
    """[K/128, R] -> [K/128, R rounded up to 128 + 128]: the row-tile-padded layout the GEMM reads."""
    out = torch.ones(s.shape[0], (rows + 127) // 128 * 128 + 128, device=s.device)
    out[:, :rows] = s
    return out


def test_layernorm_e4m3_matches_definition(cuda_dev):
    """Scales and codes equal the definition applied to the kernel's own fp32 pre-quantisation values, and those
    values equal the default LayerNorm's fp32 output bit for bit."""
    g = torch.Generator(device="cuda").manual_seed(11)
    R, C = 1000, 1280
    x = 3.0 * torch.randn(R, C, device=cuda_dev, generator=g) + 0.5
    x[7] = 0.0                                   # constant row: every output = beta
    gamma = torch.randn(C, device=cuda_dev, generator=g)
    beta = 0.1 * torch.randn(C, device=cuda_dev, generator=g)
    beta[:128] = 0.0                             # row 7, group 0: amax = 0 -> scale 1, codes 0
    y32 = torch.full((R, C), float("nan"), device=cuda_dev)
    y8, ys = probe.layernorm_e4m3(x, gamma, beta, 1e-6, y32=y32, lds=R + 24)
    ref32 = torch.empty(R, C, device=cuda_dev)
    probe.call("probe_layernorm", x.data_ptr(), gamma.data_ptr(), beta.data_ptr(), None, 0, ref32.data_ptr(), R, C,
               1e-6, 0, 0, probe.stream())
    torch.cuda.synchronize()
    assert torch.equal(y32, ref32)
    codes, s = fp8.quantize_rows(y32)
    assert torch.equal(ys[:, :R], s)
    assert torch.equal(y8, codes.view(torch.uint8))
    assert float(ys[0, 7]) == 1.0 and not bool(y8[7, :128].any())


def _check_gemm(name, A, W, M, N, K, *, act="none", bias=None, resid=None, force_bn=0, e4m3_out=False, report=None):
    qa, sa = fp8.quantize_rows(A)
    qw, sw = fp8.quantize_weight_blocks(W)
    a_scale = _pad_scales(sa, M)
    out32 = torch.full((M, N), float("nan"), device="cuda") if resid is None else resid.clone()
    out8 = out8_scale = None
    if e4m3_out:
        out8 = torch.zeros(M, N, dtype=torch.uint8, device="cuda")
        out8_scale = torch.full((N // 128, M), float("nan"), device="cuda")
    probe.gemm_fp8(qa, a_scale, qw, sw, M, N, K, bias=bias, resid=out32 if resid is not None else None,
               ldr=N if resid is not None else 0, act=act, out32=out32, ld32=N, out8=out8, out8_scale=out8_scale,
               force_bn=force_bn)
    torch.cuda.synchronize()
    Ad = fp8.dequantize_rows(qa, sa).double()
    Wd = fp8.dequantize_weight_blocks(qw, sw).double()
    acc = Ad @ Wd.t()
    mag = Ad.abs() @ Wd.abs().t()
    pre = acc + (bias.double() if bias is not None else 0.0) + (resid.double() if resid is not None else 0.0)
    terms = pre.abs() + (bias.double().abs() if bias is not None else 0.0) + (resid.double().abs() if resid is not None
                                                                               else 0.0)
    # k-block accumulation (C_BLK) + K / 128 fp32 promotion additions, then bias and residual additions
    bound = (C_BLK + (K // 128) * probe.U32) * mag + 2 * probe.U32 * terms + 2.0 ** -60
    if act == "gelu":
        # GELU: slope <= 1.13, the kernel's erf approximation within 9e-7 absolute, one fp32 rounding
        ref = probe.gelu64(pre)
        bound = 1.13 * bound + 9e-7 + 2 * probe.U32 * ref.abs()
    else:
        ref = pre
    ratio = float(((out32.double() - ref).abs() / mag.clamp_min(1e-30)).max())
    print(f"[fp8] {name}: max err / sum|a||w| = {ratio:.3g} (2^{torch.log2(torch.tensor(ratio)).item():.1f})")
    worst = probe.assert_within(name, out32, ref, bound, report)
    if e4m3_out:
        codes, s = fp8.quantize_rows(out32)
        assert torch.equal(out8_scale, s), f"{name}: e4m3 output scales differ from the definition"
        assert torch.equal(out8, codes.view(torch.uint8)), f"{name}: e4m3 output codes differ from the definition"
    return worst


# ViT shapes at bs = 64 (M = 12288) and edge shapes: M not a multiple of 128, a partial last weight block (N = 200),
# both tile widths, the in-place fp32 residual of fc2 and proj, and the e4m3 output of fc1 + GELU.
CASES = {
    "qkv": dict(M=12288, N=3840, K=1280, bias=True),
    "fc1_gelu_e4m3": dict(M=12288, N=5120, K=1280, bias=True, act="gelu", e4m3_out=True),
    "fc2_resid": dict(M=12288, N=1280, K=5120, bias=True, resid=True),
    "m1000_n200_bn64": dict(M=1000, N=200, K=384, bias=True, force_bn=64),
    "m1000_n200_bn128": dict(M=1000, N=200, K=384, bias=True, force_bn=128),
    "m1000_resid_bn64": dict(M=1000, N=1280, K=1280, resid=True, force_bn=64),
    "m1000_gelu_e4m3": dict(M=1000, N=640, K=256, bias=True, act="gelu", e4m3_out=True),
}


@pytest.mark.parametrize("case", list(CASES))
def test_gemm_fp8_against_fp64(cuda_dev, case):
    c = CASES[case]
    g = torch.Generator(device="cuda").manual_seed(list(CASES).index(case))
    M, N, K = c["M"], c["N"], c["K"]
    A = _blocky(M, K, g)
    W = 0.05 * _blocky(N, K, g)
    bias = torch.randn(N, device=cuda_dev, generator=g) if c.get("bias") else None
    resid = torch.randn(M, N, device=cuda_dev, generator=g) if c.get("resid") else None
    _check_gemm(case, A, W, M, N, K, act=c.get("act", "none"), bias=bias, resid=resid,
                force_bn=c.get("force_bn", 0), e4m3_out=c.get("e4m3_out", False))


def test_gemm_fp8_chain_uses_epilogue_scales(cuda_dev):
    """fc1's e4m3 output and its scales feed fc2 as they are (the engine's chain): the second GEMM on them equals fp64
    on the dequantised h within the same bound as on host-quantised operands."""
    g = torch.Generator(device="cuda").manual_seed(5)
    M, D, F = 640, 256, 1024
    x = torch.randn(M, D, device=cuda_dev, generator=g)
    W1, W2 = 0.1 * _blocky(F, D, g), 0.05 * _blocky(D, F, g)
    qx, sx = fp8.quantize_rows(x)
    q1, s1 = fp8.quantize_weight_blocks(W1)
    q2, s2 = fp8.quantize_weight_blocks(W2)
    h8 = torch.zeros(M, F, dtype=torch.uint8, device=cuda_dev)
    hs = torch.ones(F // 128, (M + 127) // 128 * 128 + 128, device=cuda_dev)
    h32 = torch.empty(M, F, device=cuda_dev)
    probe.gemm_fp8(qx, _pad_scales(sx, M), q1, s1, M, F, D, act="gelu", out32=h32, ld32=F, out8=h8, out8_scale=hs)
    y = torch.full((M, D), float("nan"), device=cuda_dev)
    probe.gemm_fp8(h8, hs, q2, s2, M, D, F, out32=y, ld32=D)
    torch.cuda.synchronize()
    hq, hsc = fp8.quantize_rows(h32)
    assert torch.equal(h8, hq.view(torch.uint8)) and torch.equal(hs[:, :M], hsc)
    Hd = fp8.dequantize_rows(hq, hsc).double()
    W2d = fp8.dequantize_weight_blocks(q2, s2).double()
    ref = Hd @ W2d.t()
    bound = (C_BLK + (F // 128) * probe.U32) * (Hd.abs() @ W2d.abs().t()) + 2 * probe.U32 * ref.abs() + 2.0 ** -60
    probe.assert_within("fc1 -> fc2 chain", y, ref, bound)


# ------------------------------------------------------------------------------------------------ the engine
KEYS = ("_vit_tokens", "_token_out", "_pred_body_pose_6d", "pred_cam", "pred_cam_t", "pred_keypoints_3d",
        "pred_vertices", "pred_keypoints_2d", "cls_logits_softmax")


@pytest.fixture(scope="module")
def tiny_fp8(cuda_dev):
    from tokenhmr_b200 import synth
    from tokenhmr_b200.config import tiny_config
    from tokenhmr_b200.engine import TokenHMREngine
    cfg = tiny_config(vit_depth=2)
    sd, smpl = synth.make_state_dict(cfg), synth.make_smpl(cfg)
    return cfg, sd, smpl, TokenHMREngine(cfg, sd, smpl, device=cuda_dev, use_cuda_graph=False, fp8=True)


@pytest.mark.parametrize("B", [1, 2, 5])
def test_fp8_engine_vs_emulation(tiny_fp8, B):
    """The engine against the CPU emulation of its own contract (tests/fp8_emulation.py) and against fp32: per output
    key, engine-vs-emulation must be clearly tighter than emulation-vs-fp32 (the emulation accounts for most of the
    mode's error), and engine-vs-fp32 stays within the pinned FP8 tolerance.  Measured ratios are 5-22x on the head's
    outputs and 2.1-2.7x on the ViT tokens: the emulation sums each k-block in fp64, the FP8 tensor core with fewer
    bits (C_BLK), and every such difference that moves an activation across an e4m3 rounding boundary becomes a whole
    half-step (2^-4 relative) of that code, compounding over the blocks.  Hence the 2x floor here."""
    import fp8_emulation as E
    from conftest import rel_err
    from oracle import tokenhmr_oracle as O
    from tokenhmr_b200 import synth
    cfg, sd, smpl, model = tiny_fp8
    img = synth.make_images(B, cfg, seed=B)
    out = model({"img": img}, return_taps=True)
    with torch.no_grad():
        emu = E.forward_fp8(sd, smpl, img, cfg, return_intermediates=True)
        f32 = O.forward(sd, smpl, img, cfg, emulate_fp16=False, return_intermediates=True)
    rows = {}
    for k in KEYS:
        a, b = rel_err(out[k], emu[k]), rel_err(emu[k], f32[k])
        rows[k] = (a, b, rel_err(out[k], f32[k]))
        print(f"[fp8 engine] B={B} {k}: engine-vs-emu {a:.2e}  emu-vs-fp32 {b:.2e}  ratio {b / max(a, 1e-30):.1f}  "
              f"engine-vs-fp32 {rows[k][2]:.2e}")
    for k, (a, b, c) in rows.items():
        assert a < 0.5 * b, (k, a, b)
        assert c < FP8_TOL_F32[k], (k, c)


# engine vs the fp32 reference at depth 2 (synthetic weights), relative to max|ref|: the worst over B = 1, 2, 5 measured
# on an H100 80GB HBM3 at 400 W (DESIGN.md §2), pinned with a 2x margin
FP8_TOL_F32 = {"_vit_tokens": 0.06, "_token_out": 7e-3, "_pred_body_pose_6d": 5e-3, "pred_cam": 1.5e-3,
               "pred_cam_t": 1.5e-3, "pred_keypoints_3d": 4e-3, "pred_vertices": 4e-3, "pred_keypoints_2d": 4e-3,
               "cls_logits_softmax": 0.07}


def test_fp8_graph_replay_is_bit_identical_and_stamps_cover_the_replay(tiny_fp8):
    from tokenhmr_b200 import synth
    cfg, _, _, model = tiny_fp8
    img = synth.make_images(2, cfg, seed=9)
    eager = {k: v.clone() for k, v in model({"img": img}).items() if isinstance(v, torch.Tensor)}
    model.use_cuda_graph = True
    try:
        for _ in range(2):
            g = model({"img": img})
            for k, v in eager.items():
                assert torch.equal(g[k], v), k
        imgc = img.cuda()
        rows = model.profile_in_graph(imgc, replays=3)
        names = {n for n, ms, _, _ in rows if ms > 0}
        assert {"vit.layernorm", "vit.qkv_gemm", "vit.attention", "vit.proj_gemm", "vit.fc1_gelu_gemm",
                "vit.fc2_gemm"} <= names
        total = sum(ms for _, ms, _, _ in rows)
        st = model._state(2, False, slot=-1)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        st["graph"].replay()
        e0.record()
        for _ in range(5):
            st["graph"].replay()
        e1.record()
        torch.cuda.synchronize()
        per = e0.elapsed_time(e1) / 5
        assert 0.6 * per < total < 1.4 * per, (total, per)
    finally:
        model.use_cuda_graph = False


def test_fp8_launch_count_and_vit_forward(tiny_fp8, cuda_dev):
    """The fp8 chain replaces kernels one for one (same launch count as the default engine), and the backbone-only
    entry point returns the forward's own ViT tokens."""
    from tokenhmr_b200 import synth
    from tokenhmr_b200.engine import TokenHMREngine
    cfg, sd, smpl, model = tiny_fp8
    img = synth.make_images(3, cfg, seed=4)
    out = model({"img": img}, return_taps=True)
    plain = TokenHMREngine(cfg, sd, smpl, device=cuda_dev, use_cuda_graph=False)
    plain({"img": img})
    assert model.num_launches() == plain.num_launches()
    bb = model.backbone(img)
    assert torch.equal(bb.flatten(2).transpose(1, 2), out["_vit_tokens"])


def test_fp8_four_stream_pipeline_matches_synchronous_forward(cuda_dev):
    from tokenhmr_b200 import synth
    from tokenhmr_b200.config import tiny_config
    from tokenhmr_b200.engine import TokenHMREngine, TokenHMRPipeline, load_tokenhmr
    cfg = tiny_config(vit_depth=2)
    sd, smpl = synth.make_state_dict(cfg), synth.make_smpl(cfg)
    model, _ = load_tokenhmr(sd, smpl, cfg, device=cuda_dev, use_cuda_graph=False, concurrent=True,
                             max_cached_shapes=8, fp8=True)
    assert isinstance(model, TokenHMREngine) and model.fp8
    keys = ("pred_vertices", "pred_keypoints_3d", "pred_cam", "pred_cam_t")
    batches = [synth.make_images(8, cfg, seed=60 + i).pin_memory() for i in range(9)]
    want = []
    for b in batches:
        out = model({"img": b})
        want.append({k: out[k].cpu().clone() for k in keys})
    model.use_cuda_graph = True
    pipe = TokenHMRPipeline(model, depth=4, read_back=keys, streams=4)
    tickets, got = [], []
    for b in batches:
        tickets.append(pipe.submit({"img": b}))
        if len(tickets) >= 4:
            got.append({k: v.clone() for k, v in pipe.result(tickets[len(got)]).items()})
    while len(got) < len(batches):
        got.append({k: v.clone() for k, v in pipe.result(tickets[len(got)]).items()})
    for g, w in zip(got, want):
        for k in keys:
            assert torch.equal(g[k], w[k]), k


def test_fp8_release_vs_reference_golden(cuda_dev, golden_dir):
    """Full ViT-H/16 depth-32 forward at B = 2 against the live reference's fp32 outputs, and bs = 64 sanity."""
    import numpy as np
    from conftest import rel_err
    from tokenhmr_b200 import synth
    from tokenhmr_b200.config import release_config
    from tokenhmr_b200.engine import TokenHMREngine
    g = np.load(golden_dir / "forward_release_d32.npz")
    cfg = release_config()
    model = TokenHMREngine(cfg, synth.make_state_dict(cfg, 1234), synth.make_smpl(cfg, 3), device=cuda_dev, fp8=True)
    out = model({"img": synth.make_images(2, cfg, 0)}, return_taps=True)
    t = lambda k: torch.from_numpy(g[k])
    errs = {"vit_tokens": rel_err(out["_vit_tokens"][:, ::8], t("vit_tokens_sub"))}
    for k in ("pred_cam", "pred_cam_t", "pred_keypoints_3d", "pred_vertices", "pred_keypoints_2d"):
        errs[k] = rel_err(out[k], t(k))
    same = float((out["cls_logits_softmax"].argmax(-1).cpu().numpy() == g["cls_argmax"]).mean())
    print("[fp8 release] B=2 vs fp32 reference", {k: f"{v:.2e}" for k, v in errs.items()}, f"token agreement {same:.4f}")
    for k, v in errs.items():
        assert v < FP8_TOL_RELEASE[k], (k, v)
    assert same >= FP8_MIN_TOKEN_AGREEMENT, same
    out = model({"img": synth.make_images(64, cfg, 5)})
    assert all(torch.isfinite(v).all() for v in out.values() if isinstance(v, torch.Tensor))
    torch.testing.assert_close(out["cls_logits_softmax"].sum(-1), torch.ones(64, 160, device=cuda_dev), atol=1e-4,
                               rtol=0)
    sp = out["pred_smpl_params"]
    R = torch.cat([sp["global_orient"], sp["body_pose"]], 1)
    torch.testing.assert_close(R @ R.transpose(-1, -2), torch.eye(3, device=cuda_dev).expand(64, 24, 3, 3), atol=1e-5,
                               rtol=0)


# depth 32, B = 2, vs the live reference's fp32 outputs (synthetic weights), measured on an H100 80GB HBM3 at 400 W:
# vit_tokens 6.3e-2, pred_cam 4.5e-3, pred_cam_t 2.3e-3, keypoints_3d 9.6e-3, vertices 1.04e-2, keypoints_2d 1.09e-2,
# pose tokens 294 of 320 equal (0.919).  Pinned with a 2x margin (tokens: twice the mismatches).
FP8_TOL_RELEASE = {"vit_tokens": 0.13, "pred_cam": 1e-2, "pred_cam_t": 5e-3, "pred_keypoints_3d": 2e-2,
                   "pred_vertices": 2.1e-2, "pred_keypoints_2d": 2.2e-2}
FP8_MIN_TOKEN_AGREEMENT = 0.83

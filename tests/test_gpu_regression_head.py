"""HMR 2.0's regression head (cfg.head == "transformer_decoder") on the GPU, in every numeric mode: parity with the oracle
and with goldens written by the LIVE reference head, the output contract, graph replay, the two-stream pipeline, launch
counts, and a token engine in the same process that must not notice it."""
import ctypes

import numpy as np
import pytest
import torch

from conftest import rel_err

pytestmark = pytest.mark.gpu

REG = "transformer_decoder"
# the shared keys of tests/test_gpu_engine.py's tolerances (fp16 operands / fp32 accumulation), without the logits
TOL_EMU = {"_vit_tokens": 5e-4, "_token_out": 6e-4, "_pred_body_pose_6d": 6e-4, "pred_cam": 3e-4, "pred_cam_t": 3e-4,
           "pred_keypoints_3d": 6e-4, "pred_vertices": 6e-4, "pred_keypoints_2d": 8e-4}
TOL_F32 = {k: 2 * v for k, v in TOL_EMU.items()}
KEYS = list(TOL_EMU)
OUT_KEYS = {"pred_cam", "pred_smpl_params", "pred_cam_t", "focal_length", "pred_keypoints_3d", "pred_vertices",
            "pred_keypoints_2d"}


@pytest.fixture(autouse=True)
def _flags(cuda_dev, built_lib):
    yield
    assert built_lib.thmr_check_device_flags() == 0, built_lib.thmr_last_error()


@pytest.fixture(scope="module")
def tiny(cuda_dev):
    from tokenhmr_b200 import synth
    from tokenhmr_b200.config import tiny_config
    from tokenhmr_b200.engine import TokenHMREngine
    cfg = tiny_config(vit_depth=2, head=REG)
    sd, smpl = synth.make_state_dict(cfg), synth.make_smpl(cfg)
    return cfg, sd, smpl, TokenHMREngine(cfg, sd, smpl, device=cuda_dev, use_cuda_graph=False, max_batch=320)


@pytest.mark.parametrize("B", [1, 2, 5])
def test_tiny_forward_vs_oracle(tiny, B):
    from oracle import regression_oracle as R
    from oracle import smpl_oracle as S
    from tokenhmr_b200 import synth
    cfg, sd, smpl, model = tiny
    img = synth.make_images(B, cfg, seed=B)
    out = model({"img": img}, return_taps=True)
    with torch.no_grad():
        emu = R.forward(sd, smpl, img, cfg, emulate_fp16=True, return_intermediates=True)
        f32 = R.forward(sd, smpl, img, cfg, emulate_fp16=False, return_intermediates=True)
    print(f"regression B={B} vs emu", {k: f"{rel_err(out[k], emu[k]):.1e}" for k in KEYS})
    print(f"regression B={B} vs f32", {k: f"{rel_err(out[k], f32[k]):.1e}" for k in KEYS})
    for k in KEYS:
        assert rel_err(out[k], emu[k]) < TOL_EMU[k], (k, rel_err(out[k], emu[k]))
        assert rel_err(out[k], f32[k]) < TOL_F32[k], (k, rel_err(out[k], f32[k]))
    for k in ("global_orient", "body_pose", "betas"):
        assert rel_err(out["pred_smpl_params"][k], emu["pred_smpl_params"][k]) < 1e-3
    # SMPL stage given the engine's own rotations and betas: 1e-4
    p = out["pred_smpl_params"]
    v, j = S.smpl_forward(smpl, p["global_orient"].cpu(), p["body_pose"].cpu(), p["betas"].cpu())
    assert rel_err(out["pred_vertices"], v) < 1e-4 and rel_err(out["pred_keypoints_3d"], j) < 1e-4


def test_output_contract(tiny, built_lib):
    """The reference's dict for this head (tokenhmr.py:156-187 with TYPE transformer_decoder): every key of the token
    head's except cls_logits_softmax.  Asking the C ABI for the logits is refused before anything runs."""
    from tokenhmr_b200 import _lib, synth
    cfg, _, _, model = tiny
    out = model({"img": synth.make_images(3, cfg).cuda()}, return_taps=True)
    assert {k for k in out if not k.startswith("_")} == OUT_KEYS
    assert "cls_logits_softmax" not in model._state(3, True)["t"]
    want = {"pred_cam": (3, 3), "pred_cam_t": (3, 3), "focal_length": (3, 2), "pred_keypoints_3d": (3, 44, 3),
            "pred_vertices": (3, cfg.num_verts, 3), "pred_keypoints_2d": (3, 44, 2), "_pred_body_pose_6d": (3, 144)}
    for k, shape in want.items():
        assert tuple(out[k].shape) == shape and out[k].dtype == torch.float32 and out[k].is_cuda, k
    sp = out["pred_smpl_params"]
    assert tuple(sp["global_orient"].shape) == (3, 1, 3, 3) and tuple(sp["body_pose"].shape) == (3, 23, 3, 3)
    R = torch.cat([sp["global_orient"], sp["body_pose"]], 1)
    torch.testing.assert_close(R @ R.transpose(-1, -2), torch.eye(3, device="cuda").expand(3, 24, 3, 3), atol=1e-5, rtol=0)
    assert torch.all(out["focal_length"] == 5000.0)
    # thmr_engine_forward with a logits pointer
    st = model._state(3, False)
    outs = _lib.Outputs()
    ctypes.memmove(ctypes.byref(outs), ctypes.byref(st["outs"]), ctypes.sizeof(outs))
    logits = torch.empty(3, cfg.token_num, cfg.token_class_num, device="cuda")
    outs.cls_logits_softmax = logits.data_ptr()
    rc = built_lib.thmr_engine_forward(model._h, st["t"]["img"].data_ptr(), 3, ctypes.byref(outs), st["ws_ptr"],
                                       torch.cuda.current_stream().cuda_stream)
    assert rc == -1 and b"cls_logits_softmax" in built_lib.thmr_last_error()     # THMR_ERR_INVALID
    assert model.backbone(synth.make_images(2, cfg)).shape == (2, 1280, 16, 12)


def test_cuda_graph_replay_and_batch_independence(tiny):
    from tokenhmr_b200 import synth
    cfg, _, _, model = tiny
    img = synth.make_images(4, cfg, seed=9)
    eager = {k: v.clone() for k, v in model({"img": img}).items() if isinstance(v, torch.Tensor)}
    model.use_cuda_graph = True
    try:
        for _ in range(2):
            g = model({"img": img})
            for k, v in eager.items():
                assert torch.equal(g[k], v), k
        assert not torch.equal(model({"img": synth.make_images(4, cfg, seed=10)})["pred_vertices"],
                               eager["pred_vertices"])
    finally:
        model.use_cuda_graph = False
    one = model({"img": img[2:3]})["pred_vertices"]
    assert rel_err(one, eager["pred_vertices"][2:3]) < 1e-3
    assert torch.equal(model({"img": img})["pred_vertices"], eager["pred_vertices"])


def test_two_stream_pipeline_matches_synchronous_forward(cuda_dev, tiny):
    from tokenhmr_b200 import synth
    from tokenhmr_b200.engine import TokenHMREngine, TokenHMRPipeline
    cfg, sd, smpl, _ = tiny
    model = TokenHMREngine(cfg, sd, smpl, device=cuda_dev, use_cuda_graph=False, concurrent=True, max_cached_shapes=8)
    keys = ("pred_vertices", "pred_keypoints_3d", "pred_cam", "pred_cam_t")
    batches = [synth.make_images(8, cfg, seed=60 + i).pin_memory() for i in range(6)]
    want = [{k: v.cpu().clone() for k, v in model({"img": b}).items() if k in keys} for b in batches]
    model.use_cuda_graph = True
    pipe = TokenHMRPipeline(model, depth=2, read_back=keys, streams=2)
    tickets, got = [], []
    for b in batches:
        tickets.append(pipe.submit({"img": b}))
        if len(tickets) >= 2:
            got.append({k: v.clone() for k, v in pipe.result(tickets[len(got)]).items()})
    while len(got) < len(batches):
        got.append({k: v.clone() for k, v in pipe.result(tickets[len(got)]).items()})
    for g, w in zip(got, want):
        for k in keys:
            assert torch.equal(g[k], w[k]), k


def test_release_forward_vs_reference_golden(cuda_dev, golden_dir):
    """ViT-H/16 depth 32 at B = 64 against the outputs of the LIVE reference regression head (fp32)."""
    from tokenhmr_b200 import synth
    from tokenhmr_b200.config import TokenHMRConfig
    from tokenhmr_b200.engine import TokenHMREngine
    g = np.load(golden_dir / "forward_regression_release_d32.npz")
    W, S, I, B, depth, V, stride = (int(v) for v in g["meta"])
    cfg = TokenHMRConfig(head=REG)
    assert (B, depth, V) == (64, cfg.vit_depth, cfg.num_verts)
    model = TokenHMREngine(cfg, synth.make_state_dict(cfg, W), synth.make_smpl(cfg, S), device=cuda_dev)
    out = model({"img": synth.make_images(B, cfg, I)})
    t = lambda k: torch.from_numpy(g[k])
    errs = {k: rel_err(out[k], t(k)) for k in ("pred_cam", "pred_cam_t", "pred_keypoints_3d", "pred_keypoints_2d")}
    errs["pred_vertices"] = rel_err(out["pred_vertices"][:, ::stride], t("pred_vertices_sub"))
    for k in ("global_orient", "body_pose", "betas"):
        errs[k] = rel_err(out["pred_smpl_params"][k], t(k))
    print("[regression release] B=64 vs fp32 reference", {k: f"{v:.2e}" for k, v in errs.items()})
    for k, v in errs.items():
        assert v < 2e-3, (k, v)


def test_strict_mode_vs_fp32_golden(cuda_dev, golden_dir):
    """Split-fp16 contractions (strict) against the live reference's fp32 tiny forward: vertices and keypoints 1e-4."""
    from tokenhmr_b200 import synth
    from tokenhmr_b200.config import tiny_config
    from tokenhmr_b200.engine import TokenHMREngine
    g = np.load(golden_dir / "forward_regression_tiny_d2.npz")
    cfg = tiny_config(vit_depth=2, head=REG)
    model = TokenHMREngine(cfg, synth.make_state_dict(cfg, 1234), synth.make_smpl(cfg, 3), device=cuda_dev,
                           use_cuda_graph=False, strict=True)
    out = model({"img": synth.make_images(2, cfg, 0)})
    t = lambda k: torch.from_numpy(g[k])
    errs = {k: rel_err(out[k], t(k)) for k in ("pred_keypoints_3d", "pred_keypoints_2d", "pred_cam")}
    errs["pred_vertices"] = rel_err(out["pred_vertices"], t("pred_vertices_sub"))
    print("[regression strict] vs fp32 reference", {k: f"{v:.2e}" for k, v in errs.items()})
    for k, v in errs.items():
        assert v < 1e-4, (k, v)


# FP8 mode (the ViT's QKV / fc1 / fc2 on e4m3) with the regression head: depth 32, B = 64, against the live reference's
# fp32 outputs.  Measured on an H100 80GB HBM3 at 700 W: pred_cam 5.8e-3, pred_cam_t 3.2e-3, keypoints_3d 1.2e-2,
# keypoints_2d 8.2e-3, vertices 1.7e-2 (every 16th vertex).  Pinned with a 2x margin.
FP8_TOL_REGRESSION = {"pred_cam": 1.2e-2, "pred_cam_t": 6.4e-3, "pred_keypoints_3d": 2.4e-2, "pred_vertices": 3.5e-2,
                      "pred_keypoints_2d": 1.6e-2}


def test_fp8_mode_vs_fp32_golden(cuda_dev, golden_dir):
    from tokenhmr_b200 import synth
    from tokenhmr_b200.config import TokenHMRConfig
    from tokenhmr_b200.engine import TokenHMREngine
    g = np.load(golden_dir / "forward_regression_release_d32.npz")
    W, S, I, B, _, _, stride = (int(v) for v in g["meta"])
    cfg = TokenHMRConfig(head=REG)
    model = TokenHMREngine(cfg, synth.make_state_dict(cfg, W), synth.make_smpl(cfg, S), device=cuda_dev, fp8=True)
    out = model({"img": synth.make_images(B, cfg, I)})
    assert all(torch.isfinite(v).all() for v in out.values() if isinstance(v, torch.Tensor))
    t = lambda k: torch.from_numpy(g[k])
    errs = {k: rel_err(out[k], t(k)) for k in ("pred_cam", "pred_cam_t", "pred_keypoints_3d", "pred_keypoints_2d")}
    errs["pred_vertices"] = rel_err(out["pred_vertices"][:, ::stride], t("pred_vertices_sub"))
    print("[regression fp8] B=64 vs fp32 reference", {k: f"{v:.2e}" for k, v in errs.items()})
    for k, v in errs.items():
        assert v < FP8_TOL_REGRESSION[k], (k, v)


def _graph_kernel_nodes(model, B: int) -> int:
    """Kernel nodes of the CUDA graph one forward captures (driver API: cuGraphGetNodes / cuGraphNodeGetType).  Unlike a
    torch.profiler trace, a captured graph cannot drop launches: on the GPU hosts the profiler's CUDA activity records
    were seen to lose kernels (135 of 136, or all of them) after several profiling sessions in one process."""
    cu = ctypes.CDLL("libcuda.so.1")
    st = model._state(B, False)
    g = torch.cuda.CUDAGraph(keep_graph=True)
    with torch.cuda.graph(g):
        model._launch(st, B)
    graph = ctypes.c_void_p(g.raw_cuda_graph())
    n = ctypes.c_size_t(0)
    assert cu.cuGraphGetNodes(graph, None, ctypes.byref(n)) == 0
    nodes = (ctypes.c_void_p * n.value)()
    assert cu.cuGraphGetNodes(graph, nodes, ctypes.byref(n)) == 0
    kinds = []
    for node in nodes:
        t = ctypes.c_int(-1)
        assert cu.cuGraphNodeGetType(ctypes.c_void_p(node), ctypes.byref(t)) == 0
        kinds.append(t.value)
    return kinds.count(0)                                  # CU_GRAPH_NODE_TYPE_KERNEL


@pytest.mark.parametrize("mode", ["default", "fp8", "strict"])
def test_num_launches_counts_the_kernels_of_a_forward(cuda_dev, tiny, mode):
    """num_launches() equals the kernels one forward launches, counted in the CUDA graph it captures, in every mode, and
    the step labels cover the new read-out GEMM and none of the token head's classifier or tokenizer steps."""
    from tokenhmr_b200 import synth
    from tokenhmr_b200.engine import TokenHMREngine
    cfg, sd, smpl, _ = tiny
    kw = {"default": {}, "fp8": {"fp8": True}, "strict": {"strict": True}}[mode]
    model = TokenHMREngine(cfg, sd, smpl, device=cuda_dev, use_cuda_graph=False, **kw)
    B = 3
    img = synth.make_images(B, cfg, seed=B).cuda()
    model({"img": img})                                    # builds the plans
    torch.cuda.synchronize()
    assert _graph_kernel_nodes(model, B) == model.num_launches()
    names = [n for n, *_ in model.profile(img)]
    assert "head.readout_gemm" in names and not any(n.startswith(("cls.", "tok.")) for n in names)


def test_workspace_holds_no_classifier_or_tokenizer(cuda_dev, tiny, built_lib):
    """At B = 64 the token head's fp32 logits and probabilities alone are 2 x 84 MB: the regression engine's workspace is
    smaller than the token engine's by at least that, in both the default and the strict mode."""
    from tokenhmr_b200 import synth
    from tokenhmr_b200.config import tiny_config
    from tokenhmr_b200.engine import TokenHMREngine
    cfg, sd, smpl, model = tiny
    tcfg = tiny_config(vit_depth=2)
    token = TokenHMREngine(tcfg, synth.make_state_dict(tcfg), smpl, device=cuda_dev, use_cuda_graph=False)
    logits = 2 * 64 * tcfg.token_num * tcfg.token_class_num * 4
    for a, b in ((model, token),):
        assert built_lib.thmr_engine_workspace_bytes(b._h, 64) - built_lib.thmr_engine_workspace_bytes(a._h, 64) > logits
    strict = TokenHMREngine(cfg, sd, smpl, device=cuda_dev, use_cuda_graph=False, strict=True)
    tstrict = TokenHMREngine(tcfg, synth.make_state_dict(tcfg), smpl, device=cuda_dev, use_cuda_graph=False, strict=True)
    assert built_lib.thmr_engine_workspace_bytes(tstrict._h, 64) - built_lib.thmr_engine_workspace_bytes(strict._h, 64) > logits


def test_token_engine_is_unaffected_by_a_regression_engine(cuda_dev, tiny):
    """A token engine built and run next to a regression engine computes bit for bit what a token engine built alone
    computes, launch count included."""
    from tokenhmr_b200 import synth
    from tokenhmr_b200.config import tiny_config
    from tokenhmr_b200.engine import TokenHMREngine
    tcfg = tiny_config(vit_depth=2)
    tsd, smpl = synth.make_state_dict(tcfg), synth.make_smpl(tcfg)
    img = synth.make_images(5, tcfg, seed=31)
    alone = TokenHMREngine(tcfg, tsd, smpl, device=cuda_dev, use_cuda_graph=False)
    want = {k: v.clone() for k, v in alone({"img": img}, return_taps=True).items() if isinstance(v, torch.Tensor)}
    n_alone = alone.num_launches()
    del alone
    cfg, _, _, reg = tiny
    token = TokenHMREngine(tcfg, tsd, smpl, device=cuda_dev, use_cuda_graph=False)
    reg({"img": img})
    got = token({"img": img}, return_taps=True)
    reg({"img": img})
    assert set(got) == set(want) | {"pred_smpl_params"}
    for k, v in want.items():
        assert torch.equal(got[k], v), k
    assert token.num_launches() == n_alone and reg.num_launches() < n_alone


def test_gather_logits_is_refused(tiny):
    from tokenhmr_b200 import _lib
    from tokenhmr_b200.dist import ShardedTokenHMR
    from tokenhmr_b200.engine import ShardSpec
    cfg, _, _, model = tiny
    with pytest.raises(_lib.ThmrError, match="cls_logits_softmax"):
        ShardedTokenHMR(model, transport="torch", gather_logits=True)
    with pytest.raises(_lib.ThmrError, match="cls_logits_softmax"):
        model({"img": torch.zeros(1, 3, 256, 256)}, shard=ShardSpec(0, 1, 0, 1, True))

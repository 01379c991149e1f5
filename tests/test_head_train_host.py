"""Training HMR 2.0's regression head, on the host: the C library's parameter list against the checkpoint layout and the
live reference head's state_dict, the fp64 restatement's autograd against the gradients of the live reference head
(tests/golden/regression_head_grads.npz, scripts/regression_grads_golden.py), and the rejection table of
RegressionHead and of the C entry points (each descriptor check runs before any CUDA call)."""
import ctypes

import numpy as np
import pytest
import torch

from scripts import regression_grads_golden as G
from tokenhmr_b200 import synth
from tokenhmr_b200._lib import ThmrError
from tokenhmr_b200.config import tiny_config

REG = "transformer_decoder"


def _cfg():
    return tiny_config(vit_depth=2, head=REG)


def test_param_info_lists_the_checkpoint_layout(built_lib):
    from tokenhmr_b200.heads import param_layout
    cfg = _cfg()
    layout, total = param_layout(cfg.dec_depth, cfg.dec_heads, cfg.dec_mlp_dim)
    sd = synth.make_state_dict(cfg)
    want = {k[len("smpl_head."):]: tuple(v.shape) for k, v in sd.items()
            if k.startswith("smpl_head.") and not k.startswith("smpl_head.init_")}
    assert {n: s for n, s, _ in layout} == want
    assert len(layout) == len(want)
    ends = 0
    for _, shape, off in layout:
        assert off % 64 == 0 and off >= ends
        ends = off + int(np.prod(shape))
    assert total >= ends and total - ends < 64
    assert 39_000_000 < sum(int(np.prod(s)) for _, s, _ in layout) < 40_000_000     # the release decoder's 39.5 M


def test_state_dict_keys_equal_the_live_reference_head():
    from oracle import ref_import
    from oracle import regression_oracle as R
    if not ref_import.available():
        pytest.skip("reference checkout not configured (TOKENHMR_REFERENCE)")
    from tokenhmr_b200.heads import param_layout
    cfg = _cfg()
    live = R.build_regression_head(ref_import.load_modules(), synth.make_state_dict(cfg), cfg)
    layout, _ = param_layout(cfg.dec_depth, cfg.dec_heads, cfg.dec_mlp_dim)
    assert [n for n, _, _ in layout] == [n for n, _ in live.named_parameters()]     # also the order
    assert {n for n, _, _ in layout} | {"init_body_pose", "init_betas", "init_cam"} == set(live.state_dict())


def test_restatement_autograd_matches_the_reference_golden(golden_dir):
    """oracle.regression_oracle.regression_head_forward in fp64 with autograd (the reference of the GPU tests) against the
    live reference head's fp64 gradients: 1e-10 relative."""
    from oracle import regression_oracle as R
    from oracle import tokenhmr_oracle as O
    g = np.load(golden_dir / "regression_head_grads.npz")
    assert list(g["meta"]) == [G.W_SEED, G.FEAT_SEED, G.UP_SEED, G.B, G.NPROJ, G.SAMPLE]
    cfg = _cfg()
    sd = {k: v.double().requires_grad_("init_" not in k) for k, v in synth.make_state_dict(cfg, G.W_SEED).items()
          if k.startswith("smpl_head.")}
    feats, up = G.inputs(cfg)
    params, cam, _ = R.regression_head_forward(sd, feats.flatten(2).transpose(1, 2), cfg, O.Numerics(False))
    rot = torch.cat([params["global_orient"], params["body_pose"]], 1)
    rel = lambda a, b: float(np.abs(np.asarray(a) - b).max() / max(np.abs(b).max(), 1e-300))
    assert rel(rot.detach().numpy(), g["rotmats"]) < 1e-10
    assert rel(params["betas"].detach().numpy(), g["betas"]) < 1e-10
    assert rel(cam.detach().numpy(), g["cam"]) < 1e-10
    loss = (rot * up[0]).sum() + (params["betas"] * up[1]).sum() + (cam * up[2]).sum()
    names = [k for k, v in sd.items() if v.requires_grad]
    grads = torch.autograd.grad(loss, [sd[k] for k in names], allow_unused=True)
    seen = 0
    for k, gr in zip(names, grads):
        name = k[len("smpl_head."):]
        gr = torch.zeros_like(sd[k]) if gr is None else gr
        proj = [(gr * G.projection_matrix(name, i, gr.shape)).sum().item() for i in range(G.NPROJ)]
        assert rel(proj, g["proj/" + name]) < 1e-10, name
        assert rel(gr.norm().item(), g["norm/" + name]) < 1e-10, name
        if not G.is_matrix(gr.shape):
            assert rel(G.sampled(gr).numpy(), g["grad/" + name]) < 1e-10, name
        seen += 1
    assert seen == len([k for k in g.files if k.startswith("proj/")])
    # the reference leaves to_token_embedding.weight without a gradient (its input is zero): stored as zeros
    assert float(g["norm/transformer.to_token_embedding.weight"]) == 0.0


@pytest.fixture
def sd():
    return synth.make_state_dict(_cfg())


def test_regression_head_rejections(sd, built_lib):
    from tokenhmr_b200.heads import RegressionHead
    with pytest.raises(ThmrError, match="token head's is not built"):
        RegressionHead(tiny_config(vit_depth=2), synth.make_state_dict(tiny_config(vit_depth=2)), "cuda")
    for key in ("dropout", "emb_dropout"):
        y = {"MODEL": {"SMPL_HEAD": {"TYPE": REG, "TRANSFORMER_DECODER": {key: 0.1}}}}
        with pytest.raises(ThmrError, match=f"TRANSFORMER_DECODER.{key}"):
            RegressionHead(_cfg(), sd, "cuda", model_cfg=y)
    with pytest.raises(ThmrError, match="no CPU fallback"):
        RegressionHead(_cfg(), sd, "cpu", model_cfg={"MODEL": {"SMPL_HEAD": {"TRANSFORMER_DECODER": {"dropout": 0.0}}}})


def _desc(**kw):
    from tokenhmr_b200 import _lib
    d = _lib.RegHeadDesc()
    d.B, d.depth, d.heads, d.mlp_dim = 2, 6, 8, 1024
    fake = 1 << 20                      # never dereferenced: every case below fails a host-side check first
    for n in ("params", "grads", "init_body_pose", "init_betas", "init_cam", "feats", "pose6d", "betas", "cam",
              "rotmats", "workspace"):
        setattr(d, n, fake)
    d.workspace_bytes = 1 << 40
    for k, v in kw.items():
        setattr(d, k, v)
    return d


@pytest.mark.parametrize("fields,msg", [
    ({"B": 0}, "B=0"),
    ({"heads": 9}, "unsupported dims"),
    ({"depth": 0}, "unsupported dims"),
    ({"mlp_dim": 0}, "unsupported dims"),
    ({"params": None}, "null input pointer"),
    ({"feats": None}, "null input pointer"),
    ({"init_cam": None}, "null input pointer"),
    ({"workspace": None}, "null workspace"),
    ({"workspace_bytes": 1024}, "workspace too small"),
    ({"workspace": (1 << 20) + 4}, "aligned"),
])
def test_c_descriptor_rejections(built_lib, fields, msg):
    for fn, extra in ((built_lib.thmr_reg_head_train_forward, {}), (built_lib.thmr_reg_head_backward, {})):
        d = _desc(**fields, **extra)
        assert fn(ctypes.byref(d)) == -1
        assert msg.encode() in built_lib.thmr_last_error()
    assert built_lib.thmr_reg_head_train_forward(None) == -1
    d = _desc(rotmats=None)
    assert built_lib.thmr_reg_head_train_forward(ctypes.byref(d)) == -1 and b"null output" in built_lib.thmr_last_error()
    d = _desc(grads=None)
    assert built_lib.thmr_reg_head_backward(ctypes.byref(d)) == -1 and b"null gradient" in built_lib.thmr_last_error()


def test_workspace_and_info_queries(built_lib):
    assert built_lib.thmr_reg_head_workspace_bytes(0, 6, 8, 1024) == 0
    assert built_lib.thmr_reg_head_workspace_bytes(48, 6, 9, 1024) == 0
    w48, w96 = (built_lib.thmr_reg_head_workspace_bytes(b, 6, 8, 1024) for b in (48, 96))
    assert 0 < w48 < w96
    name, nd = ctypes.c_char_p(), ctypes.c_int()
    shape, off = (ctypes.c_int64 * 3)(), ctypes.c_int64()
    assert built_lib.thmr_reg_head_param_info(6, 8, 1024, 10 ** 6, ctypes.byref(name), ctypes.byref(nd), shape,
                                              ctypes.byref(off)) == -1
    assert b"outside" in built_lib.thmr_last_error()
    assert built_lib.thmr_reg_head_param_info(6, 8, 1024, 0, ctypes.byref(name), ctypes.byref(nd), shape,
                                              ctypes.byref(off)) == 0
    assert name.value == b"transformer.pos_embedding" and nd.value == 3 and list(shape) == [1, 1, 1024]

"""Training TokenHMR's token head, on the host: the C library's trainable and frozen layouts against the checkpoint and
the live reference head, the fp64 restatement (oracle.tokenhmr_oracle.head_forward) with autograd against the gradients
of the live reference head at both class_pred_layer scales (tests/golden/token_head_grads.npz,
scripts/token_grads_golden.py), and the rejection tables of TokenHead and of the C entry points (each descriptor check
runs before any CUDA call)."""
import ctypes
import dataclasses

import numpy as np
import pytest
import torch

from scripts import token_grads_golden as G
from tokenhmr_b200 import synth
from tokenhmr_b200._lib import ThmrError
from tokenhmr_b200.config import tiny_config


def _cfg():
    return tiny_config(vit_depth=2)


def test_trainable_layout_is_the_checkpoint_layout(built_lib):
    from tokenhmr_b200.heads import token_param_layout
    cfg = _cfg()
    layout, total = token_param_layout(cfg.dec_depth, cfg.dec_heads, cfg.dec_mlp_dim)
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


def test_the_decoder_part_is_shared_with_the_regression_head(built_lib):
    from tokenhmr_b200.heads import param_layout, token_param_layout
    reg, _ = param_layout(6, 8, 1024)
    tok, _ = token_param_layout(6, 8, 1024)
    dec = [e for e in reg if e[0].startswith("transformer.")]
    assert tok[:len(dec)] == dec


def test_frozen_layout_covers_what_the_tokenizer_decoder_reads(built_lib):
    from oracle import tokenhmr_oracle as O
    from tokenhmr_b200.heads import tokenizer_layout
    cfg = _cfg()
    layout, total = tokenizer_layout()
    sd = synth.make_state_dict(cfg)
    read = set()

    class Spy(dict):
        def __getitem__(self, k):
            read.add(k)
            return dict.__getitem__(self, k)

    O.tokenizer_decode(Spy(sd), torch.full((1, cfg.token_num, cfg.nb_code), 1.0 / cfg.nb_code), cfg, O.Numerics(False))
    assert {n for n, _, _ in layout} == read
    for name, shape, off in layout:
        assert tuple(sd[name].shape) == shape and off % 64 == 0
    assert total >= max(off + int(np.prod(s)) for _, s, off in layout)


def test_state_dict_keys_equal_the_live_reference_head():
    from oracle import ref_import
    if not ref_import.available():
        pytest.skip("reference checkout not configured (TOKENHMR_REFERENCE)")
    from tokenhmr_b200.heads import token_param_layout
    cfg = _cfg()
    live = ref_import.build_head(ref_import.load_modules(), synth.make_state_dict(cfg), cfg)
    layout, _ = token_param_layout(cfg.dec_depth, cfg.dec_heads, cfg.dec_mlp_dim)
    assert [n for n, _, _ in layout] == [n for n, _ in live.named_parameters()]     # also the order
    assert {n for n, _, _ in layout} | {"init_body_pose", "init_betas", "init_cam"} == set(live.state_dict())


@pytest.mark.parametrize("tag,scale", G.SETS)
def test_restatement_autograd_matches_the_reference_golden(golden_dir, tag, scale):
    """oracle.tokenhmr_oracle.head_forward in fp64 with autograd (the reference of the GPU tests) against the live
    reference head's fp64 outputs and gradients: 1e-10 relative."""
    from oracle import tokenhmr_oracle as O
    g = np.load(golden_dir / "token_head_grads.npz")
    assert list(g["meta"]) == [G.W_SEED, G.FEAT_SEED, G.UP_SEED, G.B, G.NPROJ, G.SAMPLE, G.PROBS_SAMPLE]
    cfg = _cfg()
    sd = {k: v.double().requires_grad_(k.startswith("smpl_head.") and "init_" not in k)
          for k, v in G.state_dict(cfg, scale).items() if k.startswith(("smpl_head.", "tokenizer."))}
    feats, up = G.inputs(cfg)
    params, cam, aux = O.head_forward(sd, feats.flatten(2).transpose(1, 2), cfg, O.Numerics(False))
    rot = torch.cat([params["global_orient"], params["body_pose"]], 1)
    probs = aux["cls_logits_softmax"]
    rel = lambda a, b: float(np.abs(np.asarray(a) - b).max() / max(np.abs(b).max(), 1e-300))
    assert rel(rot.detach().numpy(), g[tag + "rotmats"]) < 1e-10
    assert rel(params["betas"].detach().numpy(), g[tag + "betas"]) < 1e-10
    assert rel(cam.detach().numpy(), g[tag + "cam"]) < 1e-10
    loss = G.loss_of(rot, params["betas"], cam, probs, up)
    names = [k for k, v in sd.items() if v.requires_grad]
    grads = torch.autograd.grad(loss, [sd[k] for k in names], allow_unused=True)
    tab = G.table(g, tag)
    seen = 0
    for k, gr in [(tag + "cls_logits_softmax", probs.detach())] + \
                 [(tag + k[len("smpl_head."):], gr) for k, gr in zip(names, grads)]:
        gr = torch.zeros_like(sd["smpl_head." + k[len(tag):]]) if gr is None else gr
        want_proj, want_norm, want_sampled = tab[k]
        proj = [(gr * G.projection_matrix(k, i, gr.shape)).sum().item() for i in range(G.NPROJ)]
        assert rel(proj, want_proj) < 1e-10, k
        assert rel(gr.norm().item(), want_norm) < 1e-10, k
        if want_sampled is not None:
            every = G.PROBS_SAMPLE if k.endswith("cls_logits_softmax") else G.SAMPLE
            assert rel(gr.reshape(-1)[::every].numpy(), want_sampled) < 1e-10, k
        seen += 1
    assert seen == len(tab)


@pytest.fixture
def sd():
    return synth.make_state_dict(_cfg())


def test_token_head_rejections(sd, built_lib):
    from tokenhmr_b200.heads import RegressionHead, TokenHead
    with pytest.raises(ThmrError, match="trains the 'token' head"):
        TokenHead(tiny_config(head="transformer_decoder"), sd, "cuda")
    with pytest.raises(ThmrError, match="token head's is not built by it; use TokenHead"):
        RegressionHead(_cfg(), sd, "cuda")
    for k, v in (("token_class_num", 1024), ("cls_blocks", 2), ("tok_width", 256), ("token_num", 80)):
        with pytest.raises(ThmrError, match=f"{k} = {v}; the CUDA token head is built for the release"):
            TokenHead(dataclasses.replace(_cfg(), **{k: v}), sd, "cuda")
    for key in ("dropout", "emb_dropout"):
        y = {"MODEL": {"SMPL_HEAD": {"TRANSFORMER_DECODER": {key: 0.1}}}}
        with pytest.raises(ThmrError, match=f"TokenHead: MODEL.SMPL_HEAD.TRANSFORMER_DECODER.{key}"):
            TokenHead(_cfg(), sd, "cuda", model_cfg=y)
    with pytest.raises(ThmrError, match="TokenHead: needs a CUDA device"):
        TokenHead(_cfg(), sd, "cpu")


def _desc(**kw):
    from tokenhmr_b200 import _lib
    d = _lib.TokHeadDesc()
    d.B, d.depth, d.heads, d.mlp_dim = 2, 6, 8, 1024
    fake = 1 << 20                      # never dereferenced: every case below fails a host-side check first
    for n in ("params", "grads", "tokenizer", "init_body_pose", "init_betas", "init_cam", "feats", "pose6d", "betas",
              "cam", "rotmats", "cls_probs", "workspace"):
        setattr(d, n, fake)
    d.workspace_bytes = 1 << 40
    for k, v in kw.items():
        setattr(d, k, v)
    return d


@pytest.mark.parametrize("fields,msg", [
    ({"B": 0}, "B=0"),
    ({"B": -3}, "B=-3"),
    ({"heads": 9}, "unsupported dims"),
    ({"depth": 0}, "unsupported dims"),
    ({"depth": 65}, "unsupported dims"),
    ({"mlp_dim": 0}, "unsupported dims"),
    ({"params": None}, "null input pointer"),
    ({"tokenizer": None}, "null input pointer"),
    ({"feats": None}, "null input pointer"),
    ({"init_body_pose": None}, "null input pointer"),
    ({"workspace": None}, "null workspace"),
    ({"workspace_bytes": 1024}, "workspace too small"),
    ({"workspace": (1 << 20) + 4}, "aligned"),
    ({"tokenizer": (1 << 20) + 4}, "aligned"),
    ({"params": (1 << 20) + 8}, "aligned"),
])
def test_c_descriptor_rejections(built_lib, fields, msg):
    for fn in (built_lib.thmr_tok_head_train_forward, built_lib.thmr_tok_head_backward):
        d = _desc(**fields)
        assert fn(ctypes.byref(d)) == -1
        assert msg.encode() in built_lib.thmr_last_error()
    assert built_lib.thmr_tok_head_train_forward(None) == -1
    assert built_lib.thmr_tok_head_backward(None) == -1


@pytest.mark.parametrize("field", ["betas", "cam", "rotmats", "cls_probs"])
def test_c_rejects_null_outputs_and_gradients(built_lib, field):
    d = _desc(**{field: None})
    assert built_lib.thmr_tok_head_train_forward(ctypes.byref(d)) == -1
    assert b"null output" in built_lib.thmr_last_error()
    d = _desc(grads=None)
    assert built_lib.thmr_tok_head_backward(ctypes.byref(d)) == -1 and b"null gradient" in built_lib.thmr_last_error()
    d = _desc(cls_probs=None)
    assert built_lib.thmr_tok_head_backward(ctypes.byref(d)) == -1 and b"null cls_probs" in built_lib.thmr_last_error()
    d = _desc(grads=(1 << 20) + 4)
    assert built_lib.thmr_tok_head_backward(ctypes.byref(d)) == -1 and b"aligned" in built_lib.thmr_last_error()


def test_workspace_and_info_queries(built_lib):
    W = built_lib.thmr_tok_head_workspace_bytes
    assert W(0, 6, 8, 1024) == 0 and W(48, 6, 9, 1024) == 0 and W(48, 0, 8, 1024) == 0
    w1, w48, w130 = (W(b, 6, 8, 1024) for b in (1, 48, 130))
    assert 0 < w1 < w48 < w130
    assert w48 - built_lib.thmr_reg_head_workspace_bytes(48, 6, 8, 1024) > 48 * 160 * 2048 * 4   # holds dP
    name, nd = ctypes.c_char_p(), ctypes.c_int()
    shape, off = (ctypes.c_int64 * 3)(), ctypes.c_int64()
    n, total = ctypes.c_int(), ctypes.c_int64()
    assert built_lib.thmr_tok_head_num_params(6, 8, 1024, ctypes.byref(n), ctypes.byref(total)) == 0
    for i in (-1, n.value, 10 ** 6):
        assert built_lib.thmr_tok_head_param_info(6, 8, 1024, i, ctypes.byref(name), ctypes.byref(nd), shape,
                                                  ctypes.byref(off)) == -1
        assert b"outside" in built_lib.thmr_last_error()
    assert built_lib.thmr_tok_head_param_info(6, 8, 1024, n.value - 1, ctypes.byref(name), ctypes.byref(nd), shape,
                                              ctypes.byref(off)) == 0
    assert name.value == b"decpose.class_pred_layer.bias" and nd.value == 1 and shape[0] == 2048
    assert built_lib.thmr_tok_head_param_info(6, 9, 1024, 0, ctypes.byref(name), ctypes.byref(nd), shape,
                                              ctypes.byref(off)) == -1
    assert b"unsupported dims" in built_lib.thmr_last_error()
    assert built_lib.thmr_tok_head_tokenizer_num(ctypes.byref(n), ctypes.byref(total)) == 0
    for i in (-1, n.value):
        assert built_lib.thmr_tok_head_tokenizer_info(i, ctypes.byref(name), ctypes.byref(nd), shape,
                                                      ctypes.byref(off)) == -1
        assert b"outside" in built_lib.thmr_last_error()
    assert built_lib.thmr_tok_head_tokenizer_info(n.value - 1, ctypes.byref(name), ctypes.byref(nd), shape,
                                                  ctypes.byref(off)) == 0
    assert name.value == b"tokenizer.quantizer.codebook" and list(shape[:2]) == [2048, 256]


def test_descriptor_structs_match_their_ctypes_mirrors(tmp_path):
    """thmr_tok_head_desc and thmr_reg_head_desc have the size the C compiler gives them, so a field inserted on one
    side only cannot drift silently."""
    import shutil
    import subprocess
    from pathlib import Path
    from tokenhmr_b200 import _lib
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("no C compiler")
    header = Path(__file__).resolve().parent.parent / "include" / "tokenhmr_b200.h"
    pairs = [("thmr_tok_head_desc", _lib.TokHeadDesc), ("thmr_reg_head_desc", _lib.RegHeadDesc)]
    body = "".join(f'  printf("%s %zu\\n", "{n}", sizeof({n}));\n' for n, _ in pairs)
    src = tmp_path / "sizes.c"
    src.write_text(f'#include <stdio.h>\n#include "{header}"\nint main(void) {{\n{body}  return 0;\n}}\n')
    exe = tmp_path / "sizes"
    subprocess.run([gcc, "-std=c99", "-Wall", "-Werror", "-o", str(exe), str(src)], check=True, capture_output=True)
    out = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()
    sizes = dict(zip(out[0::2], map(int, out[1::2])))
    for name, cls in pairs:
        assert sizes[name] == ctypes.sizeof(cls), f"{name}: C {sizes[name]} vs ctypes {ctypes.sizeof(cls)}"

"""HMR 2.0's regression head (MODEL.SMPL_HEAD.TYPE: transformer_decoder) on the host: which configurations are accepted,
how the loader tells the two heads apart, that the real checkpoint's key layout packs completely, and that the oracle's
restatement of the head equals the reference module."""
import copy

import numpy as np
import pytest
import torch
import yaml

from tokenhmr_b200 import checkpoint as C
from tokenhmr_b200 import synth
from tokenhmr_b200._lib import ThmrError
from tokenhmr_b200.config import TokenHMRConfig, tiny_config

REG = "transformer_decoder"
_TOKEN_YAML = {
    "MODEL": {"IMAGE_SIZE": 256, "BBOX_SHAPE": [192, 256], "BACKBONE": {"TYPE": "vit"},
              "SMPL_HEAD": {"TYPE": "token", "TOKENIZER": {"TOKEN_CODE_DIM": 256, "TOKEN_NUM": 160, "TOKEN_CLASS_NUM": 2048,
                                                          "TOKENIZER_TYPE": "Vanilla"},
                            "TRANSFORMER_DECODER": {"depth": 6, "heads": 8, "mlp_dim": 1024, "dim_head": 64, "norm": "layer",
                                                    "context_dim": 1280}}},
    "SMPL": {"NUM_BODY_JOINTS": 23, "GENDER": "neutral"}, "EXTRA": {"FOCAL_LENGTH": 5000},
}
# HMR 2.0's model_config.yaml: a transformer_decoder head and no TOKENIZER block
_REG_YAML = copy.deepcopy(_TOKEN_YAML)
_REG_YAML["MODEL"]["SMPL_HEAD"] = {"TYPE": REG, "IN_CHANNELS": 2048,
                                   "TRANSFORMER_DECODER": dict(_TOKEN_YAML["MODEL"]["SMPL_HEAD"]["TRANSFORMER_DECODER"])}


def _write(tmp_path, y, name="model_config.yaml"):
    p = tmp_path / name
    p.write_text(yaml.safe_dump(y))
    return str(p)


def _with(y, key, value):
    y = copy.deepcopy(y)
    y["MODEL"]["SMPL_HEAD"][key] = value
    return y


@pytest.mark.parametrize("base", ["token", REG])
@pytest.mark.parametrize("key,value,ref", [
    ("IEF_ITERS", 1, None), ("TRANSFORMER_INPUT", "zero", None), ("JOINT_REP", "6d", None),
    ("IEF_ITERS", 3, {"token": "token_head.py:86", REG: "smpl_head.py:70"}),
    ("TRANSFORMER_INPUT", "mean_shape", {"token": "token_head.py:29", REG: "smpl_head.py:21"}),
    ("JOINT_REP", "aa", {"token": "token_head.py:23", REG: "smpl_head.py:17"}),
])
def test_accept_reject_table_for_both_heads(tmp_path, base, key, value, ref):
    """The regression head is accepted with exactly the token head's three restrictions; each rejection cites the line of
    the head's own file that reads the key."""
    y = _with(_TOKEN_YAML if base == "token" else _REG_YAML, key, value)
    p = _write(tmp_path, y)
    if ref is None:
        cfg = C.config_from_files(p, {"NB_CODE": 2048, "CODE_DIM": 256} if base == "token" else None)
        assert cfg == TokenHMRConfig(head=base)
    else:
        with pytest.raises(ThmrError, match="unsupported configuration") as e:
            C.config_from_files(p, None)
        assert ref[base] in str(e.value)


def test_other_head_types_stay_rejected(tmp_path):
    for t in ("hmr", "mlp"):
        with pytest.raises(ThmrError, match="unsupported configuration: MODEL.SMPL_HEAD.TYPE"):
            C.config_from_files(_write(tmp_path, _with(_REG_YAML, "TYPE", t)), None)
    y = copy.deepcopy(_REG_YAML)
    del y["MODEL"]["SMPL_HEAD"]["TYPE"]                      # build_smpl_head's default 'hmr' raises in the reference too
    with pytest.raises(ThmrError, match="'hmr'"):
        C.config_from_files(_write(tmp_path, y), None)
    with pytest.raises(ValueError):
        TokenHMRConfig(head="hmr")


def test_regression_yaml_has_no_tokenizer_block(tmp_path):
    """The regression head needs no TOKENIZER block (nor a tokenizer's hparams), and refuses one: a TokenHMR yaml whose
    TYPE was changed to transformer_decoder mixes the two heads."""
    assert C.config_from_files(_write(tmp_path, _REG_YAML), None) == TokenHMRConfig(head=REG)
    y = copy.deepcopy(_TOKEN_YAML)
    y["MODEL"]["SMPL_HEAD"]["TYPE"] = REG
    with pytest.raises(ThmrError, match="unsupported configuration: MODEL.SMPL_HEAD.TOKENIZER with TYPE"):
        C.config_from_files(_write(tmp_path, y), None)


def _model_sd(cfg):
    return {k: v for k, v in synth.make_state_dict(cfg).items() if not k.startswith("tokenizer.")}


def test_head_is_inferred_from_the_keys():
    assert C.infer_head(_model_sd(tiny_config(vit_depth=1, head=REG))) == REG
    assert C.infer_head(_model_sd(tiny_config(vit_depth=1))) == "token"
    with pytest.raises(ThmrError, match="found neither"):
        C.infer_head({"backbone.pos_embed": torch.zeros(1)})
    both = {**_model_sd(tiny_config(vit_depth=1)), "smpl_head.decpose.weight": torch.zeros(144, 1024)}
    with pytest.raises(ThmrError, match="found both"):
        C.infer_head(both)


def test_weights_checked_against_the_regression_config():
    cfg = tiny_config(vit_depth=1, head=REG)
    sd, smpl = synth.make_state_dict(cfg), synth.make_smpl(cfg)
    C.validate_against_weights(cfg, sd, smpl)
    for name, shape in (("decpose", (138, 1024)), ("decshape", (10, 512)), ("deccam", (4, 1024))):
        bad = dict(sd)
        bad[f"smpl_head.{name}.weight"] = torch.zeros(shape)
        with pytest.raises(ThmrError, match=f"smpl_head.{name}"):
            C.validate_against_weights(cfg, bad, smpl)
    with pytest.raises(ThmrError, match="holds a regression head"):
        C.validate_against_weights(tiny_config(vit_depth=1), sd, smpl)
    with pytest.raises(ThmrError, match="holds a token head"):
        C.validate_against_weights(cfg, synth.make_state_dict(tiny_config(vit_depth=1)), smpl)


def _files(tmp_path, cfg, sd, extra=None):
    from test_checkpoint import _write_smpl_pkl
    (tmp_path / "checkpoints").mkdir()
    (tmp_path / "body_models" / "smpl").mkdir(parents=True)
    ck = tmp_path / "checkpoints" / "hmr2.ckpt"
    torch.save({"state_dict": {**sd, **(extra or {})}}, ck)
    _write_smpl_pkl(tmp_path / "body_models" / "smpl", synth.make_smpl(cfg), cfg.num_verts)
    return str(ck)


def test_loader_never_opens_a_tokenizer_for_a_regression_checkpoint(tmp_path):
    """Everything up to the engine is loaded (the CPU device is refused only then) although the tokenizer path does not
    exist; the head comes from the keys, the depth and mesh size from the files."""
    cfg = tiny_config(vit_depth=1, head=REG)
    ck = _files(tmp_path, cfg, _model_sd(cfg))
    seen = {}
    real = C.validate_against_weights

    def spy(cfg_, sd_, smpl_):
        seen["cfg"], seen["keys"] = cfg_, set(sd_)
        return real(cfg_, sd_, smpl_)

    C.validate_against_weights = spy
    try:
        with pytest.raises(ThmrError, match="no CPU fallback"):
            C.load_tokenhmr(ck, tokenizer_path=str(tmp_path / "does-not-exist" / "tokenizer.pth"), device="cpu")
        with pytest.raises(ThmrError, match="no CPU fallback"):
            C.load_tokenhmr(ck, model_cfg=_write(tmp_path, _REG_YAML), device="cpu")   # default path, also absent
    finally:
        C.validate_against_weights = real
    assert seen["cfg"] == cfg
    assert not any(k.startswith("tokenizer.") for k in seen["keys"])


def test_yaml_that_disagrees_with_the_keys_is_refused(tmp_path):
    cfg = tiny_config(vit_depth=1, head=REG)
    ck = _files(tmp_path, cfg, _model_sd(cfg))
    with pytest.raises(ThmrError, match=r"says MODEL.SMPL_HEAD.TYPE 'token' but the checkpoint .* holds a "
                                        r"'transformer_decoder' head"):
        C.load_tokenhmr(ck, model_cfg=_write(tmp_path, _TOKEN_YAML), device="cpu")


def test_packer_reads_every_key_of_a_regression_checkpoint():
    """PackedWeights (here on the CPU) reads each backbone.* / smpl_head.* entry of a regression checkpoint and nothing
    else; the classifier and tokenizer pointers stay NULL."""
    from tokenhmr_b200.weights import PackedWeights
    cfg = tiny_config(vit_depth=2, head=REG)
    sd = _model_sd(cfg)
    pw = PackedWeights(sd, cfg, torch.device("cpu"))
    assert set(pw.keys_read) == set(sd)
    W = pw.struct
    assert not any(getattr(W, n) for n in ("mt_w", "mt_b", "mn_w", "cls_w", "cls_b", "codebook_t"))
    assert not W.mixer_host and not W.conv_out.w
    # read-out: decpose | decshape | deccam | 3 zero rows, fp16 [160, 1024]
    rw = next(t for t in pw._keep if t.data_ptr() == W.readout_w)
    assert tuple(rw.shape) == (160, cfg.dec_dim) and rw.dtype == torch.float16
    assert torch.equal(rw[:144], sd["smpl_head.decpose.weight"].half()) and not rw[157:].any()
    strict = PackedWeights(sd, cfg, torch.device("cpu"), strict=True)
    rs = next(t for t in strict._keep if t.data_ptr() == strict.struct.readout_w)
    assert tuple(rs.shape) == (160, 3 * cfg.dec_dim)


def test_reference_state_dict_layout_loads_completely(tmp_path):
    """The key layout of a real HMR 2.0 checkpoint, from the LIVE reference modules' own state_dict() (ViT +
    SMPLTransformerDecoderHead) with the discriminator and SMPL buffers a Lightning checkpoint also holds: the loader
    keeps exactly backbone.* / smpl_head.*, the head is inferred, and the packer reads every kept key."""
    from oracle import ref_import
    from oracle import regression_oracle as R
    from tokenhmr_b200.weights import PackedWeights
    if not ref_import.available():
        pytest.skip("reference checkout not configured (TOKENHMR_REFERENCE)")
    ns = ref_import.load_modules()
    cfg = tiny_config(vit_depth=2, head=REG)
    syn = synth.make_state_dict(cfg)
    live = {"backbone." + k: v for k, v in ref_import.build_backbone(ns, syn, cfg).state_dict().items()}
    live.update({"smpl_head." + k: v for k, v in R.build_regression_head(ns, syn, cfg).state_dict().items()})
    extra = {"discriminator.D_conv1.weight": torch.zeros(32, 9, 1, 1), "smpl.betas": torch.zeros(1, 10),
             "smpl.shapedirs": torch.zeros(4, 3, 10)}
    torch.save({"state_dict": {**live, **extra}}, tmp_path / "hmr2.ckpt")
    sd = C.load_lightning_state_dict(tmp_path / "hmr2.ckpt")
    assert set(sd) == set(live)
    assert C.infer_head(sd) == REG
    C.validate_against_weights(cfg, sd, synth.make_smpl(cfg))
    assert set(PackedWeights(sd, cfg, torch.device("cpu")).keys_read) == set(sd)


def test_oracle_restatement_equals_the_live_reference_head():
    from oracle import ref_import
    from oracle import regression_oracle as R
    from oracle import tokenhmr_oracle as O
    if not ref_import.available():
        pytest.skip("reference checkout not configured (TOKENHMR_REFERENCE)")
    ns = ref_import.load_modules()
    cfg = tiny_config(vit_depth=2, head=REG)
    sd = synth.make_state_dict(cfg)
    head = R.build_regression_head(ns, sd, cfg)
    feats = torch.randn(3, cfg.vit_dim, cfg.grid_h, cfg.grid_w, generator=torch.Generator().manual_seed(4))
    with torch.no_grad():
        params, cam, _ = head(feats)
        p2, cam2, _ = R.regression_head_forward(sd, feats.flatten(2).transpose(1, 2), cfg, O.Numerics(False))
    rel = lambda a, b: ((a - b).abs().max() / b.abs().max()).item()
    assert rel(cam2, cam) < 1e-6
    for k in ("global_orient", "body_pose", "betas"):
        assert rel(p2[k], params[k]) < 1e-6, k


def test_oracle_matches_the_regression_golden(golden_dir):
    """The fp32 restatement against the live reference's tiny forward (oracle/regression_oracle.py wrote the golden)."""
    from oracle import regression_oracle as R
    g = np.load(golden_dir / "forward_regression_tiny_d2.npz")
    cfg = tiny_config(vit_depth=2, head=REG)
    assert list(g["meta"][:4]) == [1234, 3, 0, 2]
    sd, smpl = synth.make_state_dict(cfg, 1234), synth.make_smpl(cfg, 3)
    with torch.no_grad():
        out = R.forward(sd, smpl, synth.make_images(2, cfg, 0), cfg, return_intermediates=True)
    assert "cls_logits_softmax" not in out
    t = lambda k: torch.from_numpy(g[k])
    torch.testing.assert_close(out["_vit_tokens"][:, ::8], t("vit_tokens_sub"), rtol=0, atol=2e-5)
    torch.testing.assert_close(out["pred_cam"], t("pred_cam"), rtol=0, atol=2e-6)
    for k in ("global_orient", "body_pose", "betas"):
        torch.testing.assert_close(out["pred_smpl_params"][k], t(k), rtol=0, atol=5e-6)
    for k in ("pred_keypoints_3d", "pred_keypoints_2d"):
        torch.testing.assert_close(out[k], t(k), rtol=1e-5, atol=2e-5)
    torch.testing.assert_close(out["pred_vertices"], t("pred_vertices_sub"), rtol=1e-5, atol=2e-5)

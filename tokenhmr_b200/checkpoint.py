"""On-disk formats either side of the path -> engine inputs (SURVEY §8 row f3).  Host glue only (file I/O, renaming,
dtype conversion); nothing here touches the GPU until the engine packs the result.

Formats, with the reference code that reads them today:
  * TokenHMR Lightning checkpoint  `torch.load(path)['state_dict']`, keys `backbone.*` / `smpl_head.*` next to
    training-only entries (discriminator, loss buffers); the frozen tokenizer is NOT in it (token_classifier.py:84-86
    hides it behind a Proxy, so it is always read from MODEL.TOKENIZER_CHECKPOINT_PATH)
        tokenhmr/lib/utils/misc.py:215-256 (prepare_statedict / load_pretrained)
  * tokenizer.pth  `{'net': {...}, 'hparams': <config object with .ARCH>}`
        tokenization/models/vanilla_pose_vqvae.py:258-301 (DecodeTokens), :304-346 (EncodeTokens)
  * SMPL_NEUTRAL.pkl  (python-2 pickle, latin1, chumpy arrays + a scipy.sparse J_regressor), read by smplx.SMPLLayer
        tokenhmr/lib/models/smpl_wrapper.py:10-25, tokenhmr/lib/models/tokenhmr.py:84-85
  * SMPL_to_J19.pkl  (pickled (19, 6890) array, `joint_regressor_extra`)      smpl_wrapper.py:22-23
  * model_config.yaml  (yacs dump)                                            tokenhmr/lib/models/__init__.py:3-26

chumpy, smplx, yacs and pytorch_lightning are not needed: pickles are read with an unpickler that maps classes of
missing modules onto inert stand-ins (a chumpy `Ch` keeps its array in state['x']; config nodes become attribute
dicts); scipy is optional (a sparse matrix stand-in rebuilds CSR/CSC/COO from the pickled state).
"""
from __future__ import annotations

import io
import pickle
from pathlib import Path
from typing import Any, Dict, Optional, Tuple

import numpy as np
import torch

from .config import SMPL_EXTRA_VERTEX_IDS, TokenHMRConfig


# ------------------------------------------------------------------------------------------- tolerant unpickling
class _Stub:
    """Instance of a class whose module is not installed: keeps whatever state the pickle carries."""

    def __init__(self, *a, **k):
        self._args, self._state = a, {}

    def __setstate__(self, state):
        if isinstance(state, tuple) and len(state) == 2 and isinstance(state[1], dict):   # (None, slots) form
            state = {**(state[0] or {}), **state[1]}
        self._state = state if isinstance(state, dict) else {"state": state}
        if isinstance(self._state, dict):
            self.__dict__.update({k: v for k, v in self._state.items() if isinstance(k, str)})

    def __getitem__(self, k):
        return self._state[k]

    def get(self, k, default=None):
        return self._state.get(k, default)


class _StubDict(dict):
    """Config nodes (yacs CfgNode, argparse.Namespace look-alikes) -> dict with attribute access."""

    def __getattr__(self, k):
        try:
            return self[k]
        except KeyError as e:
            raise AttributeError(k) from e

    def __setstate__(self, state):
        if isinstance(state, dict):
            self.update(state)


def _stub_class(module: str, name: str):
    if module.startswith("yacs") or name in ("CfgNode", "Namespace", "DictConfig"):
        return type(name, (_StubDict,), {"__module__": module})
    return type(name, (_Stub,), {"__module__": module})


class _TolerantUnpickler(pickle.Unpickler):
    def find_class(self, module, name):
        try:
            return super().find_class(module, name)
        except (ImportError, AttributeError):
            return _stub_class(module, name)


def _tolerant_pickle_module():
    """A `pickle_module` for torch.load whose Unpickler tolerates missing classes (tokenizer.pth's hparams)."""
    import types
    m = types.ModuleType("tokenhmr_b200._tolerant_pickle")
    m.Unpickler = _TolerantUnpickler
    m.load = lambda f, **kw: _TolerantUnpickler(f, **kw).load()
    m.loads = lambda b, **kw: _TolerantUnpickler(io.BytesIO(b), **kw).load()
    m.dump, m.dumps, m.Pickler, m.HIGHEST_PROTOCOL = pickle.dump, pickle.dumps, pickle.Pickler, pickle.HIGHEST_PROTOCOL
    m.__name__ = "pickle"
    return m


def _to_array(v) -> np.ndarray:
    """chumpy Ch / sparse matrix / array-like -> dense numpy array."""
    if isinstance(v, np.ndarray):
        return v
    if isinstance(v, _Stub):
        st = v._state
        if "x" in st:                                                   # chumpy.ch.Ch: the array lives in 'x'
            return np.asarray(st["x"])
        if {"data", "indices", "indptr"} <= set(st):                     # scipy.sparse csc / csr
            shape = tuple(st.get("_shape", st.get("shape")))
            dense = np.zeros(shape, dtype=np.asarray(st["data"]).dtype)
            data, ind, ptr = np.asarray(st["data"]), np.asarray(st["indices"]), np.asarray(st["indptr"])
            csc = "csc" in type(v).__name__.lower() or len(ptr) == shape[1] + 1 != shape[0] + 1
            for j in range(len(ptr) - 1):
                sl = slice(ptr[j], ptr[j + 1])
                if csc:
                    dense[ind[sl], j] = data[sl]
                else:
                    dense[j, ind[sl]] = data[sl]
            return dense
        if "data" in st and ("coords" in st or {"row", "col"} <= set(st)):   # coo (scipy >= 1.13 stores `coords`)
            row, col = st["coords"] if "coords" in st else (st["row"], st["col"])
            dense = np.zeros(tuple(st.get("_shape", st.get("shape"))), dtype=np.asarray(st["data"]).dtype)
            np.add.at(dense, (np.asarray(row), np.asarray(col)), np.asarray(st["data"]))
            return dense
        raise ValueError(f"cannot convert pickled {type(v).__module__}.{type(v).__name__} to an array")
    if hasattr(v, "toarray"):
        return np.asarray(v.toarray())
    if hasattr(v, "r"):                                                  # a live chumpy object
        return np.asarray(v.r)
    return np.asarray(v)


def _load_pickle(path) -> Any:
    with open(path, "rb") as f:
        return _TolerantUnpickler(f, encoding="latin1").load()


# ------------------------------------------------------------------------------------------- SMPL
def load_smpl_pkl(model_path, joint_regressor_extra: Optional[str] = None, num_betas: int = 10) -> Dict[str, torch.Tensor]:
    """SMPL_NEUTRAL.pkl (+ SMPL_to_J19.pkl) -> the buffers smplx.SMPLLayer registers, as tokenhmr_b200.ops.SMPLModel
    expects them: v_template (V,3), shapedirs (V,3,num_betas), posedirs (207,3V), J_regressor (24,V) dense,
    lbs_weights (V,24), parents (24,), faces (F,3), joint_regressor_extra (19,V), extra_vertex_ids (21,).
    `model_path` may be the .pkl or the directory holding SMPL_NEUTRAL.pkl (smplx's convention)."""
    p = Path(model_path)
    if p.is_dir():
        p = p / "SMPL_NEUTRAL.pkl"
    data = _load_pickle(p)
    get = lambda k: _to_array(data[k])
    v_template = get("v_template").astype(np.float32)
    V = v_template.shape[0]
    shapedirs = get("shapedirs").astype(np.float32)[:, :, :num_betas]
    posedirs = get("posedirs").astype(np.float32)                        # (V,3,207)
    posedirs = posedirs.reshape(-1, posedirs.shape[-1]).T                # smplx body_models: (207, 3V)
    kin = get("kintree_table").astype(np.int64)
    parents = kin[0].copy()
    parents[0] = -1
    out = {
        "v_template": torch.from_numpy(v_template),
        "shapedirs": torch.from_numpy(np.ascontiguousarray(shapedirs)),
        "posedirs": torch.from_numpy(np.ascontiguousarray(posedirs)),
        "J_regressor": torch.from_numpy(get("J_regressor").astype(np.float32)),
        "lbs_weights": torch.from_numpy(get("weights").astype(np.float32)),
        "parents": torch.from_numpy(parents),
        "faces": torch.from_numpy(get("f").astype(np.int64)),
        "extra_vertex_ids": torch.tensor(SMPL_EXTRA_VERTEX_IDS if V == 6890 else [(i * 7919) % V for i in range(21)],
                                         dtype=torch.int64),
    }
    if joint_regressor_extra is not None:
        out["joint_regressor_extra"] = torch.from_numpy(_to_array(_load_pickle(joint_regressor_extra)).astype(np.float32))
    assert out["J_regressor"].shape == (24, V) and out["lbs_weights"].shape == (V, 24), "not an SMPL (24-joint) model"
    return out


# ------------------------------------------------------------------------------------------- checkpoints
def _torch_load(path):
    try:
        return torch.load(path, map_location="cpu", weights_only=False, pickle_module=_tolerant_pickle_module())
    except TypeError:                                                     # older torch: no weights_only
        return torch.load(path, map_location="cpu", pickle_module=_tolerant_pickle_module())


def load_lightning_state_dict(path) -> Dict[str, torch.Tensor]:
    """ckpt['state_dict'] restricted to what the forward uses: `backbone.*` and `smpl_head.*` (misc.py:241-256)."""
    ckpt = _torch_load(path)
    sd = ckpt["state_dict"] if isinstance(ckpt, dict) and "state_dict" in ckpt else ckpt
    return {k: v for k, v in sd.items() if k.startswith(("backbone.", "smpl_head."))}


def load_tokenizer_checkpoint(path) -> Tuple[Dict[str, torch.Tensor], Dict[str, Any]]:
    """tokenizer.pth -> (net, arch): `net` without the body-model buffers (prepare_statedict's ignore_partname,
    vanilla_pose_vqvae.py:24-40,299-301), `arch` = hparams.ARCH as a plain dict (CODE_DIM, NB_CODE, WIDTH, ...)."""
    ckpt = _torch_load(path)
    net = {k: v for k, v in ckpt["net"].items() if "body_model" not in k}
    hp = ckpt.get("hparams")
    arch = getattr(hp, "ARCH", None) if hp is not None else None
    if arch is None and isinstance(hp, dict):
        arch = hp.get("ARCH")
    arch = dict(arch) if isinstance(arch, dict) else {k: v for k, v in vars(arch).items() if k.isupper()} if arch else {}
    return net, arch


def merge_state_dicts(model_sd: Dict[str, torch.Tensor], tokenizer_net: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
    """Flat naming of this repo: model keys as they are, tokenizer keys under `tokenizer.`."""
    out = dict(model_sd)
    for k, v in tokenizer_net.items():
        if k.startswith(("decoder.", "encoder.", "quantizer.")):
            out["tokenizer." + k] = v
    return out


def _unsupported(what: str, got, want, ref: str):
    from ._lib import ThmrError
    raise ThmrError(f"unsupported configuration: {what} = {got!r}; this engine implements {want} only ({ref})")


REGRESSION_HEAD = "transformer_decoder"


def validate_model_config(y: Dict[str, Any]) -> None:
    """Reject every reference variant the engine does not implement instead of silently running the release path.
    Defaults are the reference's own `.get()` defaults."""
    m = y.get("MODEL", {}) or {}
    head = m.get("SMPL_HEAD", {}) or {}
    # build_smpl_head (heads/__init__.py:4-13): default 'hmr' raises in the reference too; 'token' and
    # 'transformer_decoder' (HMR 2.0's regression head) are built here
    if "SMPL_HEAD" in m and head.get("TYPE", "hmr") not in ("token", REGRESSION_HEAD):
        _unsupported("MODEL.SMPL_HEAD.TYPE", head.get("TYPE", "hmr"), "'token' (SMPLTokenDecoderHead)", "heads/__init__.py:4-13")
    regression = "SMPL_HEAD" in m and head.get("TYPE") == REGRESSION_HEAD
    # the regression head reads the same three keys at the same places as the token head (smpl_head.py lines)
    if int(head.get("IEF_ITERS", 1)) != 1:
        _unsupported("MODEL.SMPL_HEAD.IEF_ITERS", head.get("IEF_ITERS"), "1 iteration",
                     "smpl_head.py:70" if regression else "token_head.py:86")
    if head.get("TRANSFORMER_INPUT", "zero") != "zero":
        _unsupported("MODEL.SMPL_HEAD.TRANSFORMER_INPUT", head.get("TRANSFORMER_INPUT"), "'zero' (constant query token)",
                     "smpl_head.py:21-24,72-75" if regression else "token_head.py:29,88-91")
    if head.get("JOINT_REP", "6d") != "6d":
        _unsupported("MODEL.SMPL_HEAD.JOINT_REP", head.get("JOINT_REP"), "'6d'",
                     "smpl_head.py:17-18,61-62" if regression else "token_head.py:23-24")
    tk = head.get("TOKENIZER", {}) or {}
    # MODEL.SMPL_HEAD.TOKENIZER configures the token classifier and the tokenizer (token_head.py:25-26,45-47), which the
    # regression head does not have (smpl_head.py:14-48) and HMR 2.0's configs do not carry: a yaml with both is a
    # TokenHMR yaml whose TYPE was changed, and its token settings would go unused, so it is refused, not guessed at
    if regression and "TOKENIZER" in head:
        _unsupported("MODEL.SMPL_HEAD.TOKENIZER with TYPE 'transformer_decoder'", sorted(tk),
                     "no TOKENIZER block for the regression head (it has no token classifier)",
                     "smpl_head.py:14-48, token_head.py:25-26,45-47")
    if not regression and tk.get("TOKENIZER_TYPE", "Vanilla") not in ("Vanilla",):
        _unsupported("MODEL.SMPL_HEAD.TOKENIZER.TOKENIZER_TYPE", tk.get("TOKENIZER_TYPE"), "'Vanilla'",
                     "token_classifier.py:12-20")
    dec = head.get("TRANSFORMER_DECODER", {}) or {}
    if dec.get("norm", "layer") != "layer":
        _unsupported("TRANSFORMER_DECODER.norm", dec.get("norm"), "'layer'", "pose_transformer.py:33-37")
    if int(dec.get("context_dim", 1280)) != 1280 or int(dec.get("dim", 1024)) != 1024:
        _unsupported("TRANSFORMER_DECODER.context_dim/dim", (dec.get("context_dim"), dec.get("dim")), "1280 / 1024",
                     "tokenhmr_release.yaml:73-81")
    if int(dec.get("dim_head", 64)) != 64 or int(dec.get("heads", 8)) > 8:
        _unsupported("TRANSFORMER_DECODER.dim_head/heads", (dec.get("dim_head"), dec.get("heads")), "<= 8 heads x 64",
                     "tokenhmr_release.yaml:73-81")
    bb = m.get("BACKBONE", {}) or {}
    if bb.get("TYPE", "vit") != "vit":
        _unsupported("MODEL.BACKBONE.TYPE", bb.get("TYPE"), "'vit' (ViT-H/16)", "backbones/__init__.py")
    smpl = y.get("SMPL", {}) or {}
    if smpl.get("update_hips", smpl.get("UPDATE_HIPS", False)):
        _unsupported("SMPL.update_hips", True, "False", "smpl_wrapper.py:33-36")
    if int(smpl.get("NUM_BODY_JOINTS", 23)) != 23:
        _unsupported("SMPL.NUM_BODY_JOINTS", smpl.get("NUM_BODY_JOINTS"), "23", "tokenhmr_release.yaml:31-37")
    if (smpl.get("GENDER", "neutral") or "neutral") not in ("neutral", "male", "female"):
        _unsupported("SMPL.GENDER", smpl.get("GENDER"), "an SMPL .pkl gender", "smpl_wrapper.py:10")


def infer_head(sd: Dict[str, torch.Tensor]) -> str:
    """The SMPL head a checkpoint holds, from its keys: `smpl_head.decpose.weight` (npose, dec_dim) is the regression
    head's pose read-out (smpl_head.py:32), `smpl_head.decpose.mixer_trans.*` the token head's classifier
    (token_head.py:45, token_classifier.py:67-69)."""
    from ._lib import ThmrError
    regression = "smpl_head.decpose.weight" in sd and sd["smpl_head.decpose.weight"].dim() == 2
    token = any(k.startswith("smpl_head.decpose.mixer_trans.") for k in sd)
    if regression == token:
        raise ThmrError("cannot tell the SMPL head from the checkpoint keys: expected either smpl_head.decpose.weight "
                        "(MODEL.SMPL_HEAD.TYPE 'transformer_decoder') or smpl_head.decpose.mixer_trans.* ('token')"
                        + (", found both" if token else ", found neither"))
    return REGRESSION_HEAD if regression else "token"


def validate_against_weights(cfg: TokenHMRConfig, sd: Dict[str, torch.Tensor], smpl: Dict[str, torch.Tensor]) -> None:
    """Shapes the files imply must agree with the configuration the engine is built for."""
    from ._lib import ThmrError
    if cfg.head == REGRESSION_HEAD:
        if any(k.startswith("smpl_head.decpose.mixer_trans.") for k in sd):
            raise ThmrError("the configuration says MODEL.SMPL_HEAD.TYPE 'transformer_decoder' but the checkpoint holds "
                            "a token head (smpl_head.decpose.mixer_trans.*)")
        # decpose / decshape / deccam read the decoder's output token (smpl_head.py:32-34)
        for name, rows in (("decpose", cfg.npose), ("decshape", cfg.num_betas), ("deccam", 3)):
            w, b = sd.get(f"smpl_head.{name}.weight"), sd.get(f"smpl_head.{name}.bias")
            if w is None or b is None:
                raise ThmrError(f"regression head: smpl_head.{name}.weight / .bias missing from the checkpoint")
            if tuple(w.shape) != (rows, cfg.dec_dim) or tuple(b.shape) != (rows,):
                raise ThmrError(f"regression head: smpl_head.{name} is {tuple(w.shape)} but the engine reads "
                                f"({rows}, {cfg.dec_dim}) (npose / betas / camera x dec_dim)")
    elif "smpl_head.decpose.weight" in sd:
        raise ThmrError("the configuration says MODEL.SMPL_HEAD.TYPE 'token' but the checkpoint holds a regression head "
                        "(smpl_head.decpose.weight): build it with TokenHMRConfig(head='transformer_decoder')")
    cb = sd.get("tokenizer.quantizer.codebook")
    if cb is not None and tuple(cb.shape) != (cfg.token_class_num, cfg.code_dim):
        raise ThmrError(f"tokenizer codebook is {tuple(cb.shape)} but the classifier predicts {cfg.token_class_num} classes "
                        f"of dimension {cfg.code_dim} (TOKEN_CLASS_NUM / TOKEN_CODE_DIM vs tokenizer NB_CODE / CODE_DIM)")
    if cfg.nb_code != cfg.token_class_num:
        raise ThmrError(f"tokenizer NB_CODE {cfg.nb_code} != MODEL.SMPL_HEAD.TOKENIZER.TOKEN_CLASS_NUM {cfg.token_class_num}")
    te = sd.get("smpl_head.transformer.to_token_embedding.weight")
    if te is not None and te.shape[1] != 1:
        raise ThmrError(f"to_token_embedding takes {te.shape[1]} inputs: a TRANSFORMER_INPUT='mean_shape' checkpoint "
                        "(token_head.py:29-33) is not supported")
    if "joint_regressor_extra" not in smpl:
        import warnings
        warnings.warn("no joint_regressor_extra (SMPL_to_J19.pkl): pred_keypoints_3d/2d will have 25 instead of 44 joints "
                      "(smpl_wrapper.py:22-23,37-39)")


def config_from_files(model_cfg_yaml: Optional[str], arch: Optional[Dict[str, Any]] = None,
                      head: Optional[str] = None) -> TokenHMRConfig:
    """model_config.yaml (MODEL.* of the yacs dump, models/__init__.py:6-17) + tokenizer hparams -> TokenHMRConfig.
    `head`: the SMPL head when the yaml does not name one (MODEL.SMPL_HEAD.TYPE wins)."""
    kw: Dict[str, Any] = {"head": head} if head else {}
    if model_cfg_yaml:
        import yaml
        with open(model_cfg_yaml) as f:
            y = yaml.safe_load(f) or {}
        validate_model_config(y)
        m = y.get("MODEL", {})
        if "IMAGE_SIZE" in m:
            kw["image_size"] = int(m["IMAGE_SIZE"])
        if m.get("BBOX_SHAPE"):
            kw["crop_w"] = int(m["BBOX_SHAPE"][0])
        head = m.get("SMPL_HEAD", {})
        if head.get("TYPE"):
            kw["head"] = str(head["TYPE"])
        t = head.get("TOKENIZER", {})
        for src, dst in (("TOKEN_CODE_DIM", "code_dim"), ("TOKEN_NUM", "token_num"), ("TOKEN_CLASS_NUM", "token_class_num")):
            if src in t:
                kw[dst] = int(t[src])
        d = head.get("TRANSFORMER_DECODER", {})
        for src, dst in (("depth", "dec_depth"), ("heads", "dec_heads"), ("mlp_dim", "dec_mlp_dim"), ("dim_head", "dec_dim_head")):
            if src in d:
                kw[dst] = int(d[src])
        if "EXTRA" in y and "FOCAL_LENGTH" in y["EXTRA"]:
            kw["focal_length"] = float(y["EXTRA"]["FOCAL_LENGTH"])
    for src, dst in (("CODE_DIM", "code_dim"), ("NB_CODE", "nb_code"), ("WIDTH", "tok_width"), ("DEPTH", "tok_depth"),
                     ("DILATION_RATE", "tok_dilation_rate"), ("TOKEN_SIZE_DIV", "tok_size_div"),
                     ("TOKEN_SIZE_MUL", "tok_size_mul")):
        if arch and src in arch:
            kw[dst] = int(arch[src])
    return TokenHMRConfig(**kw)


def load_tokenhmr(checkpoint_path: str, model_cfg: Optional[str] = None, tokenizer_path: Optional[str] = None,
                  smpl_model_path: Optional[str] = None, joint_regressor_extra: Optional[str] = None,
                  device: str = "cuda:0", **engine_kw):
    """File-based counterpart of lib.models.load_tokenhmr (tokenhmr/lib/models/__init__.py:3-26): returns (model, cfg).
    Paths default to the reference's layout relative to the checkpoint (data/checkpoints/tokenizer.pth,
    data/body_models/smpl, data/body_models/SMPL_to_J19.pkl).
    The SMPL head is the yaml's MODEL.SMPL_HEAD.TYPE, or without a yaml the one the checkpoint's keys hold
    (infer_head); an HMR 2.0 checkpoint ('transformer_decoder') has no tokenizer and tokenizer.pth is never opened."""
    from ._lib import ThmrError
    from .engine import TokenHMREngine
    ck = Path(checkpoint_path)
    root = ck.parent.parent if ck.parent.name == "checkpoints" else ck.parent
    smpl_model_path = smpl_model_path or str(root / "body_models" / "smpl")
    if joint_regressor_extra is None and (root / "body_models" / "SMPL_to_J19.pkl").exists():
        joint_regressor_extra = str(root / "body_models" / "SMPL_to_J19.pkl")
    model_sd = load_lightning_state_dict(checkpoint_path)
    head = infer_head(model_sd)
    yaml_head = config_from_files(model_cfg, head=head).head if model_cfg else head
    if yaml_head != head:
        raise ThmrError(f"{model_cfg} says MODEL.SMPL_HEAD.TYPE {yaml_head!r} but the checkpoint {checkpoint_path} holds "
                        f"a {head!r} head")
    net, arch = {}, None
    if head == "token":
        net, arch = load_tokenizer_checkpoint(tokenizer_path or str(ck.parent / "tokenizer.pth"))
    cfg = config_from_files(model_cfg, arch, head=head)
    sd = merge_state_dicts(model_sd, net)
    smpl = load_smpl_pkl(smpl_model_path, joint_regressor_extra, num_betas=cfg.num_betas)
    # what the files themselves imply: number of ViT blocks, mesh size
    import dataclasses
    import re
    blocks = {int(m.group(1)) for k in sd for m in [re.match(r"backbone\.blocks\.(\d+)\.", k)] if m}
    cfg = dataclasses.replace(cfg, vit_depth=max(blocks) + 1 if blocks else cfg.vit_depth,
                              num_verts=int(smpl["v_template"].shape[0]))
    validate_against_weights(cfg, sd, smpl)
    return TokenHMREngine(cfg, sd, smpl, device=device, **engine_kw), cfg

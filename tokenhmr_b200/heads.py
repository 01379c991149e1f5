"""The SMPL heads as trainable modules on the GPU: HMR 2.0's regression head and TokenHMR's token head.

    model = TokenHMREngine(cfg, sd, smpl)                   # frozen backbone, inference kernels
    head = TokenHead(cfg, sd, device)                       # or RegressionHead for a transformer_decoder checkpoint
    opt = torch.optim.AdamW(head.parameters(), lr=..., weight_decay=1e-4)
    params, cam, lst = head(model.backbone(img))            # the reference head's forward outputs
    ...
    sd.update({"smpl_head." + k: v for k, v in head.state_dict().items()})   # serve the fine-tuned weights

Each head holds the reference head's parameters (SMPLTransformerDecoderHead, heads/smpl_head.py:14-48, or
SMPLTokenDecoderHead, heads/token_head.py:20-63) as fp32 views of one flat buffer, under the reference's state_dict names,
plus the three init_* buffers.  Its forward and backward are two CUDA calls (thmr_reg_head_* / thmr_tok_head_*): the
backward writes the gradient of every parameter and takes none for the features.  The C library owns the parameter
layouts (thmr_reg_head_param_info, thmr_tok_head_param_info); this module only builds tensors from them.

The token head's tokenizer (its decoder and codebook) is frozen, as in the reference, which reaches it through a Proxy:
it lives in a second flat buffer, a non-persistent buffer of the module, so it is in neither state_dict() nor
parameters().
"""
from __future__ import annotations

import ctypes
from typing import Dict, List, Optional, Tuple

import torch
from torch import nn

from . import _lib
from ._lib import check, lib
from .config import TokenHMRConfig, release_config

_NUM_BETAS, _NPOSE = 10, 144
_TOKENS, _CLASSES = 160, 2048

Layout = List[Tuple[str, Tuple[int, ...], int]]


def _read_layout(count_fn, info_fn, dims: tuple) -> Tuple[Layout, int]:
    n, total = ctypes.c_int(0), ctypes.c_int64(0)
    check(count_fn(*dims, ctypes.byref(n), ctypes.byref(total)))
    out = []
    name, nd = ctypes.c_char_p(), ctypes.c_int(0)
    shape, off = (ctypes.c_int64 * 3)(), ctypes.c_int64(0)
    for i in range(n.value):
        check(info_fn(*dims, i, ctypes.byref(name), ctypes.byref(nd), shape, ctypes.byref(off)))
        out.append((name.value.decode(), tuple(int(shape[k]) for k in range(nd.value)), int(off.value)))
    return out, int(total.value)


def param_layout(depth: int, heads: int, mlp_dim: int) -> Tuple[Layout, int]:
    """[(state_dict name, shape, offset in floats)] of the regression head's parameters and the floats of the flat
    buffer, from the C library."""
    L = lib()
    return _read_layout(L.thmr_reg_head_num_params, L.thmr_reg_head_param_info, (depth, heads, mlp_dim))


def token_param_layout(depth: int, heads: int, mlp_dim: int) -> Tuple[Layout, int]:
    """The same for the token head's trainable parameters."""
    L = lib()
    return _read_layout(L.thmr_tok_head_num_params, L.thmr_tok_head_param_info, (depth, heads, mlp_dim))


def tokenizer_layout() -> Tuple[Layout, int]:
    """[(checkpoint name, shape, offset in floats)] of the token head's frozen tokenizer tensors, and their floats."""
    L = lib()
    return _read_layout(L.thmr_tok_head_tokenizer_num, L.thmr_tok_head_tokenizer_info, ())


def _model_cfg_dict(model_cfg) -> Optional[dict]:
    if model_cfg is None or isinstance(model_cfg, dict):
        return model_cfg
    import yaml
    with open(model_cfg) as f:
        return yaml.safe_load(f) or {}


def _flat_from(layout: Layout, total: int, src: Dict[str, torch.Tensor], device, who: str, prefix: str):
    """One flat fp32 buffer holding src's tensors at the layout's offsets."""
    flat = torch.zeros(total, dtype=torch.float32, device=device)
    for name, shape, off in layout:
        if name not in src:
            raise _lib.ThmrError(f"{who}: the state dict has no {prefix}{name}")
        t = src[name]
        if tuple(t.shape) != shape:
            raise _lib.ThmrError(f"{who}: {prefix}{name} has shape {tuple(t.shape)}, expected {shape}")
        flat[off:off + t.numel()].view(shape).copy_(t.detach().to(device=device, dtype=torch.float32))
    return flat


class _FlatHead(nn.Module):
    """What both trainable heads share: the checks on the configuration and on the features, the flat parameter buffer
    with one nn.Parameter view per reference parameter, the init_* buffers and the descriptor's common fields."""

    def __init__(self, cfg: TokenHMRConfig, state_dict: Dict[str, torch.Tensor], device, model_cfg, layout_fn):
        super().__init__()
        who = type(self).__name__
        y = _model_cfg_dict(model_cfg)
        if y is not None:
            dec = y.get("MODEL", {}).get("SMPL_HEAD", {}).get("TRANSFORMER_DECODER", {})
            for k in ("dropout", "emb_dropout"):
                if float(dec.get(k, 0.0)) != 0.0:
                    raise _lib.ThmrError(f"{who}: MODEL.SMPL_HEAD.TRANSFORMER_DECODER.{k} = {dec[k]}; "
                                         "training with dropout is not supported (it must be 0)")
        if (cfg.dec_dim, cfg.dec_dim_head, cfg.vit_dim, cfg.num_tokens, cfg.num_joints, cfg.num_betas) != \
                (1024, 64, 1280, 192, 24, 10):
            raise _lib.ThmrError(f"{who}: needs dim 1024, dim_head 64, 1280 x 192 features, 24 joints and 10 betas")
        device = torch.device(device)
        if device.type != "cuda":
            raise _lib.ThmrError(f"{who}: needs a CUDA device (tokenhmr_b200 has no CPU fallback)")
        self.cfg = cfg
        self.dims = (cfg.dec_depth, cfg.dec_heads, cfg.dec_mlp_dim)
        layout, total = layout_fn(*self.dims)
        self._layout = layout
        src = {k[len("smpl_head."):]: v for k, v in state_dict.items() if k.startswith("smpl_head.")}
        self._flat = _flat_from(layout, total, src, device, who, "smpl_head.")
        for name, shape, off in layout:
            mod, leaf = self._submodule(name)
            mod.register_parameter(leaf, nn.Parameter(self._flat[off:off + _numel(shape)].view(shape)))
        self._param_list = [(name, self.get_parameter(name), off) for name, _, off in layout]   # layout order
        for name, n in (("init_body_pose", _NPOSE), ("init_betas", _NUM_BETAS), ("init_cam", 3)):
            t = src.get(name)
            if t is None or t.numel() != n:
                raise _lib.ThmrError(f"{who}: smpl_head.{name} missing or not {n} values")
            self.register_buffer(name, t.detach().to(device=device, dtype=torch.float32).reshape(1, n).clone())

    def _submodule(self, name: str) -> Tuple[nn.Module, str]:
        *path, leaf = name.split(".")
        mod: nn.Module = self
        for p in path:
            if p not in mod._modules:
                mod.add_module(p, nn.Module())
            mod = mod._modules[p]
        return mod, leaf

    def _params(self) -> List[torch.Tensor]:
        """The parameters in layout order, checked to still be views of the flat buffer the kernels read."""
        out = []
        base = self._flat.data_ptr()
        for name, p, off in self._param_list:
            if self.get_parameter(name) is not p or p.data_ptr() != base + 4 * off or p.dtype != torch.float32:
                raise _lib.ThmrError(f"{type(self).__name__}: parameter {name} no longer lives in the head's flat fp32 "
                                     "buffer (was it replaced or moved?); update it in place, e.g. with copy_")
            out.append(p)
        return out

    def _check_feats(self, feats) -> None:
        who = type(self).__name__
        if not isinstance(feats, torch.Tensor) or feats.dim() != 4 or tuple(feats.shape[1:]) != (
                self.cfg.vit_dim, self.cfg.grid_h, self.cfg.grid_w) or feats.shape[0] < 1:
            raise _lib.ThmrError(f"{who}: features must be (B, {self.cfg.vit_dim}, {self.cfg.grid_h}, "
                                 f"{self.cfg.grid_w}), got {tuple(getattr(feats, 'shape', ()))}")
        if feats.dtype != torch.float32:
            raise _lib.ThmrError(f"{who}: features must be float32, got {feats.dtype}")
        if feats.device != self._flat.device:
            raise _lib.ThmrError(f"{who}: features on {feats.device}, the head on {self._flat.device}")
        if not feats.is_contiguous():
            raise _lib.ThmrError(f"{who}: features must be contiguous")
        if feats.requires_grad:
            raise _lib.ThmrError(f"{who}: features require grad, but the gradient with respect to the "
                                 "features is not built (detach them, as with a frozen backbone)")

    def _fill_desc(self, d, B: int, feats: torch.Tensor, ws: torch.Tensor):
        d.B, (d.depth, d.heads, d.mlp_dim) = B, self.dims
        d.params = self._flat.data_ptr()
        d.init_body_pose, d.init_betas = self.init_body_pose.data_ptr(), self.init_betas.data_ptr()
        d.init_cam = self.init_cam.data_ptr()
        d.feats = feats.data_ptr()
        d.workspace, d.workspace_bytes = ws.data_ptr(), ws.numel()
        d.stream = torch.cuda.current_stream(feats.device).cuda_stream
        return d

    def _grads_out(self, grads: torch.Tensor):
        return [grads[off:off + _numel(shape)].view(shape) for _, shape, off in self._layout]


def _set_upstream(d, held: list, grads) -> None:
    """Points d's optional upstream-gradient fields at contiguous fp32 copies kept alive in held."""
    for name, g, shape in grads:
        if g is not None:
            g = g.to(torch.float32).contiguous()
            assert tuple(g.shape) == shape, (name, tuple(g.shape))
            held.append(g)
            setattr(d, name, g.data_ptr())


class RegressionHead(_FlatHead):
    """SMPLTransformerDecoderHead (MODEL.SMPL_HEAD.TYPE transformer_decoder) with fp32 CUDA forward and backward.

    cfg: the engine's TokenHMRConfig (cfg.head must be "transformer_decoder"); state_dict: a checkpoint state dict
    whose smpl_head.* entries are read; model_cfg (optional): the model_config.yaml path or its dict, whose
    TRANSFORMER_DECODER.dropout / emb_dropout must be 0 (training with dropout would differ from the reference)."""

    def __init__(self, cfg: TokenHMRConfig, state_dict: Dict[str, torch.Tensor], device="cuda", model_cfg=None):
        if cfg.head != "transformer_decoder":
            raise _lib.ThmrError(f"RegressionHead: cfg.head is {cfg.head!r}; only the 'transformer_decoder' "
                                 "(HMR 2.0 regression) head is trained by this class, the token head's is not built "
                                 "by it; use TokenHead")
        super().__init__(cfg, state_dict, device, model_cfg, param_layout)

    def forward(self, feats: torch.Tensor):
        """feats (B, 1280, 16, 12) fp32, contiguous, on the head's device, not requiring grad ->
        (pred_smpl_params, pred_cam, pred_smpl_params_list) as SMPLTransformerDecoderHead.forward returns them."""
        self._check_feats(feats)
        params = self._params()
        keep = torch.is_grad_enabled() and any(p.requires_grad for p in params)
        pose6d, betas, cam, rot = _RegHeadFn.apply(self, keep, feats, *params)
        pred = {"global_orient": rot[:, :1], "body_pose": rot[:, 1:], "betas": betas}
        lst = {"body_pose": rot[:, 1:], "betas": betas, "cam": cam}
        return pred, cam, lst

    def _desc(self, B: int, feats: torch.Tensor, ws: torch.Tensor) -> _lib.RegHeadDesc:
        return self._fill_desc(_lib.RegHeadDesc(), B, feats, ws)

    def workspace_bytes(self, B: int) -> int:
        return int(lib().thmr_reg_head_workspace_bytes(B, *self.dims))


class _RegHeadFn(torch.autograd.Function):
    """(pose6d, betas, cam, rotmats) of the head; differentiable to every parameter, not to the features.  The forward
    keeps its activations in a workspace that lives until the backward (nothing is kept under no_grad)."""

    @staticmethod
    def forward(ctx, head: RegressionHead, keep: bool, feats: torch.Tensor, *params):
        B, dev = feats.shape[0], feats.device
        ws = torch.empty(head.workspace_bytes(B), dtype=torch.uint8, device=dev)
        pose6d = torch.empty(B, _NPOSE, device=dev)
        betas = torch.empty(B, _NUM_BETAS, device=dev)
        cam = torch.empty(B, 3, device=dev)
        rot = torch.empty(B, 24, 3, 3, device=dev)
        d = head._desc(B, feats, ws)
        d.pose6d, d.betas, d.cam, d.rotmats = pose6d.data_ptr(), betas.data_ptr(), cam.data_ptr(), rot.data_ptr()
        check(lib().thmr_reg_head_train_forward(ctypes.byref(d)))
        if keep:                       # grad mode was on where the head was called (forward itself runs without)
            ctx.head, ctx.ws, ctx.B = head, ws, B
            ctx.save_for_backward(feats)
        ctx.set_materialize_grads(False)
        return pose6d, betas, cam, rot

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, g_pose6d, g_betas, g_cam, g_rot):
        head, ws, B = ctx.head, ctx.ws, ctx.B
        (feats,) = ctx.saved_tensors
        grads = torch.empty_like(head._flat)
        d = head._desc(B, feats, ws)
        d.grads = grads.data_ptr()
        held = []                      # the contiguous upstream gradients, alive until the call returns
        _set_upstream(d, held, (("grad_pose6d", g_pose6d, (B, _NPOSE)), ("grad_betas", g_betas, (B, _NUM_BETAS)),
                                ("grad_cam", g_cam, (B, 3)), ("grad_rotmats", g_rot, (B, 24, 3, 3))))
        check(lib().thmr_reg_head_backward(ctypes.byref(d)))
        return (None, None, None, *head._grads_out(grads))


_RELEASE_TOKEN_DIMS = ("token_num", "token_class_num", "cls_hidden", "cls_hidden_inter", "cls_token_inter",
                       "cls_blocks", "code_dim", "nb_code", "tok_width", "tok_depth", "tok_dilation_rate",
                       "tok_joints", "tok_size_div")


class TokenHead(_FlatHead):
    """SMPLTokenDecoderHead (MODEL.SMPL_HEAD.TYPE token) with fp32 CUDA forward and backward: the decoder, the read-outs
    and the MLP-Mixer token classifier are trained; the tokenizer decoder and codebook are frozen and back-propagated
    through.

    cfg: the engine's TokenHMRConfig (cfg.head must be "token", with the release classifier and tokenizer dimensions);
    state_dict: a checkpoint state dict whose smpl_head.* and tokenizer.* entries are read (checkpoint.load_tokenhmr's
    or synth.make_state_dict's); model_cfg (optional): as for RegressionHead."""

    def __init__(self, cfg: TokenHMRConfig, state_dict: Dict[str, torch.Tensor], device="cuda", model_cfg=None):
        if cfg.head != "token":
            raise _lib.ThmrError(f"TokenHead: cfg.head is {cfg.head!r}; this class trains the 'token' head (use "
                                 "RegressionHead for 'transformer_decoder')")
        rel = release_config()
        for k in _RELEASE_TOKEN_DIMS:
            if getattr(cfg, k) != getattr(rel, k):
                raise _lib.ThmrError(f"TokenHead: {k} = {getattr(cfg, k)}; the CUDA token head is built for the "
                                     f"release classifier and tokenizer ({k} = {getattr(rel, k)})")
        super().__init__(cfg, state_dict, device, model_cfg, token_param_layout)
        layout, total = tokenizer_layout()
        src = {k: v for k, v in state_dict.items() if k.startswith("tokenizer.")}
        self.register_buffer("_tokenizer", _flat_from(layout, total, src, self._flat.device, "TokenHead", ""),
                             persistent=False)

    def forward(self, feats: torch.Tensor):
        """feats (B, 1280, 16, 12) fp32, contiguous, on the head's device, not requiring grad ->
        (pred_smpl_params, pred_cam, pred_smpl_params_list) as SMPLTokenDecoderHead.forward returns them;
        pred_smpl_params_list holds body_pose, betas, cam and cls_logits_softmax (B, 160, 2048)."""
        self._check_feats(feats)
        params = self._params()
        keep = torch.is_grad_enabled() and any(p.requires_grad for p in params)
        pose6d, betas, cam, rot, probs = _TokHeadFn.apply(self, keep, feats, *params)
        pred = {"global_orient": rot[:, :1], "body_pose": rot[:, 1:], "betas": betas}
        lst = {"body_pose": rot[:, 1:], "betas": betas, "cam": cam, "cls_logits_softmax": probs}
        return pred, cam, lst

    def _desc(self, B: int, feats: torch.Tensor, ws: torch.Tensor) -> _lib.TokHeadDesc:
        d = self._fill_desc(_lib.TokHeadDesc(), B, feats, ws)
        d.tokenizer = self._tokenizer.data_ptr()
        return d

    def workspace_bytes(self, B: int) -> int:
        return int(lib().thmr_tok_head_workspace_bytes(B, *self.dims))


class _TokHeadFn(torch.autograd.Function):
    """(pose6d, betas, cam, rotmats, cls_logits_softmax) of the token head; differentiable to every trainable
    parameter, not to the features or the tokenizer.  The forward keeps its activations in a workspace that lives until
    the backward (nothing is kept under no_grad)."""

    @staticmethod
    def forward(ctx, head: TokenHead, keep: bool, feats: torch.Tensor, *params):
        B, dev = feats.shape[0], feats.device
        ws = torch.empty(head.workspace_bytes(B), dtype=torch.uint8, device=dev)
        pose6d = torch.empty(B, _NPOSE, device=dev)
        betas = torch.empty(B, _NUM_BETAS, device=dev)
        cam = torch.empty(B, 3, device=dev)
        rot = torch.empty(B, 24, 3, 3, device=dev)
        probs = torch.empty(B, _TOKENS, _CLASSES, device=dev)
        d = head._desc(B, feats, ws)
        d.pose6d, d.betas, d.cam, d.rotmats = pose6d.data_ptr(), betas.data_ptr(), cam.data_ptr(), rot.data_ptr()
        d.cls_probs = probs.data_ptr()
        check(lib().thmr_tok_head_train_forward(ctypes.byref(d)))
        if keep:                       # the backward reads P from probs: saving it makes autograd refuse in-place edits
            ctx.head, ctx.ws, ctx.B = head, ws, B
            ctx.save_for_backward(feats, probs)
        ctx.set_materialize_grads(False)
        return pose6d, betas, cam, rot, probs

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, g_pose6d, g_betas, g_cam, g_rot, g_probs):
        head, ws, B = ctx.head, ctx.ws, ctx.B
        feats, probs = ctx.saved_tensors
        grads = torch.empty_like(head._flat)
        d = head._desc(B, feats, ws)
        d.grads, d.cls_probs = grads.data_ptr(), probs.data_ptr()
        held = []
        _set_upstream(d, held, (("grad_pose6d", g_pose6d, (B, _NPOSE)), ("grad_betas", g_betas, (B, _NUM_BETAS)),
                                ("grad_cam", g_cam, (B, 3)), ("grad_rotmats", g_rot, (B, 24, 3, 3)),
                                ("grad_cls_probs", g_probs, (B, _TOKENS, _CLASSES))))
        check(lib().thmr_tok_head_backward(ctypes.byref(d)))
        return (None, None, None, *head._grads_out(grads))


def _numel(shape) -> int:
    n = 1
    for s in shape:
        n *= s
    return n

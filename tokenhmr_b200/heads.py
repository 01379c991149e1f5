"""HMR 2.0's regression head as a trainable module on the GPU.

    model = TokenHMREngine(cfg, sd, smpl)                   # frozen backbone, inference kernels
    head = RegressionHead(cfg, sd, device)                  # trainable fp32 head, CUDA forward and backward
    opt = torch.optim.AdamW(head.parameters(), lr=..., weight_decay=1e-4)
    params, cam, _ = head(model.backbone(img))              # SMPLTransformerDecoderHead.forward's outputs
    ...
    sd.update({"smpl_head." + k: v for k, v in head.state_dict().items()})   # serve the fine-tuned weights

`RegressionHead` holds the reference head's parameters (SMPLTransformerDecoderHead, heads/smpl_head.py:14-48) as fp32
views of one flat buffer, under the reference's state_dict names, plus the three init_* buffers.  Its forward and
backward are two CUDA calls (thmr_reg_head_train_forward / thmr_reg_head_backward): the backward writes the gradient
of every parameter and takes none for the features.  The C library owns the parameter layout
(thmr_reg_head_param_info); this module only builds tensors from it.
"""
from __future__ import annotations

import ctypes
from typing import Dict, List, Optional, Tuple

import torch
from torch import nn

from . import _lib
from ._lib import check, lib
from .config import TokenHMRConfig

_NUM_BETAS, _NPOSE = 10, 144


def param_layout(depth: int, heads: int, mlp_dim: int) -> Tuple[List[Tuple[str, Tuple[int, ...], int]], int]:
    """[(state_dict name, shape, offset in floats)] of the head's parameters and the floats of the flat buffer, from
    the C library."""
    L = lib()
    n, total = ctypes.c_int(0), ctypes.c_int64(0)
    check(L.thmr_reg_head_num_params(depth, heads, mlp_dim, ctypes.byref(n), ctypes.byref(total)))
    out = []
    name, nd = ctypes.c_char_p(), ctypes.c_int(0)
    shape, off = (ctypes.c_int64 * 3)(), ctypes.c_int64(0)
    for i in range(n.value):
        check(L.thmr_reg_head_param_info(depth, heads, mlp_dim, i, ctypes.byref(name), ctypes.byref(nd), shape,
                                         ctypes.byref(off)))
        out.append((name.value.decode(), tuple(int(shape[k]) for k in range(nd.value)), int(off.value)))
    return out, int(total.value)


def _model_cfg_dict(model_cfg) -> Optional[dict]:
    if model_cfg is None or isinstance(model_cfg, dict):
        return model_cfg
    import yaml
    with open(model_cfg) as f:
        return yaml.safe_load(f) or {}


class RegressionHead(nn.Module):
    """SMPLTransformerDecoderHead (MODEL.SMPL_HEAD.TYPE transformer_decoder) with fp32 CUDA forward and backward.

    cfg: the engine's TokenHMRConfig (cfg.head must be "transformer_decoder"); state_dict: a checkpoint state dict
    whose smpl_head.* entries are read; model_cfg (optional): the model_config.yaml path or its dict, whose
    TRANSFORMER_DECODER.dropout / emb_dropout must be 0 (training with dropout would differ from the reference)."""

    def __init__(self, cfg: TokenHMRConfig, state_dict: Dict[str, torch.Tensor], device="cuda", model_cfg=None):
        super().__init__()
        if cfg.head != "transformer_decoder":
            raise _lib.ThmrError(f"RegressionHead: cfg.head is {cfg.head!r}; only the 'transformer_decoder' "
                                 "(HMR 2.0 regression) head has a CUDA backward, the token head's is not built")
        y = _model_cfg_dict(model_cfg)
        if y is not None:
            dec = y.get("MODEL", {}).get("SMPL_HEAD", {}).get("TRANSFORMER_DECODER", {})
            for k in ("dropout", "emb_dropout"):
                if float(dec.get(k, 0.0)) != 0.0:
                    raise _lib.ThmrError(f"RegressionHead: MODEL.SMPL_HEAD.TRANSFORMER_DECODER.{k} = {dec[k]}; "
                                         "training with dropout is not supported (it must be 0)")
        if (cfg.dec_dim, cfg.dec_dim_head, cfg.vit_dim, cfg.num_tokens, cfg.num_joints, cfg.num_betas) != \
                (1024, 64, 1280, 192, 24, 10):
            raise _lib.ThmrError("RegressionHead: needs dim 1024, dim_head 64, 1280 x 192 features, 24 joints and "
                                 "10 betas")
        device = torch.device(device)
        if device.type != "cuda":
            raise _lib.ThmrError("RegressionHead: needs a CUDA device (tokenhmr_b200 has no CPU fallback)")
        self.cfg = cfg
        self.dims = (cfg.dec_depth, cfg.dec_heads, cfg.dec_mlp_dim)
        layout, total = param_layout(*self.dims)
        self._flat = torch.zeros(total, dtype=torch.float32, device=device)
        self._layout = layout
        src = {k[len("smpl_head."):]: v for k, v in state_dict.items() if k.startswith("smpl_head.")}
        for name, shape, off in layout:
            if name not in src:
                raise _lib.ThmrError(f"RegressionHead: the state dict has no smpl_head.{name}")
            t = src[name]
            if tuple(t.shape) != shape:
                raise _lib.ThmrError(f"RegressionHead: smpl_head.{name} has shape {tuple(t.shape)}, expected {shape}")
            n = t.numel()
            view = self._flat[off:off + n].view(shape)
            view.copy_(t.detach().to(device=device, dtype=torch.float32))
            mod, leaf = self._submodule(name)
            mod.register_parameter(leaf, nn.Parameter(view))
        self._param_list = [(name, self.get_parameter(name), off) for name, _, off in layout]   # layout order
        for name, n in (("init_body_pose", _NPOSE), ("init_betas", _NUM_BETAS), ("init_cam", 3)):
            t = src.get(name)
            if t is None or t.numel() != n:
                raise _lib.ThmrError(f"RegressionHead: smpl_head.{name} missing or not {n} values")
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
                raise _lib.ThmrError(f"RegressionHead: parameter {name} no longer lives in the head's flat fp32 "
                                     "buffer (was it replaced or moved?); update it in place, e.g. with copy_")
            out.append(p)
        return out

    def forward(self, feats: torch.Tensor):
        """feats (B, 1280, 16, 12) fp32, contiguous, on the head's device, not requiring grad ->
        (pred_smpl_params, pred_cam, pred_smpl_params_list) as SMPLTransformerDecoderHead.forward returns them."""
        if not isinstance(feats, torch.Tensor) or feats.dim() != 4 or tuple(feats.shape[1:]) != (
                self.cfg.vit_dim, self.cfg.grid_h, self.cfg.grid_w) or feats.shape[0] < 1:
            raise _lib.ThmrError(f"RegressionHead: features must be (B, {self.cfg.vit_dim}, {self.cfg.grid_h}, "
                                 f"{self.cfg.grid_w}), got {tuple(getattr(feats, 'shape', ()))}")
        if feats.dtype != torch.float32:
            raise _lib.ThmrError(f"RegressionHead: features must be float32, got {feats.dtype}")
        if feats.device != self._flat.device:
            raise _lib.ThmrError(f"RegressionHead: features on {feats.device}, the head on {self._flat.device}")
        if not feats.is_contiguous():
            raise _lib.ThmrError("RegressionHead: features must be contiguous")
        if feats.requires_grad:
            raise _lib.ThmrError("RegressionHead: features require grad, but the gradient with respect to the "
                                 "features is not built (detach them, as with a frozen backbone)")
        params = self._params()
        keep = torch.is_grad_enabled() and any(p.requires_grad for p in params)
        pose6d, betas, cam, rot = _RegHeadFn.apply(self, keep, feats, *params)
        B = feats.shape[0]
        pred = {"global_orient": rot[:, :1], "body_pose": rot[:, 1:], "betas": betas}
        lst = {"body_pose": rot[:, 1:], "betas": betas, "cam": cam}
        return pred, cam, lst

    def _desc(self, B: int, feats: torch.Tensor, ws: torch.Tensor) -> _lib.RegHeadDesc:
        d = _lib.RegHeadDesc()
        d.B, (d.depth, d.heads, d.mlp_dim) = B, self.dims
        d.params = self._flat.data_ptr()
        d.init_body_pose, d.init_betas = self.init_body_pose.data_ptr(), self.init_betas.data_ptr()
        d.init_cam = self.init_cam.data_ptr()
        d.feats = feats.data_ptr()
        d.workspace, d.workspace_bytes = ws.data_ptr(), ws.numel()
        d.stream = torch.cuda.current_stream(feats.device).cuda_stream
        return d

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
        for name, g, shape in (("grad_pose6d", g_pose6d, (B, _NPOSE)), ("grad_betas", g_betas, (B, _NUM_BETAS)),
                               ("grad_cam", g_cam, (B, 3)), ("grad_rotmats", g_rot, (B, 24, 3, 3))):
            if g is not None:
                g = g.to(torch.float32).contiguous()
                assert tuple(g.shape) == shape, (name, tuple(g.shape))
                held.append(g)
                setattr(d, name, g.data_ptr())
        check(lib().thmr_reg_head_backward(ctypes.byref(d)))
        out = [grads[off:off + _numel(shape)].view(shape) for _, shape, off in head._layout]
        return (None, None, None, *out)


def _numel(shape) -> int:
    n = 1
    for s in shape:
        n *= s
    return n

"""Host-side weight packer: reference state_dicts -> device tensors laid out for the engine.

Accepts the key names of the reference checkpoints:
  * TokenHMR Lightning checkpoint ckpt['state_dict'] with prefixes 'backbone.' / 'smpl_head.'
    (tokenhmr/lib/utils/misc.py:215-256 prepare_statedict / load_pretrained); with cfg.head == "transformer_decoder"
    the HMR 2.0 checkpoint's head (heads/smpl_head.py:14-50: transformer.*, decpose, decshape, deccam, init_*),
  * tokenizer.pth {'net': {'decoder.*', 'quantizer.codebook', ...}, 'hparams': ...} under the prefix
    'tokenizer.' (tokenization/models/vanilla_pose_vqvae.py:24-40,299-301; 'body_model' keys skipped),
and produces fp16 [out,in] matrices / fp32 vectors on the GPU plus the ctypes thmr_weights struct.
Pure data movement (casts, concatenations, transposes): host glue, not part of the hot path.
"""
from __future__ import annotations

import ctypes
from typing import Dict, List

import torch

from . import _lib
from . import fp8 as _fp8
from .config import TokenHMRConfig


def strip_checkpoint(state_dict: Dict[str, torch.Tensor], tokenizer_net: Dict[str, torch.Tensor] | None = None
                     ) -> Dict[str, torch.Tensor]:
    """Merge a TokenHMR checkpoint state_dict and a tokenizer 'net' dict into the flat naming used here."""
    out = {k: v for k, v in state_dict.items() if k.startswith(("backbone.", "smpl_head."))}
    if tokenizer_net is not None:
        for k, v in tokenizer_net.items():
            if "body_model" in k:
                continue
            if k.startswith(("decoder.", "quantizer.")):
                out["tokenizer." + k] = v
    return out


STRICT_W_SCALE = 256.0     # kStrictWScale (csrc/strict.cuh)


def split_weight(t: torch.Tensor, taps: int = 1) -> torch.Tensor:
    """[out, taps*in] -> f16 [out, taps*3*in], per tap [hi | hi | lo] of w * STRICT_W_SCALE (hi = fp16(w * 2^8),
    lo = fp16(w * 2^8 - hi)): the B operand of the split-precision GEMMs (csrc/strict.cuh)."""
    t = t.detach().to(dtype=torch.float32)
    amax = float(t.abs().max()) if t.numel() else 0.0
    if not amax < 65504.0 / STRICT_W_SCALE:
        raise _lib.ThmrError(f"split precision: weight magnitude {amax:g} exceeds the split-fp16 range "
                             f"(|w| < {65504.0 / STRICT_W_SCALE:g})")
    ws = t * STRICT_W_SCALE
    hi = ws.to(torch.float16)
    lo = (ws - hi.to(torch.float32)).to(torch.float16)
    out_f, k = t.shape
    cin = k // taps
    hi3, lo3 = hi.view(out_f, taps, cin), lo.view(out_f, taps, cin)
    return torch.cat([hi3, hi3, lo3], dim=2).reshape(out_f, taps * 3 * cin).contiguous()


class PackedWeights:
    """Owns the device tensors the engine points into (must outlive the engine)."""

    def __init__(self, sd: Dict[str, torch.Tensor], cfg: TokenHMRConfig, device: torch.device, strict: bool = False,
                 fp8: bool = False):
        """strict: matrices are packed for the split-fp16 GEMMs of strict mode (csrc/strict.cuh): f16 [out, 3*in] =
        [hi | hi | lo] of w * 2^8 with hi = fp16(w * 2^8), lo = fp16(w * 2^8 - hi); conv weights per tap.
        fp8: each ViT block's qkv, fc1 and fc2 weights are e4m3 [out, in] codes with one power-of-two scale per
        128 x 128 block (tokenhmr_b200/fp8.py, quantised from fp32 on the device); everything else as by default."""
        if strict and fp8:
            raise _lib.ThmrError("strict and fp8 are exclusive numeric modes")
        self.cfg = cfg
        self.device = device
        self.strict = bool(strict)
        self.fp8 = bool(fp8)
        self._keep: List[torch.Tensor] = []
        self.keys_read: List[str] = []     # every state-dict entry the packer used, in order

        def g(n: str) -> torch.Tensor:
            self.keys_read.append(n)
            return sd[n]

        def f16(t: torch.Tensor, taps: int = 1) -> int:
            if self.strict:
                t = split_weight(t.detach().to(device=device), taps)
            else:
                t = t.detach().to(device=device, dtype=torch.float16).contiguous()
            self._keep.append(t)
            return t.data_ptr()

        def vit_w(t: torch.Tensor, i: int, scale_field: str) -> int:
            """A ViT GEMM weight that the FP8 mode runs on e4m3: its codes, with the block scales recorded."""
            if not self.fp8:
                return f16(t)
            codes, scales = _fp8.quantize_weight_blocks(t.detach().to(device=device, dtype=torch.float32))
            self._keep += [codes, scales]
            setattr(self.block_scales[i], scale_field, scales.data_ptr())
            return codes.data_ptr()

        def f32(t: torch.Tensor) -> int:
            t = t.detach().to(device=device, dtype=torch.float32).contiguous()
            self._keep.append(t)
            return t.data_ptr()

        def conv(prefix: str) -> _lib.Conv:
            w = g(prefix + ".weight")                      # [Cout, Cin, k]
            cout, cin, k = w.shape
            wt = w.permute(0, 2, 1).reshape(cout, k * cin)  # tap-major: column = tap*Cin + c
            return _lib.Conv(f16(wt, taps=k), f32(g(prefix + ".bias")))

        W = _lib.Weights()
        D = cfg.vit_dim
        # ---- ViT
        W.patch_w = f16(g("backbone.patch_embed.proj.weight").reshape(D, -1))
        W.patch_b = f32(g("backbone.patch_embed.proj.bias"))
        pos = g("backbone.pos_embed")
        W.pos = f32(pos[0, 1:] + pos[0, :1])               # vit.py:327
        self.blocks = (_lib.VitBlock * cfg.vit_depth)()
        self.block_scales = (_lib.VitBlockScales * cfg.vit_depth)()
        for i in range(cfg.vit_depth):
            p = f"backbone.blocks.{i}."
            b = self.blocks[i]
            b.ln1_g, b.ln1_b = f32(g(p + "norm1.weight")), f32(g(p + "norm1.bias"))
            b.qkv_w, b.qkv_b = vit_w(g(p + "attn.qkv.weight"), i, "qkv_ws"), f32(g(p + "attn.qkv.bias"))
            b.proj_w, b.proj_b = f16(g(p + "attn.proj.weight")), f32(g(p + "attn.proj.bias"))
            b.ln2_g, b.ln2_b = f32(g(p + "norm2.weight")), f32(g(p + "norm2.bias"))
            b.fc1_w, b.fc1_b = vit_w(g(p + "mlp.fc1.weight"), i, "fc1_ws"), f32(g(p + "mlp.fc1.bias"))
            b.fc2_w, b.fc2_b = vit_w(g(p + "mlp.fc2.weight"), i, "fc2_ws"), f32(g(p + "mlp.fc2.bias"))
        W.blocks_host = ctypes.cast(self.blocks, ctypes.POINTER(_lib.VitBlock))
        if self.fp8:
            W.block_scales_host = ctypes.cast(self.block_scales, ctypes.POINTER(_lib.VitBlockScales))
        W.last_g, W.last_b = f32(g("backbone.last_norm.weight")), f32(g("backbone.last_norm.bias"))
        # ---- decoder
        t = "smpl_head.transformer."
        inner = cfg.dec_inner
        # to_token_embedding(zeros(B, 1, 1)) = its bias: the weight multiplies the zero query token (token_head.py:91,
        # smpl_head.py:75); a (E, npose + 13) weight would be TRANSFORMER_INPUT='mean_shape', which is not implemented
        if g(t + "to_token_embedding.weight").shape[1] != 1:
            raise _lib.ThmrError("to_token_embedding takes more than one input: a TRANSFORMER_INPUT='mean_shape' "
                                 "checkpoint is not supported")
        W.token0 = f32(g(t + "to_token_embedding.bias") + g(t + "pos_embedding")[0, 0])
        W.kv_w = f16(torch.cat([g(f"{t}transformer.layers.{l}.1.fn.to_kv.weight") for l in range(cfg.dec_depth)], 0))
        self.dec = (_lib.DecLayer * cfg.dec_depth)()
        for l in range(cfg.dec_depth):
            p = f"{t}transformer.layers.{l}."
            d = self.dec[l]
            d.ln0_g, d.ln0_b = f32(g(p + "0.norm.weight")), f32(g(p + "0.norm.bias"))
            d.sa_v_w = f16(g(p + "0.fn.to_qkv.weight")[2 * inner:3 * inner])
            d.sa_out_w, d.sa_out_b = f16(g(p + "0.fn.to_out.0.weight")), f32(g(p + "0.fn.to_out.0.bias"))
            d.ln1_g, d.ln1_b = f32(g(p + "1.norm.weight")), f32(g(p + "1.norm.bias"))
            d.ca_q_w = f16(g(p + "1.fn.to_q.weight"))
            d.ca_out_w, d.ca_out_b = f16(g(p + "1.fn.to_out.0.weight")), f32(g(p + "1.fn.to_out.0.bias"))
            d.ln2_g, d.ln2_b = f32(g(p + "2.norm.weight")), f32(g(p + "2.norm.bias"))
            d.ff1_w, d.ff1_b = f16(g(p + "2.fn.net.0.weight")), f32(g(p + "2.fn.net.0.bias"))
            d.ff2_w, d.ff2_b = f16(g(p + "2.fn.net.3.weight")), f32(g(p + "2.fn.net.3.bias"))
        W.dec_host = ctypes.cast(self.dec, ctypes.POINTER(_lib.DecLayer))
        h = "smpl_head."
        regression = cfg.head == "transformer_decoder"
        if regression:
            order, rows = ["decpose", "decshape", "deccam"], 160            # 144 | 10 | 3 (+3 zero rows)
        else:
            order, rows = ["decpose_grot", "decpose_hands", "decshape", "deccam"], 32   # 6 | 12 | 10 | 3 (+1 zero row)
        rw = torch.cat([g(h + n + ".weight") for n in order], 0)
        rb = torch.cat([g(h + n + ".bias") for n in order], 0)
        pad = rows - rw.shape[0]
        rw = torch.cat([rw, torch.zeros(pad, cfg.dec_dim)], 0)
        rb = torch.cat([rb, torch.zeros(pad)], 0)
        W.readout_w, W.readout_b = f16(rw), f32(rb)
        W.init_pose = f32(g(h + "init_body_pose").reshape(-1))
        W.init_betas = f32(g(h + "init_betas").reshape(-1))
        W.init_cam = f32(g(h + "init_cam").reshape(-1))
        if regression:
            # no classifier and no tokenizer: their pointers stay NULL (thmr_engine_create_head)
            self.mixer = None
            self.struct = W
            return
        # ---- classifier
        c = h + "decpose."
        W.mt_w, W.mt_b = f16(g(c + "mixer_trans.ff.0.weight")), f32(g(c + "mixer_trans.ff.0.bias"))
        W.mt_ln_g, W.mt_ln_b = f32(g(c + "mixer_trans.ff.1.weight")), f32(g(c + "mixer_trans.ff.1.bias"))
        self.mixer = (_lib.MixerBlock * cfg.cls_blocks)()
        for i in range(cfg.cls_blocks):
            p = f"{c}mixer_head.{i}."
            m = self.mixer[i]
            m.ln1_g, m.ln1_b = f32(g(p + "layernorm1.weight")), f32(g(p + "layernorm1.bias"))
            m.tok1_w, m.tok1_b = f16(g(p + "MLP_token.ff.0.weight")), f32(g(p + "MLP_token.ff.0.bias"))
            m.tok2_w, m.tok2_b = f16(g(p + "MLP_token.ff.3.weight")), f32(g(p + "MLP_token.ff.3.bias"))
            m.ln2_g, m.ln2_b = f32(g(p + "layernorm2.weight")), f32(g(p + "layernorm2.bias"))
            m.ch1_w, m.ch1_b = f16(g(p + "MLP_channel.ff.0.weight")), f32(g(p + "MLP_channel.ff.0.bias"))
            m.ch2_w, m.ch2_b = f16(g(p + "MLP_channel.ff.3.weight")), f32(g(p + "MLP_channel.ff.3.bias"))
        W.mixer_host = ctypes.cast(self.mixer, ctypes.POINTER(_lib.MixerBlock))
        W.mn_w, W.mn_b = f16(g(c + "mixer_norm_layer.ff.0.weight")), f32(g(c + "mixer_norm_layer.ff.0.bias"))
        W.mn_ln_g, W.mn_ln_b = f32(g(c + "mixer_norm_layer.ff.1.weight")), f32(g(c + "mixer_norm_layer.ff.1.bias"))
        W.cls_w, W.cls_b = f16(g(c + "class_pred_layer.weight")), f32(g(c + "class_pred_layer.bias"))
        # ---- tokenizer (Sequential indices of PoseSPDecoderV1.decoder, vanilla_pose_vqvae.py:135-154)
        tk = "tokenizer.decoder.decoder."
        W.codebook_t = f16(g("tokenizer.quantizer.codebook").t())
        W.conv_in = conv(tk + "0")
        idx = 2
        for u in range(len(cfg.upsample_sizes)):
            W.conv_up[u] = conv(f"{tk}{idx + 1}")
            idx += 3
        for d_ in range(cfg.tok_depth):
            W.res_conv1[d_] = conv(f"{tk}{idx}.0.model.{d_}.conv1")
            W.res_conv2[d_] = conv(f"{tk}{idx}.0.model.{d_}.conv2")
        W.conv_post = conv(f"{tk}{idx}.1")
        W.conv_out = conv(f"{tk}{idx + 1}")
        self.struct = W

    def nbytes(self) -> int:
        return sum(t.numel() * t.element_size() for t in self._keep)


def make_config_struct(cfg: TokenHMRConfig, strict: bool = False, concurrent: bool = False,
                       fp8: bool = False) -> _lib.Config:
    if strict and fp8:
        raise _lib.ThmrError("strict and fp8 are exclusive numeric modes")
    c = _lib.Config()
    c.strict = 1 if strict else 0
    c.concurrent = 1 if concurrent else 0
    c.fp8 = 1 if fp8 else 0
    for f in ("image_size", "crop_w", "patch", "patch_pad", "vit_dim", "vit_depth", "vit_heads", "vit_mlp_ratio",
              "vit_ln_eps", "dec_dim", "dec_depth", "dec_heads", "dec_dim_head", "dec_mlp_dim", "ln_eps", "token_num",
              "token_class_num", "cls_hidden", "cls_hidden_inter", "cls_token_inter", "cls_blocks", "code_dim",
              "tok_width", "tok_depth", "tok_dilation_rate", "tok_joints", "focal_length"):
        setattr(c, f, getattr(cfg, f))
    ups = cfg.upsample_sizes
    c.n_upsample = len(ups)
    for i, v in enumerate(ups):
        c.upsample_sizes[i] = v
    return c

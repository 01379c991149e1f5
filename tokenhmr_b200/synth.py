"""Seeded synthetic weights and a synthetic SMPL-shaped body model.

The reference ships no checkpoints, no SMPL .pkl, no mean params and no tokenizer.pth (licence-gated,
fetch_demo_data.sh:26-34), so parity tests and the benchmark use tensors generated here.  Names and
shapes are exactly those of the reference state_dicts, so a real checkpoint loads through the same
packer (tokenhmr_b200/weights.py):

  backbone.*    ViT             tokenhmr/lib/models/backbones/vit.py:209-255
  smpl_head.*   token head      tokenhmr/lib/models/heads/token_head.py:20-63, token_classifier.py:52-86,
                                components/pose_transformer.py:160-201,301-347
                or, with cfg.head == "transformer_decoder", the regression head  heads/smpl_head.py:14-50
  tokenizer.*   'net' dict of tokenizer.pth: decoder.* / quantizer.codebook
                                tokenization/models/vanilla_pose_vqvae.py:113-154, quantize_cnn.py:14-18
  smpl.*        body-model buffers of smplx.SMPLLayer + joint_regressor_extra (smpl_wrapper.py:11-25)

Every tensor is drawn from its own torch CPU generator seeded by (seed, crc32(name)): a depth-2 model is
a strict subset of the depth-32 model, and generation is reproducible on any host with the same torch.
"""
from __future__ import annotations

import zlib
from typing import Dict

import numpy as np
import torch

from .config import SMPL_EXTRA_VERTEX_IDS, SMPL_PARENTS, TokenHMRConfig


def _gen(seed: int, name: str) -> torch.Generator:
    g = torch.Generator(device="cpu")
    g.manual_seed((seed * 1000003 + zlib.crc32(name.encode())) % (2 ** 63 - 1))
    return g


class _Maker:
    def __init__(self, seed: int):
        self.seed = seed
        self.sd: Dict[str, torch.Tensor] = {}

    def normal(self, name, shape, std):
        self.sd[name] = torch.randn(*shape, generator=_gen(self.seed, name), dtype=torch.float32) * std
        return self.sd[name]

    def uniform(self, name, shape, bound):
        self.sd[name] = (torch.rand(*shape, generator=_gen(self.seed, name), dtype=torch.float32) * 2 - 1) * bound
        return self.sd[name]

    def linear(self, prefix, out_f, in_f, bias=True, gain=1.0):
        # PyTorch nn.Linear default: U(-1/sqrt(fan_in), 1/sqrt(fan_in)) for weight and bias
        b = gain / np.sqrt(in_f)
        self.uniform(prefix + ".weight", (out_f, in_f), b)
        if bias:
            self.uniform(prefix + ".bias", (out_f,), b)

    def conv1d(self, prefix, out_c, in_c, k):
        b = 1.0 / np.sqrt(in_c * k)
        self.uniform(prefix + ".weight", (out_c, in_c, k), b)
        self.uniform(prefix + ".bias", (out_c,), b)

    def layernorm(self, prefix, dim):
        # perturbed affine so that gamma/beta handling is actually tested
        self.sd[prefix + ".weight"] = 1.0 + 0.1 * torch.randn(dim, generator=_gen(self.seed, prefix + ".weight"))
        self.sd[prefix + ".bias"] = 0.05 * torch.randn(dim, generator=_gen(self.seed, prefix + ".bias"))


def make_state_dict(cfg: TokenHMRConfig, seed: int = 1234) -> Dict[str, torch.Tensor]:
    """Synthetic fp32 parameters for backbone.*, smpl_head.* and tokenizer.* (CPU tensors).  The regression head
    (cfg.head == "transformer_decoder") has the same backbone.* and smpl_head.transformer.* tensors and no tokenizer."""
    m = _Maker(seed)
    D = cfg.vit_dim
    # ---- ViT (vit.py:240-255)
    b = 1.0 / np.sqrt(3 * cfg.patch * cfg.patch)
    m.uniform("backbone.patch_embed.proj.weight", (D, 3, cfg.patch, cfg.patch), b)
    m.uniform("backbone.patch_embed.proj.bias", (D,), b)
    m.normal("backbone.pos_embed", (1, cfg.num_tokens + 1, D), 0.02)
    for i in range(cfg.vit_depth):
        p = f"backbone.blocks.{i}"
        m.layernorm(p + ".norm1", D)
        m.linear(p + ".attn.qkv", 3 * D, D)
        m.linear(p + ".attn.proj", D, D)
        m.layernorm(p + ".norm2", D)
        m.linear(p + ".mlp.fc1", cfg.vit_mlp_ratio * D, D)
        m.linear(p + ".mlp.fc2", D, cfg.vit_mlp_ratio * D)
    m.layernorm("backbone.last_norm", D)

    # ---- decoder (pose_transformer.py:301-347, 160-189)
    E = cfg.dec_dim
    inner = cfg.dec_inner
    m.linear("smpl_head.transformer.to_token_embedding", E, 1)
    m.normal("smpl_head.transformer.pos_embedding", (1, 1, E), 1.0)
    for l in range(cfg.dec_depth):
        p = f"smpl_head.transformer.transformer.layers.{l}"
        m.layernorm(p + ".0.norm", E)
        m.linear(p + ".0.fn.to_qkv", 3 * inner, E, bias=False)
        m.linear(p + ".0.fn.to_out.0", E, inner)
        m.layernorm(p + ".1.norm", E)
        m.linear(p + ".1.fn.to_kv", 2 * inner, cfg.vit_dim, bias=False)
        m.linear(p + ".1.fn.to_q", inner, E, bias=False)
        m.linear(p + ".1.fn.to_out.0", E, inner)
        m.layernorm(p + ".2.norm", E)
        m.linear(p + ".2.fn.net.0", cfg.dec_mlp_dim, E)
        m.linear(p + ".2.fn.net.3", E, cfg.dec_mlp_dim)
    if cfg.head == "transformer_decoder":
        # read-outs (smpl_head.py:32-34); the small decpose gain keeps all 24 rotations near the identity mean pose
        # (well-conditioned 6D), as decpose_grot's does for the token head
        m.linear("smpl_head.decpose", cfg.npose, E, gain=0.1)
        m.linear("smpl_head.decshape", 10, E, gain=0.5)
        m.linear("smpl_head.deccam", 3, E, gain=0.1)
        _mean_params(m, cfg)
        return m.sd
    # read-outs (token_head.py:40-43); small gain keeps the pose near the mean pose (well-conditioned 6D)
    m.linear("smpl_head.decpose_grot", 6, E, gain=0.3)
    m.linear("smpl_head.decshape", 10, E, gain=0.5)
    m.linear("smpl_head.deccam", 3, E, gain=0.1)
    m.linear("smpl_head.decpose_hands", 12, E, gain=0.3)
    _mean_params(m, cfg)

    # ---- token classifier (token_classifier.py:67-80, modules.py)
    H = cfg.cls_hidden
    c = "smpl_head.decpose"
    m.linear(c + ".mixer_trans.ff.0", cfg.token_num * H, E)
    m.layernorm(c + ".mixer_trans.ff.1", cfg.token_num * H)
    for i in range(cfg.cls_blocks):
        p = f"{c}.mixer_head.{i}"
        m.layernorm(p + ".layernorm1", H)
        m.linear(p + ".MLP_token.ff.0", cfg.cls_token_inter, cfg.token_num)
        m.linear(p + ".MLP_token.ff.3", cfg.token_num, cfg.cls_token_inter)
        m.layernorm(p + ".layernorm2", H)
        m.linear(p + ".MLP_channel.ff.0", cfg.cls_hidden_inter, H)
        m.linear(p + ".MLP_channel.ff.3", H, cfg.cls_hidden_inter)
    m.linear(c + ".mixer_norm_layer.ff.0", H, H)
    m.layernorm(c + ".mixer_norm_layer.ff.1", H)
    m.linear(c + ".class_pred_layer", cfg.token_class_num, H, gain=20.0)  # peaky softmax (SURVEY §7 hard parts)

    # ---- tokenizer decoder + codebook (vanilla_pose_vqvae.py:135-154; Sequential indices as saved)
    W = cfg.tok_width
    t = "tokenizer.decoder.decoder"
    m.conv1d(f"{t}.0", W, cfg.code_dim, 3)
    idx = 2
    for _ in cfg.upsample_sizes:
        m.conv1d(f"{t}.{idx + 1}", W, W, 3)   # [Upsample, Conv1d, ReLU]
        idx += 3
    for d in range(cfg.tok_depth):            # Resnet1D blocks (resnet.py:12-68)
        m.conv1d(f"{t}.{idx}.0.model.{d}.conv1", W, W, 3)
        m.conv1d(f"{t}.{idx}.0.model.{d}.conv2", W, W, 1)
    m.conv1d(f"{t}.{idx}.1", W, W, 3)
    m.conv1d(f"{t}.{idx + 1}", 6, W, 3)
    m.normal("tokenizer.quantizer.codebook", (cfg.nb_code, cfg.code_dim), 1.0)
    return m.sd


def _mean_params(m: _Maker, cfg: TokenHMRConfig) -> None:
    """Mean params (token_head.py:57-63, smpl_head.py:42-48): identity 6D pose, zero shape, cam [0.9, 0, 0]."""
    m.sd["smpl_head.init_body_pose"] = torch.tensor([1., 0., 0., 0., 1., 0.] * cfg.num_joints).view(1, -1)
    m.sd["smpl_head.init_betas"] = torch.zeros(1, cfg.num_betas)
    m.sd["smpl_head.init_cam"] = torch.tensor([[0.9, 0.0, 0.0]])


def make_tokenizer_encoder_state_dict(cfg: TokenHMRConfig, seed: int = 1234) -> Dict[str, torch.Tensor]:
    """Synthetic 'tokenizer.encoder.encoder.*' parameters (PoseSPEncoderV1, vanilla_pose_vqvae.py:65-86; Sequential
    indices as the reference saves them) + 'tokenizer.quantizer.codebook' (the same tensor make_state_dict produces:
    every tensor is seeded by its own name).  Kept out of make_state_dict: the forward path does not use them."""
    m = _Maker(seed)
    W = cfg.tok_width
    t = "tokenizer.encoder.encoder"
    m.conv1d(f"{t}.0", W, 6, 3)
    m.conv1d(f"{t}.3", W, W, 3)
    idx = 5
    for _ in range(cfg.tok_size_mul - 1):
        m.conv1d(f"{t}.{idx + 1}", W, W, 3)
        idx += 3
    m.conv1d(f"{t}.{idx}.0", W, W, 4)
    for d in range(cfg.tok_depth):
        m.conv1d(f"{t}.{idx}.1.model.{d}.conv1", W, W, 3)
        m.conv1d(f"{t}.{idx}.1.model.{d}.conv2", W, W, 1)
    m.conv1d(f"{t}.{idx + 1}", cfg.code_dim, W, 3)
    # random-init latents are ~0.03 in scale against a unit-variance codebook (every query would pick the code of
    # smallest norm): scale the last conv so that the arg-min actually depends on the query
    for n in (f"{t}.{idx + 1}.weight", f"{t}.{idx + 1}.bias"):
        m.sd[n] = m.sd[n] * 40.0
    m.normal("tokenizer.quantizer.codebook", (cfg.nb_code, cfg.code_dim), 1.0)
    return m.sd


def make_smpl(cfg: TokenHMRConfig, seed: int = 3) -> Dict[str, torch.Tensor]:
    """Synthetic SMPL-shaped body model (fp32 CPU tensors), keys as the smplx buffers:
    v_template (V,3), shapedirs (V,3,10), posedirs (207, V*3), J_regressor (24,V), lbs_weights (V,24),
    parents (24,), joint_regressor_extra (19,V), extra_vertex_ids (21,), joint_map (25,)."""
    V, J = cfg.num_verts, cfg.num_joints
    g = lambda n: _gen(seed, "smpl." + n)
    out: Dict[str, torch.Tensor] = {}
    out["v_template"] = (torch.rand(V, 3, generator=g("v_template")) * 2 - 1) * torch.tensor([0.3, 0.9, 0.15])
    out["shapedirs"] = torch.randn(V, 3, cfg.num_betas, generator=g("shapedirs")) * 0.01
    out["posedirs"] = torch.randn((J - 1) * 9, V * 3, generator=g("posedirs")) * 0.003

    def sparse_rows(name, rows, nnz):
        w = torch.zeros(rows, V)
        idx = torch.randint(0, V, (rows, nnz), generator=g(name + ".idx"))
        val = torch.rand(rows, nnz, generator=g(name + ".val")) + 0.05
        w.scatter_add_(1, idx, val)
        return w / w.sum(1, keepdim=True)

    out["J_regressor"] = sparse_rows("J_regressor", J, 30)
    out["joint_regressor_extra"] = sparse_rows("J_extra", 19, 30)
    # skinning weights: 4 non-zeros per vertex, rows sum to one
    lw = torch.zeros(V, J)
    jidx = torch.randint(0, J, (V, 4), generator=g("lbs.idx"))
    jval = torch.rand(V, 4, generator=g("lbs.val")) + 0.05
    lw.scatter_add_(1, jidx, jval)
    out["lbs_weights"] = lw / lw.sum(1, keepdim=True)
    out["parents"] = torch.tensor(SMPL_PARENTS[:J], dtype=torch.int64)
    ids = SMPL_EXTRA_VERTEX_IDS if V == 6890 else [(i * 7919) % V for i in range(21)]
    out["extra_vertex_ids"] = torch.tensor(ids, dtype=torch.int64)
    return out


def make_images(batch: int, cfg: TokenHMRConfig, seed: int = 0) -> torch.Tensor:
    """ImageNet-normalised crops are ~N(0,1): batch['img'] stand-in, (B,3,256,256) fp32."""
    return torch.randn(batch, 3, cfg.image_size, cfg.image_size, generator=_gen(seed, "img"), dtype=torch.float32)

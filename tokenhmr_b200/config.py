"""Plain hyper-parameter struct for the TokenHMR forward path.

Mirrors the keys the reference reads at construction time (SURVEY.md §8 header):
  ViT        tokenhmr/lib/models/backbones/vit.py:12-24
  decoder    tokenhmr/lib/configs_hydra/experiment/tokenhmr_release.yaml:73-81, heads/token_head.py:30-38
  classifier heads/token_classifier.py:56-63, tokenhmr_release.yaml:69-72
  tokenizer  tokenization/configs/tokenizer_amass_moyo.yaml:41-53, models/vanilla_pose_vqvae.py:258-293
  regression head  heads/smpl_head.py:14-34 (MODEL.SMPL_HEAD.TYPE: transformer_decoder)
  SMPL       tokenhmr_release.yaml:31-37;  EXTRA.FOCAL_LENGTH / MODEL.IMAGE_SIZE default.yaml:12, release:57
"""
from __future__ import annotations

from dataclasses import asdict, dataclass
from typing import List

import numpy as np


HEADS = ("token", "transformer_decoder")


@dataclass(frozen=True)
class TokenHMRConfig:
    # --- ViT-H/16 backbone (input 256x256, centre-cropped to 256x192: vit.py:341-343)
    image_size: int = 256          # MODEL.IMAGE_SIZE: forward() takes (B,3,256,256)
    crop_w: int = 192              # width after x[:, :, :, 32:-32]
    patch: int = 16
    patch_pad: int = 2             # PatchEmbed padding = 4 + 2*(ratio//2-1) with ratio=1 (vit.py:168)
    vit_dim: int = 1280
    vit_depth: int = 32
    vit_heads: int = 16
    vit_mlp_ratio: int = 4
    vit_ln_eps: float = 1e-6       # vit.py:222
    # --- one-token cross-attention decoder
    dec_dim: int = 1024
    dec_depth: int = 6
    dec_heads: int = 8
    dec_dim_head: int = 64
    dec_mlp_dim: int = 1024
    ln_eps: float = 1e-5           # torch default, t_cond_mlp.py:51-52 / modules.py:17,50,52
    # --- MLP-Mixer token classifier
    token_num: int = 160
    token_class_num: int = 2048
    cls_hidden: int = 64
    cls_hidden_inter: int = 256
    cls_token_inter: int = 64
    cls_blocks: int = 4
    # --- VQ-VAE tokenizer (decoder + codebook)
    code_dim: int = 256
    nb_code: int = 2048
    tok_width: int = 512
    tok_depth: int = 2
    tok_dilation_rate: int = 3
    tok_size_div: int = 4
    tok_size_mul: int = 4          # ARCH.TOKEN_SIZE_MUL (encoder: 21 -> 40 -> 80 -> 160 -> 320 -> stride 2 -> 160)
    tok_joints: int = 21
    # --- SMPL
    num_verts: int = 6890
    num_joints: int = 24
    num_betas: int = 10
    focal_length: float = 5000.0
    # --- SMPL head (MODEL.SMPL_HEAD.TYPE, heads/__init__.py:4-13): "token" (SMPLTokenDecoderHead: token classifier +
    # tokenizer decoder) or "transformer_decoder" (SMPLTransformerDecoderHead, HMR 2.0's regression head: decpose /
    # decshape / deccam read the decoder's output token directly, smpl_head.py:32-34,82-84; no token classifier, no
    # tokenizer, no cls_logits_softmax)
    head: str = "token"

    def __post_init__(self):
        if self.head not in HEADS:
            raise ValueError(f"TokenHMRConfig.head = {self.head!r}; one of {HEADS}")

    # derived ------------------------------------------------------------------------------------
    @property
    def grid_h(self) -> int:
        return (self.image_size + 2 * self.patch_pad - self.patch) // self.patch + 1

    @property
    def grid_w(self) -> int:
        return (self.crop_w + 2 * self.patch_pad - self.patch) // self.patch + 1

    @property
    def num_tokens(self) -> int:
        return self.grid_h * self.grid_w           # 16 * 12 = 192

    @property
    def head_dim(self) -> int:
        return self.vit_dim // self.vit_heads      # 80

    @property
    def crop_x0(self) -> int:
        return (self.image_size - self.crop_w) // 2  # 32

    @property
    def dec_inner(self) -> int:
        return self.dec_heads * self.dec_dim_head  # 512

    @property
    def upsample_sizes(self) -> List[int]:
        """nn.Upsample(size) targets of PoseSPDecoderV1 (vanilla_pose_vqvae.py:139): 125, 90, 55, 21."""
        return [int(v) for v in np.linspace(self.tok_joints, self.token_num, self.tok_size_div,
                                            endpoint=False, dtype=int)[::-1]]

    @property
    def npose(self) -> int:
        return 6 * self.num_joints                 # 144

    def to_dict(self) -> dict:
        return asdict(self)


def release_config() -> TokenHMRConfig:
    """The TokenHMR release configuration (ViT-H/16, 630.9 M backbone parameters)."""
    return TokenHMRConfig()


def tiny_config(vit_depth: int = 2, num_verts: int = 431, head: str = "token") -> TokenHMRConfig:
    """Same layer shapes, fewer ViT blocks / SMPL vertices: for CPU-speed tests."""
    return TokenHMRConfig(vit_depth=vit_depth, num_verts=num_verts, head=head)


# SMPL kinematic tree (smplx body_models, SMPL: 24 joints)
SMPL_PARENTS = [-1, 0, 0, 0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 9, 9, 12, 13, 14, 16, 17, 18, 19, 20, 21]
# smplx.vertex_ids.vertex_ids['smplh'] in VertexJointSelector order (face, feet, finger tips): 21 extras
SMPL_EXTRA_VERTEX_IDS = [332, 6260, 2800, 4071, 583, 3216, 3226, 3387, 6617, 6624, 6787,
                         2746, 2319, 2445, 2556, 2673, 6191, 5782, 5905, 6016, 6133]
# tokenhmr/lib/models/smpl_wrapper.py:19-20
SMPL_TO_OPENPOSE = [24, 12, 17, 19, 21, 16, 18, 20, 0, 2, 5, 8, 1, 4, 7, 25, 26, 27, 28, 29, 30, 31, 32, 33, 34]

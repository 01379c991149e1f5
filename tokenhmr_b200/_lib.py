"""ctypes binding of libtokenhmr_b200.so (the C ABI in include/tokenhmr_b200.h).

There is deliberately no fallback: if the shared library is missing or a call fails, we raise.
"""
from __future__ import annotations

import ctypes
from ctypes import POINTER, Structure, c_char_p, c_float, c_int, c_int32, c_int64, c_size_t, c_void_p
from pathlib import Path

LIB_PATH = Path(__file__).resolve().parent / "libtokenhmr_b200.so"
_lib = None


class ThmrError(RuntimeError):
    pass


# ---- structs mirroring include/tokenhmr_b200.h -------------------------------------------------------
class SmplDesc(Structure):
    _fields_ = [("num_verts", c_int), ("num_betas", c_int), ("v_template", c_void_p), ("shapedirs", c_void_p),
                ("posedirs", c_void_p), ("J_regressor", c_void_p), ("lbs_weights", c_void_p),
                ("parents_host", POINTER(c_int32)), ("joint_regressor_extra", c_void_p), ("n_extra", c_int),
                ("extra_vertex_ids_host", POINTER(c_int32)), ("joint_map_host", POINTER(c_int32))]


class SmplifyDesc(Structure):
    _fields_ = [("B", c_int), ("num_iters", c_int), ("num_joints", c_int),
                ("step_size", ctypes.c_double), ("margin", ctypes.c_double), ("loss_thresh_f2d", ctypes.c_double),
                ("loss_thresh_f3d", ctypes.c_double),
                ("global_orient", c_void_p), ("body_pose", c_void_p), ("pred_cam_t", c_void_p), ("betas", c_void_p),
                ("focal_length", c_void_p), ("gt_keypoints_2d", c_void_p), ("gt_keypoints_3d", c_void_p),
                ("vertices", c_void_p), ("joints", c_void_p), ("pj2ds", c_void_p), ("reprojection_loss", c_void_p),
                ("history", c_void_p), ("iters_run", c_void_p)]


class LossDesc(Structure):
    _fields_ = [("B", c_int), ("num_joints", c_int), ("num_betas", c_int), ("tals", c_int), ("pelvis_id", c_int),
                ("loose_weight", ctypes.c_double), ("w_keypoints_2d", ctypes.c_double),
                ("w_keypoints_3d", ctypes.c_double), ("w_global_orient", ctypes.c_double),
                ("w_body_pose", ctypes.c_double), ("w_betas", ctypes.c_double)] + \
               [(n, c_void_p) for n in ("pred_keypoints_2d", "pred_keypoints_3d", "pred_rotmats", "pred_betas",
                                        "gt_keypoints_2d", "gt_keypoints_3d", "gt_global_orient", "gt_body_pose",
                                        "gt_betas", "has_global_orient", "has_body_pose", "has_betas", "valid_3d",
                                        "is_axis_angle_global_orient", "is_axis_angle_body_pose",
                                        "is_axis_angle_betas", "losses", "grad_keypoints_2d", "grad_keypoints_3d",
                                        "grad_rotmats", "grad_betas")]


class Config(Structure):
    _fields_ = [("image_size", c_int), ("crop_w", c_int), ("patch", c_int), ("patch_pad", c_int),
                ("vit_dim", c_int), ("vit_depth", c_int), ("vit_heads", c_int), ("vit_mlp_ratio", c_int),
                ("vit_ln_eps", c_float),
                ("dec_dim", c_int), ("dec_depth", c_int), ("dec_heads", c_int), ("dec_dim_head", c_int),
                ("dec_mlp_dim", c_int), ("ln_eps", c_float),
                ("token_num", c_int), ("token_class_num", c_int), ("cls_hidden", c_int), ("cls_hidden_inter", c_int),
                ("cls_token_inter", c_int), ("cls_blocks", c_int),
                ("code_dim", c_int), ("tok_width", c_int), ("tok_depth", c_int), ("tok_dilation_rate", c_int),
                ("tok_joints", c_int), ("n_upsample", c_int), ("upsample_sizes", c_int * 8),
                ("focal_length", c_float), ("strict", c_int), ("concurrent", c_int), ("fp8", c_int)]


HEAD_TOKEN, HEAD_REGRESSION = 0, 1          # thmr_engine_create_head (THMR_HEAD_TOKEN / THMR_HEAD_REGRESSION)


class VitBlock(Structure):
    _fields_ = [(n, c_void_p) for n in ("ln1_g", "ln1_b", "qkv_w", "qkv_b", "proj_w", "proj_b", "ln2_g", "ln2_b",
                                        "fc1_w", "fc1_b", "fc2_w", "fc2_b")]


class VitBlockScales(Structure):
    _fields_ = [(n, c_void_p) for n in ("qkv_ws", "fc1_ws", "fc2_ws")]


class DecLayer(Structure):
    _fields_ = [(n, c_void_p) for n in ("ln0_g", "ln0_b", "sa_v_w", "sa_out_w", "sa_out_b", "ln1_g", "ln1_b",
                                        "ca_q_w", "ca_out_w", "ca_out_b", "ln2_g", "ln2_b", "ff1_w", "ff1_b",
                                        "ff2_w", "ff2_b")]


class MixerBlock(Structure):
    _fields_ = [(n, c_void_p) for n in ("ln1_g", "ln1_b", "tok1_w", "tok1_b", "tok2_w", "tok2_b", "ln2_g", "ln2_b",
                                        "ch1_w", "ch1_b", "ch2_w", "ch2_b")]


class Conv(Structure):
    _fields_ = [("w", c_void_p), ("b", c_void_p)]


class Weights(Structure):
    _fields_ = [("patch_w", c_void_p), ("patch_b", c_void_p), ("pos", c_void_p),
                ("blocks_host", POINTER(VitBlock)), ("last_g", c_void_p), ("last_b", c_void_p),
                ("token0", c_void_p), ("kv_w", c_void_p), ("dec_host", POINTER(DecLayer)),
                ("readout_w", c_void_p), ("readout_b", c_void_p),
                ("init_pose", c_void_p), ("init_betas", c_void_p), ("init_cam", c_void_p),
                ("mt_w", c_void_p), ("mt_b", c_void_p), ("mt_ln_g", c_void_p), ("mt_ln_b", c_void_p),
                ("mixer_host", POINTER(MixerBlock)),
                ("mn_w", c_void_p), ("mn_b", c_void_p), ("mn_ln_g", c_void_p), ("mn_ln_b", c_void_p),
                ("cls_w", c_void_p), ("cls_b", c_void_p),
                ("codebook_t", c_void_p), ("conv_in", Conv), ("conv_up", Conv * 8),
                ("res_conv1", Conv * 8), ("res_conv2", Conv * 8), ("conv_post", Conv), ("conv_out", Conv),
                ("block_scales_host", POINTER(VitBlockScales))]


class TokConv(Structure):
    _fields_ = [("w", c_void_p), ("b", c_void_p)]


class TokEncoderDesc(Structure):
    _fields_ = [("joints", c_int), ("in_dim", c_int), ("width", c_int), ("depth", c_int), ("dilation_rate", c_int),
                ("size_mul", c_int), ("code_dim", c_int), ("nb_code", c_int),
                ("conv_in", TokConv), ("conv_up", TokConv * 8), ("conv_down", TokConv),
                ("res_conv1", TokConv * 8), ("res_conv2", TokConv * 8), ("conv_out", TokConv), ("codebook", c_void_p)]


class PreprocCfg(Structure):
    _fields_ = [("image_size", c_int), ("bbox_w", c_int), ("bbox_h", c_int),
                ("mean", ctypes.c_double * 3), ("std", ctypes.c_double * 3)]


RENDER_MAX_LIGHTS = 16
RENDER_MAX_MESHES = 1024
LIGHT_DIRECTIONAL, LIGHT_POINT = 0, 1
BG_NONE, BG_HWC, BG_CHW_NORMALIZED = 0, 1, 2


class RenderLight(Structure):
    _fields_ = [("type", c_int), ("vec", c_float * 3), ("intensity", c_float)]


class RenderDesc(Structure):
    _fields_ = [("topology", c_void_p), ("n_meshes", c_int), ("n_images", c_int), ("mesh_image_host", POINTER(c_int32)),
                ("vertices", c_void_p), ("translations", c_void_p), ("rotation", c_float * 9),
                ("rotate_translation", c_int), ("width", c_int), ("height", c_int), ("focal", c_float),
                ("znear", c_float), ("base_color", c_float * 3), ("bg_color", c_float * 3), ("ambient", c_float),
                ("n_lights", c_int), ("lights", RenderLight * RENDER_MAX_LIGHTS), ("bg_layout", c_int),
                ("bg_image", c_void_p), ("mean", c_float * 3), ("std", c_float * 3),
                ("rgba", c_void_p), ("composite", c_void_p), ("face_id", c_void_p), ("depth", c_void_p)]


POSE_KEYPOINTS = 44
POSE_MAX_WIDTH = 11718


class PoseGridDesc(Structure):
    _fields_ = [("n", c_int), ("width", c_int), ("height", c_int), ("images", c_void_p), ("front", c_void_p),
                ("side", c_void_p), ("pred_keypoints", c_void_p), ("gt_keypoints", c_void_p), ("img_res", c_float),
                ("nrow", c_int), ("padding", c_int), ("out", c_void_p), ("out_stride_c", c_int64),
                ("out_stride_y", c_int64)]


class Outputs(Structure):
    _fields_ = [(n, c_void_p) for n in ("cls_logits_softmax", "pred_cam", "rotmats", "betas", "pred_cam_t",
                                        "focal_length", "pred_keypoints_3d", "pred_vertices", "pred_keypoints_2d",
                                        "vit_tokens", "token_out", "pose6d")]


def lib() -> ctypes.CDLL:
    global _lib
    if _lib is None:
        if not LIB_PATH.exists():
            raise ThmrError(
                f"{LIB_PATH} not found: build it with `python -m tokenhmr_b200._build` "
                "(the engine has no non-CUDA fallback)")
        _lib = ctypes.CDLL(str(LIB_PATH))
        _declare(_lib)
    return _lib


def check(status: int) -> None:
    if status != 0:
        msg = lib().thmr_last_error().decode(errors="replace")
        raise ThmrError(f"tokenhmr_b200 call failed ({status}): {msg}")


# name -> (restype, argtypes); tests/test_abi.py checks every symbol declared in the header is listed here
SIGNATURES = {
    "thmr_abi_version": (c_int, []),
    "thmr_last_error": (c_char_p, []),
    "thmr_check_device_flags": (c_int, []),
    "thmr_gemm_f16": (c_int, [c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_int, c_int,
                              c_void_p, c_int, c_void_p, c_int, c_int, c_void_p]),
    "thmr_conv1d_k3_f16": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_int, c_void_p, c_int, c_int,
                                   c_void_p, c_void_p, c_void_p]),
    "thmr_layernorm": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_float, c_int, c_void_p, c_void_p,
                               c_void_p]),
    "thmr_vit_attention": (c_int, [c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "thmr_vq_workspace_bytes": (c_size_t, [c_int64, c_int, c_int]),
    "thmr_vq_argmin": (c_int, [c_void_p, c_int64, c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "thmr_vq_dequantize": (c_int, [c_void_p, c_int64, c_void_p, c_int, c_void_p, c_void_p]),
    "thmr_vq_dequant_logits": (c_int, [c_void_p, c_int64, c_int, c_void_p, c_int, c_void_p, c_void_p]),
    "thmr_rot6d_to_rotmat": (c_int, [c_void_p, c_int64, c_void_p, c_void_p]),
    "thmr_regress_joints": (c_int, [c_void_p, c_int, c_void_p, c_int, c_int, c_void_p, c_void_p]),
    "thmr_eval_pose": (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p,
                               c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    "thmr_cam_crop_to_full": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_float, c_int, c_void_p, c_void_p]),
    "thmr_preprocess_workspace_bytes": (c_size_t, [c_int, c_int, c_int]),
    "thmr_preprocess_plan": (c_int, [c_void_p, c_int, POINTER(PreprocCfg), c_void_p, c_void_p, c_void_p, c_void_p]),
    "thmr_preprocess_boxes": (c_int, [c_void_p, c_int, c_int, c_int64, c_void_p, c_int, POINTER(PreprocCfg), c_void_p,
                                      c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "thmr_tok_encoder_create": (c_int, [POINTER(TokEncoderDesc), POINTER(c_void_p)]),
    "thmr_tok_encoder_destroy": (None, [c_void_p]),
    "thmr_tok_encoder_num_tokens": (c_int, [c_void_p]),
    "thmr_tok_encoder_workspace_bytes": (c_size_t, [c_void_p, c_int]),
    "thmr_tok_encode": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    "thmr_render_topology_create": (c_int, [c_void_p, c_int, c_int, POINTER(c_void_p)]),
    "thmr_render_topology_destroy": (None, [c_void_p]),
    "thmr_render_workspace_bytes": (c_size_t, [c_void_p, c_int, c_int, c_int, c_int]),
    "thmr_render_meshes": (c_int, [POINTER(RenderDesc), c_void_p, c_void_p]),
    "thmr_pose_grid_size": (c_int, [c_int, c_int, c_int, c_int, c_int, c_int, POINTER(c_int), POINTER(c_int)]),
    "thmr_pose_grid_workspace_bytes": (c_size_t, [c_int, c_int, c_int, c_int]),
    "thmr_pose_grid": (c_int, [POINTER(PoseGridDesc), c_void_p, c_void_p]),
    "thmr_smpl_create": (c_int, [POINTER(SmplDesc), POINTER(c_void_p)]),
    "thmr_smpl_destroy": (None, [c_void_p]),
    "thmr_smpl_workspace_bytes": (c_size_t, [c_void_p, c_int]),
    "thmr_lbs": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    "thmr_smpl_forward": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_float, c_float,
                                  c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "thmr_smpl_backward_workspace_bytes": (c_size_t, [c_void_p, c_int]),
    "thmr_smpl_backward": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p,
                                   c_void_p, c_void_p]),
    "thmr_lbs_backward": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p,
                                  c_void_p, c_void_p]),
    "thmr_smplify_workspace_bytes": (c_size_t, [c_void_p, c_int, c_int]),
    "thmr_smplify_inv": (c_int, [c_void_p, POINTER(SmplifyDesc), c_void_p, c_void_p]),
    "thmr_camera_tail": (c_int, [c_void_p, c_void_p, c_int, c_int, c_float, c_float, c_void_p, c_void_p, c_void_p,
                                 c_void_p]),
    "thmr_camera_tail_backward": (c_int, [c_void_p, c_void_p, c_int, c_int, c_float, c_float, c_void_p, c_void_p,
                                          c_void_p, c_void_p, c_void_p]),
    "thmr_tokenhmr_loss_workspace_bytes": (c_size_t, [c_int]),
    "thmr_tokenhmr_loss": (c_int, [POINTER(LossDesc), c_void_p, c_void_p]),
    "thmr_engine_create": (c_int, [POINTER(Config), POINTER(Weights), c_void_p, POINTER(c_void_p)]),
    "thmr_engine_create_head": (c_int, [POINTER(Config), c_int, POINTER(Weights), c_void_p, POINTER(c_void_p)]),
    "thmr_engine_destroy": (None, [c_void_p]),
    "thmr_engine_workspace_bytes": (c_size_t, [c_void_p, c_int]),
    "thmr_engine_forward": (c_int, [c_void_p, c_void_p, c_int, POINTER(Outputs), c_void_p, c_void_p]),
    "thmr_engine_num_launches": (c_int, [c_void_p]),
    "thmr_engine_num_steps": (c_int, [c_void_p]),
    "thmr_engine_step_info": (c_int, [c_void_p, c_int, POINTER(c_char_p), POINTER(ctypes.c_double),
                                      POINTER(ctypes.c_double)]),
    "thmr_engine_profile": (c_int, [c_void_p, c_void_p, c_int, POINTER(Outputs), c_void_p, c_void_p,
                                    POINTER(c_float), c_int]),
    "thmr_engine_vit_forward": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p]),
    "thmr_engine_forward_stamped": (c_int, [c_void_p, c_void_p, c_int, POINTER(Outputs), c_void_p, c_void_p]),
    "thmr_engine_read_stamps": (c_int, [c_void_p, POINTER(ctypes.c_uint64), c_int]),
    "thmr_comm_unique_id": (c_int, [c_void_p]),
    "thmr_comm_create": (c_int, [c_void_p, c_int, c_int, POINTER(c_void_p)]),
    "thmr_comm_destroy": (None, [c_void_p]),
    "thmr_comm_nranks": (c_int, [c_void_p]),
    "thmr_comm_rank": (c_int, [c_void_p]),
    "thmr_allgather_outputs": (c_int, [c_void_p, c_void_p, POINTER(Outputs), c_int, c_void_p]),
}


def _declare(L: ctypes.CDLL) -> None:
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(L, name)
        fn.restype = res
        fn.argtypes = args

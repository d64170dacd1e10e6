"""ctypes binding of libvfeat.so (the C ABI declared in include/vfeat.h).

There is no fallback: if the shared library is missing or a call fails, an exception is raised.
"""
from __future__ import annotations

import ctypes as C
import os
import threading

_HERE = os.path.dirname(os.path.abspath(__file__))
# VF_LIBVFEAT selects another build of the same library (A/B variants of one kernel, scripts/build_variants.sh)
LIB_PATH = os.environ.get("VF_LIBVFEAT") or os.path.join(_HERE, "libvfeat.so")

VF_OK = 0
VF_ACT_NONE, VF_ACT_QUICKGELU, VF_ACT_RELU, VF_ACT_SIGMOID, VF_ACT_TANH, VF_ACT_LEAKY = 0, 1, 2, 3, 4, 5
VF_ACT_GELU = 6
VF_FILTER_BILINEAR, VF_FILTER_BICUBIC = 2, 3
VF_POOL_GENERAL, VF_POOL_FAST, VF_POOL_SAME3 = 0, 1, 2


class VfError(RuntimeError):
    def __init__(self, code: int, text: str):
        super().__init__(f"libvfeat error {code}: {text}")
        self.code = code


class ClipLayerWeights(C.Structure):
    _fields_ = [(n, C.POINTER(C.c_float)) for n in (
        "ln_1_w", "ln_1_b", "in_proj_w", "in_proj_b", "out_proj_w", "out_proj_b",
        "ln_2_w", "ln_2_b", "c_fc_w", "c_fc_b", "c_proj_w", "c_proj_b")]


class ClipWeights(C.Structure):
    _fields_ = [(n, C.POINTER(C.c_float)) for n in (
        "conv1_w", "class_embedding", "positional_embedding",
        "ln_pre_w", "ln_pre_b", "ln_post_w", "ln_post_b", "proj")] + [("layers", ClipLayerWeights * 12)]


class ConvUnitW(C.Structure):
    _fields_ = [("w", C.POINTER(C.c_float)), ("bn_w", C.POINTER(C.c_float)), ("bn_b", C.POINTER(C.c_float)),
                ("bn_mean", C.POINTER(C.c_float)), ("bn_var", C.POINTER(C.c_float)),
                ("cout", C.c_int), ("cin", C.c_int), ("k", C.c_int)]


I3D_UNITS = 57


class I3DWeights(C.Structure):
    _fields_ = [("units", ConvUnitW * I3D_UNITS)]


class NamedTensor(C.Structure):
    _fields_ = [("name", C.c_char_p), ("data", C.POINTER(C.c_float)), ("numel", C.c_int64)]


def named_tensors(state_dict):
    """The floating-point tensors of ``state_dict`` (a mapping, or (name, tensor) pairs) as a ``NamedTensor`` array of
    fp32 host copies: returns (array, count, keep).  ``keep`` holds the copies and names the array points into; it must
    stay alive until the create call that reads the array returns."""
    import numpy as np
    import torch
    items = state_dict.items() if hasattr(state_dict, "items") else state_dict
    items = [(k, v) for k, v in items if torch.is_tensor(v) and v.dtype.is_floating_point]
    keep = []
    arr = (NamedTensor * max(len(items), 1))()
    for i, (k, v) in enumerate(items):
        a = np.ascontiguousarray(v.detach().to("cpu", torch.float32).numpy())
        nm = k.encode()
        keep.append((a, nm))
        arr[i].name = nm
        arr[i].data = a.ctypes.data_as(C.POINTER(C.c_float))
        arr[i].numel = a.size
    return arr, len(items), keep


_lock = threading.Lock()
_lib = None

# name -> (restype, argtypes); every symbol declared in include/vfeat.h
SIGNATURES = {
    "vf_version": (C.c_int, []),
    "vf_last_error": (C.c_char_p, []),
    "vf_sample_indices": (C.c_int, [C.c_char_p, C.c_int, C.c_int64, C.c_double, C.POINTER(C.c_int64), C.c_int64,
                                    C.POINTER(C.c_int64)]),
    "vf_shard_range": (C.c_int, [C.c_int64, C.c_int, C.c_int, C.POINTER(C.c_int64), C.POINTER(C.c_int64)]),
    "vf_resize_u8": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int,
                               C.c_void_p, C.c_void_p]),
    "vf_resize_geometry": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    "vf_clip_normalize_u8": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "vf_gemm_f16": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p,
                              C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]),
    "vf_gemm_f16_accumulate": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p,
                                         C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]),
    "vf_gemm_f16_split": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p,
                                    C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]),
    "vf_conv_gemm_f16": (C.c_int, [C.c_void_p, C.c_int, C.c_int64, C.c_void_p, C.c_int, C.c_int, C.c_int,
                                   C.POINTER(C.c_int), C.c_int, C.c_uint64, C.c_int, C.POINTER(C.c_int), C.c_void_p,
                                   C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]),
    "vf_gemm_profile": (C.c_int, [C.c_int]),
    "vf_gemm_profile_read": (C.c_int, [C.POINTER(C.c_double), C.POINTER(C.c_int64), C.POINTER(C.c_double)]),
    "vf_clip_create": (C.c_int, [C.POINTER(C.c_void_p), C.POINTER(ClipWeights), C.c_int, C.c_int]),
    "vf_clip_create_vit": (C.c_int, [C.POINTER(C.c_void_p), C.POINTER(ClipWeights), C.c_int, C.c_int, C.c_int]),
    "vf_clip_destroy": (C.c_int, [C.c_void_p]),
    "vf_clip_encode_f32": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    "vf_clip_encode_u8": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "vf_clip_encode_u8_host": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "vf_clip_encode_u8_host_dev": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p,
                                             C.c_void_p]),
    "vf_clip_encode_u8_host_async": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p,
                                               C.c_void_p, C.POINTER(C.c_int64)]),
    "vf_clip_wait": (C.c_int, [C.c_void_p, C.c_int64]),
    "vf_clip_block_attention": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p]),
    "vf_clip_debug_embed_f32": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    "vf_clip_debug_embed_u8": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "vf_clip_debug_blocks": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "vf_clip_debug_head": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    "vf_clip_launch_count": (C.c_int64, [C.c_void_p]),
    "vf_i3d_create": (C.c_int, [C.POINTER(C.c_void_p), C.POINTER(I3DWeights), C.c_int, C.c_int, C.c_int, C.c_int]),
    "vf_i3d_destroy": (C.c_int, [C.c_void_p]),
    "vf_i3d_forward_f32": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "vf_i3d_forward_u8": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "vf_i3d_forward_u8_strided": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int64, C.c_int, C.c_int, C.c_void_p,
                                            C.c_void_p]),
    "vf_i3d_forward_flow": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "vf_i3d_read_stage": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int64, C.POINTER(C.c_int), C.c_void_p]),
    "vf_i3d_launch_count": (C.c_int64, [C.c_void_p]),
    "vf_i3d_conv": (C.c_int, [C.c_void_p, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_uint64), C.c_void_p, C.c_void_p,
                              C.c_void_p]),
    "vf_i3d_debug_mixed": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "vf_raft_create": (C.c_int, [C.POINTER(C.c_void_p), C.POINTER(NamedTensor), C.c_int, C.c_int, C.c_int, C.c_int, C.c_int]),
    "vf_raft_destroy": (C.c_int, [C.c_void_p]),
    "vf_raft_flow": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                               C.c_void_p, C.c_void_p]),
    "vf_raft_padded_size": (C.c_int, [C.c_int, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    "vf_raft_debug_read": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int64, C.POINTER(C.c_int), C.c_void_p]),
    "vf_raft_launch_count": (C.c_int64, [C.c_void_p]),
    "vf_raft_conv": (C.c_int, [C.c_void_p, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_uint64), C.c_void_p, C.c_void_p,
                               C.c_void_p]),
    "vf_pwc_create": (C.c_int, [C.POINTER(C.c_void_p), C.POINTER(NamedTensor), C.c_int, C.c_int, C.c_int, C.c_int, C.c_int]),
    "vf_pwc_destroy": (C.c_int, [C.c_void_p]),
    "vf_pwc_flow": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p,
                              C.c_void_p]),
    "vf_pwc_debug_read": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int64, C.POINTER(C.c_int), C.c_void_p]),
    "vf_pwc_launch_count": (C.c_int64, [C.c_void_p]),
    "vf_pwc_conv": (C.c_int, [C.c_void_p, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_uint64), C.c_void_p, C.c_void_p,
                              C.c_void_p]),
    "vf_resnet_create": (C.c_int, [C.POINTER(C.c_void_p), C.POINTER(NamedTensor), C.c_int, C.c_int, C.c_int, C.c_int]),
    "vf_resnet_destroy": (C.c_int, [C.c_void_p]),
    "vf_resnet_forward_f32": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    "vf_resnet_forward_u8": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "vf_resnet_read_stage": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int64, C.POINTER(C.c_int), C.c_void_p]),
    "vf_resnet_launch_count": (C.c_int64, [C.c_void_p]),
    "vf_resnet_conv": (C.c_int, [C.c_void_p, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_uint64), C.c_void_p,
                                 C.c_void_p, C.c_void_p]),
    "vf_r21d_create": (C.c_int, [C.POINTER(C.c_void_p), C.POINTER(NamedTensor), C.c_int, C.c_int, C.c_int, C.c_int]),
    "vf_r21d_create2": (C.c_int, [C.POINTER(C.c_void_p), C.POINTER(NamedTensor), C.c_int, C.c_int, C.c_int, C.c_int,
                                  C.c_double]),
    "vf_r21d_destroy": (C.c_int, [C.c_void_p]),
    "vf_r21d_forward_f32": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "vf_r21d_forward_u8": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_int), C.c_int,
                                     C.c_int, C.c_void_p, C.c_void_p]),
    "vf_r21d_read_stage": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int64, C.POINTER(C.c_int), C.c_void_p]),
    "vf_r21d_launch_count": (C.c_int64, [C.c_void_p]),
    "vf_r21d_conv": (C.c_int, [C.c_void_p, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_uint64), C.c_void_p,
                               C.c_void_p, C.c_void_p]),
    "vf_s3d_create": (C.c_int, [C.POINTER(C.c_void_p), C.POINTER(NamedTensor), C.c_int, C.c_int, C.c_int, C.c_int]),
    "vf_s3d_destroy": (C.c_int, [C.c_void_p]),
    "vf_s3d_forward_f32": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "vf_s3d_forward_u8": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_int), C.c_int,
                                    C.c_int, C.c_void_p, C.c_void_p]),
    "vf_s3d_read_stage": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int64, C.POINTER(C.c_int), C.c_void_p]),
    "vf_s3d_launch_count": (C.c_int64, [C.c_void_p]),
    "vf_s3d_conv": (C.c_int, [C.c_void_p, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_uint64), C.c_void_p,
                              C.c_void_p, C.c_void_p]),
    "vf_s3d_debug_mixed": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "vf_debug_maxpool3d": (C.c_int, [C.c_void_p, C.POINTER(C.c_int), C.c_void_p, C.POINTER(C.c_int), C.c_int,
                                     C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int),
                                     C.c_void_p]),
    "vf_debug_i3d_head": (C.c_int, [C.c_void_p, C.POINTER(C.c_int), C.c_int, C.c_void_p, C.c_void_p]),
    "vf_clip_rn_create": (C.c_int, [C.POINTER(C.c_void_p), C.POINTER(NamedTensor), C.c_int, C.c_int, C.c_int]),
    "vf_clip_rn_destroy": (C.c_int, [C.c_void_p]),
    "vf_clip_rn_info": (C.c_int, [C.c_void_p, C.POINTER(C.c_int)]),
    "vf_clip_rn_encode_f32": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    "vf_clip_rn_encode_u8": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "vf_clip_rn_read_stage": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int64, C.POINTER(C.c_int), C.c_void_p]),
    "vf_clip_rn_launch_count": (C.c_int64, [C.c_void_p]),
    "vf_clip_rn_conv": (C.c_int, [C.c_void_p, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_uint64), C.c_void_p,
                                  C.c_void_p, C.c_void_p]),
    "vf_clip_rn_read_pairs": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int64, C.c_void_p]),
    "vf_clip_rn_debug_block": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                         C.c_void_p]),
    "vf_clip_rn_debug_attnpool": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    "vf_clip_rn_debug_attnpool_read": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int64, C.c_void_p]),
    "vf_debug_clip_rn_attention": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p,
                                             C.c_void_p]),
    "vf_swin3d_create": (C.c_int, [C.POINTER(C.c_void_p), C.POINTER(NamedTensor), C.c_int, C.c_int, C.c_int, C.c_int]),
    "vf_swin3d_destroy": (C.c_int, [C.c_void_p]),
    "vf_swin3d_info": (C.c_int, [C.c_void_p, C.POINTER(C.c_int)]),
    "vf_swin3d_forward_f32": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "vf_swin3d_forward_u8": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_int), C.c_int,
                                       C.c_int, C.c_void_p, C.c_void_p]),
    "vf_swin3d_read_stage": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int64, C.POINTER(C.c_int), C.c_void_p]),
    "vf_swin3d_attention": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                      C.c_int, C.c_void_p, C.c_void_p]),
    "vf_swin3d_launch_count": (C.c_int64, [C.c_void_p]),
    "vf_mvit_create": (C.c_int, [C.POINTER(C.c_void_p), C.POINTER(NamedTensor), C.c_int, C.c_int, C.c_int]),
    "vf_mvit_destroy": (C.c_int, [C.c_void_p]),
    "vf_mvit_info": (C.c_int, [C.c_void_p, C.POINTER(C.c_int)]),
    "vf_mvit_forward_f32": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "vf_mvit_forward_u8": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_int), C.c_int,
                                     C.c_int, C.c_void_p, C.c_void_p]),
    "vf_mvit_read_stage": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int64, C.POINTER(C.c_int), C.c_void_p]),
    "vf_mvit_attention": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                    C.c_int, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int), C.c_int, C.c_int,
                                    C.c_void_p, C.c_void_p]),
    "vf_mvit_head_pool": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                    C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "vf_mvit_skip_pool": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "vf_mvit_launch_count": (C.c_int64, [C.c_void_p]),
    "vf_clip_vitl_create": (C.c_int, [C.POINTER(C.c_void_p), C.POINTER(NamedTensor), C.c_int, C.c_int, C.c_int]),
    "vf_clip_vitl_destroy": (C.c_int, [C.c_void_p]),
    "vf_clip_vitl_info": (C.c_int, [C.c_void_p, C.POINTER(C.c_int)]),
    "vf_clip_vitl_encode_f32": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    "vf_clip_vitl_encode_u8": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "vf_clip_vitl_debug_embed_f32": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    "vf_clip_vitl_debug_embed_u8": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p,
                                              C.c_void_p]),
    "vf_clip_vitl_debug_blocks": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "vf_clip_vitl_debug_head": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    "vf_clip_vitl_attention": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "vf_clip_vitl_launch_count": (C.c_int64, [C.c_void_p]),
    "vf_vggish_create": (C.c_int, [C.POINTER(C.c_void_p), C.POINTER(NamedTensor), C.c_int, C.c_void_p, C.c_void_p,
                                   C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int]),
    "vf_vggish_destroy": (C.c_int, [C.c_void_p]),
    "vf_vggish_forward_pcm16": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_int, C.c_void_p, C.c_int64,
                                          C.POINTER(C.c_int64), C.c_void_p]),
    "vf_vggish_forward_logmel_f32": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    "vf_vggish_read_stage": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int64, C.POINTER(C.c_int), C.c_void_p]),
    "vf_vggish_launch_count": (C.c_int64, [C.c_void_p]),
    "vf_vggish_conv": (C.c_int, [C.c_void_p, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_uint64), C.c_void_p,
                                 C.c_void_p, C.c_void_p]),
    "vf_vggish_time_register": (C.c_int, [C.c_int, C.c_int64, C.c_int64, C.c_void_p]),
    "vf_clip_text_create": (C.c_int, [C.POINTER(C.c_void_p), C.POINTER(NamedTensor), C.c_int, C.c_int, C.c_int]),
    "vf_clip_text_destroy": (C.c_int, [C.c_void_p]),
    "vf_clip_text_info": (C.c_int, [C.c_void_p, C.POINTER(C.c_int)]),
    "vf_clip_text_encode": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    "vf_clip_text_blocks": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "vf_clip_text_attention": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "vf_l2_normalize_rows": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "vf_clip_text_launch_count": (C.c_int64, [C.c_void_p]),
    "vf_dinov2_create": (C.c_int, [C.POINTER(C.c_void_p), C.POINTER(NamedTensor), C.c_int, C.c_int, C.c_int]),
    "vf_dinov2_destroy": (C.c_int, [C.c_void_p]),
    "vf_dinov2_info": (C.c_int, [C.c_void_p, C.POINTER(C.c_int)]),
    "vf_dinov2_encode_f32": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    "vf_dinov2_encode_u8": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "vf_dinov2_debug_embed_f32": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    "vf_dinov2_debug_embed_u8": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "vf_dinov2_debug_blocks": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "vf_dinov2_debug_head": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    "vf_dinov2_swiglu": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "vf_dinov2_attention": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "vf_dinov2_launch_count": (C.c_int64, [C.c_void_p]),
    "vf_head_create": (C.c_int, [C.POINTER(C.c_void_p), C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int]),
    "vf_head_destroy": (C.c_int, [C.c_void_p]),
    "vf_head_info": (C.c_int, [C.c_void_p, C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    "vf_head_forward": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p,
                                  C.c_void_p, C.c_void_p, C.c_void_p]),
    "vf_clip_profile": (C.c_int, [C.c_void_p, C.c_int]),
    "vf_clip_profile_categories": (C.c_int, [C.c_void_p, C.POINTER(C.c_double)]),
    "vf_clip_profile_read": (C.c_int, [C.c_void_p, C.POINTER(C.c_double), C.POINTER(C.c_int64),
                                       C.POINTER(C.c_double)]),
}


def lib() -> C.CDLL:
    """Load libvfeat.so once; raises if it has not been built (``python -c 'import __graft_entry__ as g; g.build()'``)."""
    global _lib
    if _lib is None:
        with _lock:
            if _lib is None:
                if not os.path.exists(LIB_PATH):
                    raise FileNotFoundError(
                        f"{LIB_PATH} not found: build the CUDA extension first (__graft_entry__.build()). "
                        "There is no CPU fallback.")
                l = C.CDLL(LIB_PATH)
                for name, (res, args) in SIGNATURES.items():
                    fn = getattr(l, name)      # AttributeError if a declared symbol is not exported
                    fn.restype = res
                    fn.argtypes = args
                _lib = l
    return _lib


def check(status: int) -> None:
    if status != VF_OK:
        raise VfError(status, lib().vf_last_error().decode("utf-8", "replace"))


def read_conv(fn, handle, index: int, device):
    """Diagnostics shared by ResNetEngine.conv / R21DEngine.conv / S3DEngine.conv / ClipResNetEngine.conv: fn is
    vf_resnet_conv, vf_r21d_conv, vf_s3d_conv or vf_clip_rn_conv.  Returns dict
    n_out, ntaps, k_per_tap, shifts [(dt, dh, dw)] per tap, lo_mask, w (fp16 [n_out, 2 ntaps k_per_tap], W_hi | W_lo),
    scale, bias (fp32 [n_out]) as uploaded."""
    import torch
    geom = (C.c_int * 15)()
    mask = C.c_uint64()
    check(fn(handle, index, geom, C.byref(mask), None, None, None))
    n_out, ntaps, kpt = geom[0], geom[1], geom[2]
    w = torch.empty((n_out, 2 * ntaps * kpt), dtype=torch.float16, device=device)
    scale = torch.empty(n_out, dtype=torch.float32, device=device)
    bias = torch.empty(n_out, dtype=torch.float32, device=device)
    check(fn(handle, index, geom, C.byref(mask), w.data_ptr(), scale.data_ptr(), bias.data_ptr()))
    shifts = [tuple(geom[3 + 3 * j:6 + 3 * j]) for j in range(ntaps)]
    return dict(n_out=n_out, ntaps=ntaps, k_per_tap=kpt, shifts=shifts, lo_mask=mask.value, w=w, scale=scale, bias=bias)


# Mixed block index (0 .. 8) -> the side S of its S x S frames, and (cin, branch 0, 1, 2, 3 widths): I3D's mixed_3b ..
# mixed_5c and S3D's features.5 .. 15 are the same Inception widths
MIXED_SIDE = (28, 28, 14, 14, 14, 14, 14, 7, 7)
MIXED_WIDTHS = ((192, 64, 128, 32, 32), (256, 128, 192, 96, 64), (480, 192, 208, 48, 64), (512, 160, 224, 64, 64),
                (512, 128, 256, 64, 64), (512, 112, 288, 64, 64), (528, 256, 320, 128, 128), (832, 256, 320, 128, 128),
                (832, 384, 384, 128, 128))


def debug_mixed(fn, handle, block: int, x, device):
    """Diagnostics shared by I3DEngine.debug_mixed / S3DEngine.debug_mixed: fn is vf_i3d_debug_mixed or
    vf_s3d_debug_mixed.  x: fp16 pair volume (n, T + 2, S + 2, S + 2, 2 cin) on the device, zero border -> the block's
    concat pair volume (n, T + 2, S + 2, S + 2, 2 cout), border rows included."""
    import torch
    if not 0 <= block < len(MIXED_SIDE):
        raise ValueError(f"Mixed block {block} outside 0 .. {len(MIXED_SIDE) - 1}")
    S, cin, cout = MIXED_SIDE[block], MIXED_WIDTHS[block][0], sum(MIXED_WIDTHS[block][1:])
    # the entry copies n (T + 2) (S + 2)^2 rows of 2 cin halves from x: a wrong shape must not reach it
    if x.dtype != torch.float16 or x.dim() != 5 or tuple(x.shape[2:]) != (S + 2, S + 2, 2 * cin) or x.shape[1] < 3:
        raise ValueError(f"block {block} takes an fp16 pair volume (n, T + 2, {S + 2}, {S + 2}, {2 * cin}), T >= 1; "
                         f"got {x.dtype} {tuple(x.shape)}")
    if x.device != torch.device(device):
        raise ValueError(f"the volume is on {x.device}, the engine on {device}")
    x = x.contiguous()
    out = torch.empty(tuple(x.shape[:4]) + (2 * cout,), dtype=torch.float16, device=device)
    with torch.cuda.device(device):
        check(fn(handle, block, x.data_ptr(), x.shape[0], x.shape[1] - 2, out.data_ptr(),
                 torch.cuda.current_stream().cuda_stream))
    return out


def debug_maxpool3d(x, vol_in, vol_out, channels: int, k, s, p):
    """Diagnostics: vf_debug_maxpool3d.  x: fp16 pair rows [hi channels | lo channels] of the volume vol_in on the
    device; vol_in / vol_out: 10 ints (n, Tp, Hp, Wp, t0, t1, h0, h1, w0, w1); k, s, p: (t, h, w) window, stride and
    leading padding.  Returns (the pair volume (n, Tp, Hp, Wp, 2 channels) of vol_out, the VF_POOL_* kernel that ran)."""
    import torch
    assert x.dtype == torch.float16 and x.is_cuda
    assert x.numel() == vol_in[0] * vol_in[1] * vol_in[2] * vol_in[3] * 2 * channels, (x.shape, vol_in, channels)
    x = x.contiguous()
    out = torch.empty(tuple(vol_out[:4]) + (2 * channels,), dtype=torch.float16, device=x.device)
    path = C.c_int(-1)
    with torch.cuda.device(x.device):
        check(lib().vf_debug_maxpool3d(x.data_ptr(), (C.c_int * 10)(*vol_in), out.data_ptr(), (C.c_int * 10)(*vol_out),
                                       channels, (C.c_int * 3)(*k), (C.c_int * 3)(*s), (C.c_int * 3)(*p), C.byref(path),
                                       torch.cuda.current_stream().cuda_stream))
    return out, path.value


def debug_i3d_head(x, vol, channels: int):
    """Diagnostics: vf_debug_i3d_head, AvgPool3d((2,7,7), 1) and the mean over time of the pair volume x (rows of
    2 channels; vol: 10 ints as for debug_maxpool3d) -> (n, channels) fp32."""
    import torch
    assert x.dtype == torch.float16 and x.is_cuda
    assert x.numel() == vol[0] * vol[1] * vol[2] * vol[3] * 2 * channels, (x.shape, vol, channels)
    x = x.contiguous()
    out = torch.empty((vol[0], channels), dtype=torch.float32, device=x.device)
    with torch.cuda.device(x.device):
        check(lib().vf_debug_i3d_head(x.data_ptr(), (C.c_int * 10)(*vol), channels, out.data_ptr(),
                                      torch.cuda.current_stream().cuda_stream))
    return out


def debug_clip_rn_attention(kv, q):
    """Diagnostics: vf_debug_clip_rn_attention, the CLIP ResNet towers' attention kernel on fp32 K|V (n, T, 2E) and Q
    (n, E) on one device -> (n, 2E) fp16 pairs [hi E | lo E] of softmax((q / 8) . k) v per head of 64."""
    import torch
    if kv.dtype != torch.float32 or q.dtype != torch.float32 or kv.dim() != 3 or q.dim() != 2:
        raise ValueError(f"kv (n, T, 2E) and q (n, E) fp32; got {kv.dtype} {tuple(kv.shape)}, {q.dtype} {tuple(q.shape)}")
    n, T, E2 = kv.shape
    if E2 % 2 or tuple(q.shape) != (n, E2 // 2):
        raise ValueError(f"kv {tuple(kv.shape)} and q {tuple(q.shape)} do not agree on (n, E)")
    if not kv.is_cuda or q.device != kv.device:
        raise ValueError(f"kv on {kv.device}, q on {q.device}: both must be on one CUDA device")
    kv, q = kv.contiguous(), q.contiguous()
    out = torch.empty((n, E2), dtype=torch.float16, device=kv.device)
    with torch.cuda.device(kv.device):
        check(lib().vf_debug_clip_rn_attention(kv.data_ptr(), q.data_ptr(), n, T, E2 // 2, out.data_ptr(),
                                               torch.cuda.current_stream().cuda_stream))
    return out


def read_split_conv(fn, handle, index: int, device):
    """Diagnostics shared by I3DEngine.conv / RAFTEngine.conv: fn is vf_i3d_conv or vf_raft_conv.  Returns dict n_out,
    ntaps, k_per_tap, nsplit, shifts [(dt, dh, dw)] per tap, lo_mask, w (fp16 [n_out, nsplit ntaps k_per_tap]: W_hi,
    then W_lo when nsplit is 2), scale, bias (fp32 [n_out]) as uploaded."""
    import torch
    geom = (C.c_int * 196)()
    mask = C.c_uint64()
    check(fn(handle, index, geom, C.byref(mask), None, None, None))
    n_out, ntaps, kpt, nsplit = geom[0], geom[1], geom[2], geom[3]
    w = torch.empty((n_out, nsplit * ntaps * kpt), dtype=torch.float16, device=device)
    scale = torch.empty(n_out, dtype=torch.float32, device=device)
    bias = torch.empty(n_out, dtype=torch.float32, device=device)
    check(fn(handle, index, geom, C.byref(mask), w.data_ptr(), scale.data_ptr(), bias.data_ptr()))
    shifts = [tuple(geom[4 + 3 * j:7 + 3 * j]) for j in range(ntaps)]
    return dict(n_out=n_out, ntaps=ntaps, k_per_tap=kpt, nsplit=nsplit, shifts=shifts, lo_mask=mask.value, w=w,
                scale=scale, bias=bias)

"""``ExtractDINOv2`` -- DINOv2 frame features (``--feature_type dinov2_vit{s,b,l,g}14[_reg]``) on the H100 engine, with
ExtractResNet's surface.

Not in the reference's list of extractors: the self-supervised ViTs of ``torch.hub.load('facebookresearch/dinov2',
name)``.  The output key is the feature type; rows are float32 ``(n_frames, D)``, D = 384 / 768 / 1024 / 1536 for
S / B / L / g, the hub model's output (the class token after the final norm), plus 'fps' and 'timestamps_ms', saved
under ``{output_path}/{feature_type}``.  Every frame is read as base.FrameExtractor reads it; each chunk runs the fused
Resize(256, bicubic, Pillow-exact) + CenterCrop(224) + BGR->RGB + ToTensor + Normalize + ViT (vf_dinov2_encode_u8).
The hub checkpoints are backbones without a classifier, so ``--show_pred`` is refused (utils.sanity_check).
"""
from __future__ import annotations

from typing import Dict

import torch

from ..dinov2_engine import DINOv2Engine
from .base import FRAMES_PER_CALL, FrameExtractor, load_first

TYPES = ("dinov2_vits14", "dinov2_vitb14", "dinov2_vitl14", "dinov2_vitg14", "dinov2_vits14_reg", "dinov2_vitb14_reg",
         "dinov2_vitl14_reg", "dinov2_vitg14_reg")
_STATE_DICTS: Dict[str, Dict[str, torch.Tensor]] = {}


def checkpoint_name(feature_type: str) -> str:
    """The hub's file name: dinov2_vits14_pretrain.pth, dinov2_vits14_reg4_pretrain.pth, ..."""
    if feature_type not in TYPES:
        raise NotImplementedError(feature_type)
    if feature_type.endswith("_reg"):
        return feature_type[:-4] + "_reg4_pretrain.pth"
    return feature_type + "_pretrain.pth"


def load_dinov2_weights(feature_type: str) -> Dict[str, torch.Tensor]:
    """checkpoint_name(feature_type) in the first of base.checkpoint_dirs() that has it ($VF_CKPT_DIR, then
    $TORCH_HOME/hub/checkpoints, where torch.hub stores it); read from disk once per process."""
    if feature_type not in _STATE_DICTS:
        _STATE_DICTS[feature_type] = load_first(checkpoint_name(feature_type))
    return _STATE_DICTS[feature_type]


class ExtractDINOv2(FrameExtractor):

    def __init__(self, args):
        if args.feature_type not in TYPES:
            raise NotImplementedError(args.feature_type)
        super().__init__(args)
        self.central_crop_size = 224

    def encoder(self, device, preds):
        return self.per_device("engine", device, lambda idx: DINOv2Engine(
            load_dinov2_weights(self.feature_type), idx, max_frames=FRAMES_PER_CALL)).encode_u8

"""``ExtractSwin3D`` -- Swin3D clip features (``--feature_type swin3d_t|swin3d_s|swin3d_b``) on the H100 engine, with
ExtractS3D's surface.

Not in the reference's list of extractors: the Kinetics-400 video transformers torchvision ships as ``swin3d_t``,
``swin3d_s`` and ``swin3d_b`` (``SwinTransformer3d``), with their ``Swin3D_*_Weights.KINETICS400_V1`` transform.  The
output key is the feature type; rows are float32 ``(n_stacks, 768)`` for t / s and ``(n_stacks, 1024)`` for b,
``flatten(avgpool(norm(features(patch_embed(x)))))`` (torchvision's forward without ``head``), one row per full stack of
``form_slices(n_frames, stack_size, step_size)`` (defaults 32 / 32, torchvision's clip_len); a video shorter than one
stack gives ``np.array([])``.  Saved under ``{output_path}/{feature_type}``.

Frames are read and grouped into calls of CLIPS_PER_CALL stacks as base.StackExtractor does; each call runs the fused
BGR->RGB + Resize([256]) on uint8 of the CenterCrop(224) window + /255 + Normalize + patch rows + network
(vf_swin3d_forward_u8).
``--show_pred``: after every engine call the checkpoint's ``head`` runs on its device features (class_head.py); per
stack, the header ``{video_path} @ frames ({start}, {end})`` and the Kinetics top-5 are printed, as for S3D.
"""
from __future__ import annotations

from typing import Dict

import torch

from ..swin3d_engine import Swin3DEngine
from .base import StackExtractor, load_first

SWIN3D_KEYS = ("head.weight", "head.bias")        # torchvision SwinTransformer3d.head: Linear(C_out, 400)
# feature type -> the torchvision checkpoint's file pattern (KINETICS400_V1; swin3d_b's is the "_1k" file)
PATTERNS = {"swin3d_t": "swin3d_t-*.pth", "swin3d_s": "swin3d_s-*.pth", "swin3d_b": "swin3d_b_1k-*.pth"}
DEFAULT_SWIN3D_STEP_SIZE = 32
DEFAULT_SWIN3D_STACK_SIZE = 32
# stacks per engine call: stacks are independent, so this cannot change any feature
CLIPS_PER_CALL = 4
_STATE_DICTS: Dict[str, Dict[str, torch.Tensor]] = {}


def load_swin3d_weights(feature_type: str) -> Dict[str, torch.Tensor]:
    """The first checkpoint matching PATTERNS[feature_type] in base.checkpoint_dirs() ($VF_CKPT_DIR, then
    $TORCH_HOME/hub/checkpoints, where torchvision stores it); read from disk once per process."""
    if feature_type not in _STATE_DICTS:
        _STATE_DICTS[feature_type] = load_first(PATTERNS[feature_type])
    return _STATE_DICTS[feature_type]


class ExtractSwin3D(StackExtractor):
    feature_types = tuple(PATTERNS)
    head_keys = SWIN3D_KEYS
    default_stack = DEFAULT_SWIN3D_STACK_SIZE
    default_step = DEFAULT_SWIN3D_STEP_SIZE
    clips_per_call = CLIPS_PER_CALL

    def load_weights(self) -> Dict[str, torch.Tensor]:
        return load_swin3d_weights(self.feature_type)

    def new_engine(self, idx: int):
        # a workspace of about CLIPS_PER_CALL 32-frame stacks whatever the stack size; the engine chunks larger calls
        T = self.stack_size
        return Swin3DEngine(self.load_weights(), idx, max_clips=max(1, CLIPS_PER_CALL * 16 // ((T + 1) // 2)), max_T=T)

"""``ExtractS3D`` -- S3D clip features (``--feature_type s3d``) on the H100 engine, with ExtractR21D's surface.

Not in the reference's list of extractors: it is the Kinetics-400 clip feature upstream video_features added later as
``s3d``, here defined by torchvision's ``s3d()`` and its ``S3D_Weights.KINETICS400_V1`` transform.  Output key ``s3d``
is a float32 ``(n_stacks, 1024)`` array, ``avgpool(features(x)).mean((2, 3, 4))``, one row per full stack of
``form_slices(n_frames, stack_size, step_size)`` (defaults 64 / 64); a video shorter than one stack gives
``np.array([])``.  Saved under ``{output_path}/s3d``.  A stack needs at least 13 frames: fewer leave the (2,7,7)
average pool without a position.

Frames are read and grouped into calls of CLIPS_PER_CALL stacks as base.StackExtractor does; each call runs the fused
BGR->RGB + Resize((256, 256)) on uint8 of the CenterCrop(224) window + /255 + Normalize + S3D trunk (vf_s3d_forward_u8).
``--show_pred``: after every engine call the checkpoint's ``classifier.1`` runs on its device features
(class_head.py); per stack, the header ``{video_path} @ frames ({start}, {end})`` and the Kinetics top-5 are printed,
as for R(2+1)D.
"""
from __future__ import annotations

from typing import Dict

import torch

from ..s3d_engine import MIN_T, S3DEngine
from .base import StackExtractor, load_first

S3D_KEYS = ("classifier.1.weight", "classifier.1.bias")        # torchvision s3d: Conv3d(1024, 400, 1)
DEFAULT_S3D_STEP_SIZE = 64
DEFAULT_S3D_STACK_SIZE = 64
# stacks per engine call: stacks are independent, so this cannot change any feature
CLIPS_PER_CALL = 4
_STATE_DICT: Dict[str, torch.Tensor] = {}


def load_s3d_weights() -> Dict[str, torch.Tensor]:
    """The first ``s3d-*.pth`` found in base.checkpoint_dirs() ($VF_CKPT_DIR, then $TORCH_HOME/hub/checkpoints, where
    torchvision's ``S3D_Weights.KINETICS400_V1`` stores it); read from disk once per process."""
    if not _STATE_DICT:
        _STATE_DICT.update(load_first("s3d-*.pth"))
    return _STATE_DICT


class ExtractS3D(StackExtractor):
    feature_types = ("s3d",)
    head_keys = S3D_KEYS
    default_stack = DEFAULT_S3D_STACK_SIZE
    default_step = DEFAULT_S3D_STEP_SIZE
    clips_per_call = CLIPS_PER_CALL

    def check_sizes(self):
        if self.stack_size < MIN_T or self.step_size < 1:
            raise ValueError(f"stack_size {self.stack_size} must be >= {MIN_T} (the (2,7,7) average pool needs 13 "
                             f"frames) and step_size {self.step_size} >= 1")

    def load_weights(self) -> Dict[str, torch.Tensor]:
        return load_s3d_weights()

    def new_engine(self, idx: int) -> S3DEngine:
        # a workspace of about CLIPS_PER_CALL 64-frame stacks (about 1 GB each) whatever the stack size; the engine
        # chunks larger calls
        T = self.stack_size
        return S3DEngine(self.load_weights(), idx, max_clips=max(1, CLIPS_PER_CALL * 66 // (T + 2)), max_T=T)

"""``ExtractMViT`` -- MViT clip features (``--feature_type mvit_v1_b|mvit_v2_s``) on the H100 engine, with ExtractSwin3D's
surface.

Not in the reference's list of extractors: the Kinetics-400 Multiscale Vision Transformers torchvision ships as
``mvit_v1_b`` and ``mvit_v2_s``, with their ``MViT_*_Weights.KINETICS400_V1`` transform (Resize([256]), CenterCrop(224),
Normalize(0.45, 0.225)).  The output key is the feature type; rows are float32 ``(n_stacks, 768)``, ``norm(x)[:, 0]``
(the class token after the final norm: torchvision's forward without ``head``), one row per full stack of
``form_slices(n_frames, 16, step_size)``; a video shorter than one stack gives ``np.array([])``.  The stack size is 16
(the model's position tables fix T = 16; any other ``--stack_size`` is refused) and the step defaults to 16.  Saved under
``{output_path}/{feature_type}``.

Decoding, pinned staging, the asynchronous engine calls (vf_mvit_forward_u8), the one device->host copy per video and
``--show_pred`` (``head.1`` through class_head.py, Kinetics top-5 per stack) are base.StackExtractor's.
"""
from __future__ import annotations

from typing import Dict

import torch

from ..mvit_engine import MViTEngine
from .base import load_first
from .extract_swin3d import CLIPS_PER_CALL, ExtractSwin3D

MVIT_KEYS = ("head.1.weight", "head.1.bias")      # torchvision MViT.head: Sequential(Dropout, Linear(768, 400))
# feature type -> the torchvision checkpoint's file pattern (KINETICS400_V1)
PATTERNS = {"mvit_v1_b": "mvit_v1_b-*.pth", "mvit_v2_s": "mvit_v2_s-*.pth"}
MVIT_STACK_SIZE = 16
_STATE_DICTS: Dict[str, Dict[str, torch.Tensor]] = {}


def load_mvit_weights(feature_type: str) -> Dict[str, torch.Tensor]:
    """The first checkpoint matching PATTERNS[feature_type] in base.checkpoint_dirs() ($VF_CKPT_DIR, then
    $TORCH_HOME/hub/checkpoints, where torchvision stores it); read from disk once per process."""
    if feature_type not in _STATE_DICTS:
        _STATE_DICTS[feature_type] = load_first(PATTERNS[feature_type])
    return _STATE_DICTS[feature_type]


class ExtractMViT(ExtractSwin3D):
    feature_types = tuple(PATTERNS)
    head_keys = MVIT_KEYS
    default_stack = MVIT_STACK_SIZE
    default_step = MVIT_STACK_SIZE

    def __init__(self, args):
        super(ExtractMViT, self).__init__(args)
        if self.stack_size != MVIT_STACK_SIZE:
            raise ValueError(f"{self.feature_type} takes stacks of {MVIT_STACK_SIZE} frames: the model's position "
                             f"tables fix T = 16 (got --stack_size {self.stack_size})")

    def load_weights(self) -> Dict[str, torch.Tensor]:
        return load_mvit_weights(self.feature_type)

    def new_engine(self, idx: int) -> MViTEngine:
        return MViTEngine(self.load_weights(), idx, max_clips=CLIPS_PER_CALL)

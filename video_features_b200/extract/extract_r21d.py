"""``ExtractR21D`` -- drop-in for the reference's models/r21d/extract_r21d.py on the H100 engine.

Same constructor attributes / ``forward(indices)`` / ``extract(...)`` surface; output key ``r21d_rgb`` is a float64
``(n_stacks, 512)`` array (the reference builds it with ``.tolist()`` -> np.array), one row per full stack of
``form_slices(n_frames, stack_size, step_size)``; a video shorter than one stack gives ``np.array([])``.  No 'fps' /
'timestamps_ms' keys, as in the reference.  Saved under ``{output_path}/r21d_rgb``.

The reference decodes the whole video with torchvision's ``read_video`` (PyAV).  Here frames are read and grouped into
calls of CLIPS_PER_CALL stacks as base.StackExtractor does; each call runs the fused BGR->RGB + /255 + bilinear
Resize((128, 171)) of the CenterCrop(112) window + Normalize + R(2+1)D trunk (vf_r21d_forward_u8).
``--show_pred``: after every engine call the checkpoint's ``fc`` runs on its device features (class_head.py); per stack,
the header ``{video_path} @ frames ({start}, {end})`` and the Kinetics top-5 are printed (extract_r21d.py:113-121).

``model_name`` (``--model_name``; upstream video_features' choice for this extractor) picks the network, see MODELS:
torchvision's ``r2plus1d_18`` (the default) or one of the two R(2+1)D-34 models pre-trained on IG65M and fine-tuned on
Kinetics-400.  All three share the transform and the 400 Kinetics classes; features are 512-d under ``r21d_rgb``.
Weights are the first file matching the model's pattern in base.checkpoint_dirs() ($VF_CKPT_DIR, then
$TORCH_HOME/hub/checkpoints).
"""
from __future__ import annotations

from typing import Dict

import torch

from ..class_head import FC_KEYS, ClassHead
from ..r21d_engine import R21DEngine
from .base import StackExtractor, load_first

CENTRAL_CROP_MIN_SIDE_SIZE = 112
DEFAULT_R21D_STEP_SIZE = 16
DEFAULT_R21D_STACK_SIZE = 16
# stacks per engine call: stacks are independent, so this cannot change any feature
CLIPS_PER_CALL = 8
DEFAULT_MODEL = "r2plus1d_18_16_kinetics"
# model_name -> checkpoint pattern, BatchNorm eps, blocks per stage, default stack / step, classes of its fc.  The IG65M
# release files are (as recalled, unverified) r2plus1d_34_clip{8,32}_ft_kinetics_from_ig65m-<hash>.pth; the patterns
# match them loosely.
MODELS = {
    DEFAULT_MODEL: dict(pattern="r2plus1d_18-*.pth", bn_eps=1e-5, layers=(2, 2, 2, 2), stack=16, step=16, classes=400),
    "r2plus1d_34_32_ig65m_ft_kinetics": dict(pattern="r2plus1d_34_clip32*kinetics*.pth", bn_eps=1e-3,
                                             layers=(3, 4, 6, 3), stack=32, step=32, classes=400),
    "r2plus1d_34_8_ig65m_ft_kinetics": dict(pattern="r2plus1d_34_clip8*kinetics*.pth", bn_eps=1e-3,
                                            layers=(3, 4, 6, 3), stack=8, step=8, classes=400),
}
_STATE_DICT: Dict[str, torch.Tensor] = {}
_STATE_DICTS_34: Dict[str, Dict[str, torch.Tensor]] = {}


def load_r21d_weights() -> Dict[str, torch.Tensor]:
    """The first ``r2plus1d_18-*.pth`` found in base.checkpoint_dirs() ($VF_CKPT_DIR, then
    $TORCH_HOME/hub/checkpoints, where the reference's ``pretrained=True`` stores it); read from disk once per process."""
    if not _STATE_DICT:
        _STATE_DICT.update(load_first(MODELS[DEFAULT_MODEL]["pattern"]))
    return _STATE_DICT


def blocks_per_stage(state_dict: Dict[str, torch.Tensor]) -> tuple:
    """Blocks of layer1..4 in a VideoResNet state dict: the layerL.B.conv1.0.0.weight keys, as the engine counts them."""
    keys = {k[7:] if k.startswith("module.") else k for k in state_dict}
    out = []
    for L in range(1, 5):
        b = 0
        while f"layer{L}.{b}.conv1.0.0.weight" in keys:
            b += 1
        out.append(b)
    return tuple(out)


def load_r21d_34_weights(model_name: str) -> Dict[str, torch.Tensor]:
    """The first file matching MODELS[model_name]'s pattern in base.checkpoint_dirs(), read once per process.  A state
    dict without R(2+1)D-34's 3, 4, 6, 3 blocks is refused (the engine checks every tensor's size)."""
    if model_name not in _STATE_DICTS_34:
        m = MODELS[model_name]
        sd = load_first(m["pattern"])
        got = blocks_per_stage(sd)
        if got != m["layers"]:
            raise ValueError(f"{model_name}: the checkpoint has {got} blocks in layer1..4, not R(2+1)D-34's "
                             f"{m['layers']}")
        _STATE_DICTS_34[model_name] = sd
    return _STATE_DICTS_34[model_name]


class ExtractR21D(StackExtractor):
    feature_types = ("r21d_rgb",)
    head_keys = FC_KEYS
    clips_per_call = CLIPS_PER_CALL
    float64 = True

    def __init__(self, args):
        self.model_name = getattr(args, "model_name", None) or DEFAULT_MODEL
        if self.model_name not in MODELS:
            raise ValueError(f"unknown model_name {self.model_name!r}; choices: {', '.join(MODELS)}")
        self.model = MODELS[self.model_name]
        self.default_stack, self.default_step = self.model["stack"], self.model["step"]
        super().__init__(args)
        self.central_crop_min_side_size = CENTRAL_CROP_MIN_SIDE_SIZE

    def load_weights(self) -> Dict[str, torch.Tensor]:
        if self.model_name == DEFAULT_MODEL:
            return load_r21d_weights()
        return load_r21d_34_weights(self.model_name)

    def new_engine(self, idx: int) -> R21DEngine:
        # a workspace of about CLIPS_PER_CALL stacks of the model's default size (16, 32 or 8 frames) whatever the
        # stack size; the engine chunks larger calls
        T, base = self.stack_size, self.model["stack"] + 2
        return R21DEngine(self.load_weights(), idx, max_clips=max(1, CLIPS_PER_CALL * base // (T + 2)), max_T=T,
                          bn_eps=self.model["bn_eps"])

    def new_head(self, idx: int) -> ClassHead:
        head = ClassHead.from_state_dict(self.load_weights(), FC_KEYS, idx, f"{self.model_name} checkpoint")
        if head.n_classes != self.model["classes"]:     # the Kinetics-400 names are printed
            raise ValueError(f"--show_pred: the {self.model_name} checkpoint's fc has {head.n_classes} classes, "
                             f"not {self.model['classes']}")
        return head

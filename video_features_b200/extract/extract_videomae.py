"""``ExtractVideoMAE`` -- VideoMAE clip features (``--feature_type videomae_vits16|videomae_vitb16|videomae_vitl16``) on
the H100 engine, with ExtractMViT's surface.

The Kinetics-400 fine-tuned VideoMAE models in Hugging Face's layout (``MCG-NJU/videomae-{small,base,large}-finetuned-
kinetics``).  The output key is the feature type; rows are float32 ``(n_stacks, 384 | 768 | 1024)``, what
``VideoMAEForVideoClassification`` feeds its classifier: ``fc_norm(last_hidden_state.mean(1))``.  One row per full
stack of ``form_slices(n_frames, 16, step_size)``; a video shorter than one stack gives ``np.array([])``.  The stack
size is 16 (the sinusoid table is built for 16 frames; any other ``--stack_size`` is refused) and the step defaults to
16.  Saved under ``{output_path}/{feature_type}``.

Checkpoints are looked up, never downloaded: ``$VF_CKPT_DIR/videomae-{size}-finetuned-kinetics/``, then the Hugging Face
hub cache's snapshots (``$HF_HUB_CACHE``, else ``$HF_HOME/hub``, else ``~/.cache/huggingface/hub``).  A directory needs
``config.json`` and ``model.safetensors`` or ``pytorch_model.bin``; ``preprocessor_config.json`` gives the transform
when present, else ImageNet's mean / std (the original VideoMAE's; the processor class defaults to 0.5 / 0.5).

Decoding, pinned staging, the asynchronous engine calls (vf_videomae_forward_u8), the one device->host copy per video
and ``--show_pred`` (``classifier`` through class_head.py, Kinetics top-5 per stack, names from the config's
``id2label`` when it has them) are base.StackExtractor's.
"""
from __future__ import annotations

import glob
import json
import os
from typing import Dict, List, Optional, Tuple

import torch

from ..videomae_engine import FEATURE_TYPES, WIDTHS, T, Preset, VideoMAEConfig, VideoMAEEngine
from .base import StackExtractor

HEAD_KEYS = ("classifier.weight", "classifier.bias")
CLIPS_PER_CALL = 4
_CHECKPOINTS: Dict[str, Tuple[Dict[str, torch.Tensor], dict, Optional[dict]]] = {}


def hub_cache_dir() -> str:
    if os.environ.get("HF_HUB_CACHE"):
        return os.environ["HF_HUB_CACHE"]
    if os.environ.get("HF_HOME"):
        return os.path.join(os.environ["HF_HOME"], "hub")
    return os.path.join(os.path.expanduser("~"), ".cache", "huggingface", "hub")


def candidate_dirs(feature_type: str) -> List[str]:
    """The directories looked in, in order."""
    repo = FEATURE_TYPES[feature_type]
    dirs = []
    if os.environ.get("VF_CKPT_DIR"):
        dirs.append(os.path.join(os.environ["VF_CKPT_DIR"], repo))
    dirs += sorted(glob.glob(os.path.join(hub_cache_dir(), f"models--MCG-NJU--{repo}", "snapshots", "*")))
    return dirs


def find_checkpoint(feature_type: str) -> str:
    """The first candidate directory holding config.json and model.safetensors or pytorch_model.bin."""
    dirs = candidate_dirs(feature_type)
    for d in dirs:
        if os.path.isfile(os.path.join(d, "config.json")) and any(
                os.path.isfile(os.path.join(d, f)) for f in ("model.safetensors", "pytorch_model.bin")):
            return d
    raise FileNotFoundError(f"{feature_type}: no directory with config.json and model.safetensors (or "
                            f"pytorch_model.bin) among {dirs or '(none)'}; set VF_CKPT_DIR to a directory holding "
                            f"{FEATURE_TYPES[feature_type]}/, or HF_HUB_CACHE / HF_HOME")


def read_checkpoint(d: str) -> Tuple[Dict[str, torch.Tensor], dict, Optional[dict]]:
    """(state dict, config.json, preprocessor_config.json or None) of a checkpoint directory."""
    with open(os.path.join(d, "config.json")) as f:
        cfg = json.load(f)
    pre = None
    if os.path.isfile(os.path.join(d, "preprocessor_config.json")):
        with open(os.path.join(d, "preprocessor_config.json")) as f:
            pre = json.load(f)
    st = os.path.join(d, "model.safetensors")
    if os.path.isfile(st):
        from safetensors.torch import load_file
        sd = load_file(st)
    else:
        sd = torch.load(os.path.join(d, "pytorch_model.bin"), map_location="cpu")
    return sd, cfg, pre


def load_videomae(feature_type: str) -> Tuple[Dict[str, torch.Tensor], dict, Optional[dict]]:
    """The checkpoint of ``feature_type``, read from disk once per process."""
    if feature_type not in _CHECKPOINTS:
        sd, cfg, pre = read_checkpoint(find_checkpoint(feature_type))
        if cfg.get("hidden_size") != WIDTHS[feature_type]:
            raise ValueError(f"{feature_type}: the checkpoint's config.json has hidden_size {cfg.get('hidden_size')}, "
                             f"not {WIDTHS[feature_type]}")
        _CHECKPOINTS[feature_type] = (sd, cfg, pre)
    return _CHECKPOINTS[feature_type]


class ExtractVideoMAE(StackExtractor):
    feature_types = tuple(FEATURE_TYPES)
    head_keys = HEAD_KEYS
    default_stack = T
    default_step = T
    clips_per_call = CLIPS_PER_CALL

    def __init__(self, args):
        super(ExtractVideoMAE, self).__init__(args)
        if self.stack_size != T:
            raise ValueError(f"{self.feature_type} takes stacks of {T} frames: its sinusoid table is built for 16 "
                             f"frames (got --stack_size {self.stack_size})")

    def load_weights(self) -> Dict[str, torch.Tensor]:
        return load_videomae(self.feature_type)[0]

    def checkpoint(self):
        return load_videomae(self.feature_type)

    def class_names(self) -> Optional[List[str]]:
        if not hasattr(self, "_class_names"):     # read once: the --show_pred lines ask for every stack
            sd, cfg, _ = self.checkpoint()
            self._class_names = VideoMAEConfig.from_dict(cfg).class_names(sd[HEAD_KEYS[0]].shape[0])
        return self._class_names

    def new_engine(self, idx: int) -> VideoMAEEngine:
        sd, cfg, pre = self.checkpoint()
        return VideoMAEEngine(sd, cfg, Preset.from_dict(pre), idx, max_clips=CLIPS_PER_CALL)

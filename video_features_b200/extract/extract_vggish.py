"""``ExtractVGGish`` -- drop-in for the reference's models/vggish_torch/extract_vggish.py on the H100 engine, for
``.wav`` inputs.

Same constructor attributes / ``forward(indices)`` / ``extract(...)`` surface; output key ``feature_type`` is a float32
``(n_examples, 128)`` array (the reference returns ``tensor.cpu().numpy()``): raw embeddings after the final ReLU, no
PCA.  A 16-bit PCM WAV is read with the standard library's ``wave``; samples, mono mix, resampling to 16 kHz, log-mel
and the network run on the GPU (vggish_engine.VGGishEngine).  Audio shorter than 0.975 s has no example: like the
reference (whose ``x.view(0, -1)`` raises), that file is reported as failed and nothing is saved.  ``.mp4`` and other
containers are refused at construction: the reference extracts their audio track with ffmpeg, which this engine does
not ship.
"""
from __future__ import annotations

import pathlib
from typing import Dict

import numpy as np
import torch

from .. import audio
from ..vggish_engine import VGGishEngine
from .base import Extractor, load_first

_STATE_DICT: Dict[str, torch.Tensor] = {}


def load_vggish_weights() -> Dict[str, torch.Tensor]:
    """The first ``vggish-*.pth`` (torchvggish's hub file is vggish-10086976.pth) found in base.checkpoint_dirs(); read
    from disk once per process."""
    if not _STATE_DICT:
        _STATE_DICT.update(load_first("vggish-*.pth"))
    return _STATE_DICT


class ExtractVGGish(Extractor):
    video_args = False
    failed_at = "Extraction failed at: {}. Continuing extraction"

    def __init__(self, args):
        if args.feature_type != 'vggish_torch':
            raise NotImplementedError(f'{args.feature_type}: the TF1 VGGish (a TF .ckpt, PCA and 8-bit quantisation) '
                                      'is not built; use vggish_torch')
        super().__init__(args)
        others = [p for p in self.path_list if pathlib.Path(p).suffix != '.wav']
        if others:
            raise NotImplementedError(f'{self.feature_type}: only .wav input is read ({others[0]}); the reference '
                                      'extracts the audio of other files with ffmpeg, which this engine does not ship')
        self.output_direct = args.output_direct

    def extract_video(self, device, video_path):
        return self.extract(device, video_path)

    def extract(self, device: torch.device, video_path=None) -> Dict[str, np.ndarray]:
        samples, rate = audio.read_wav_pcm16(video_path)
        eng = self.per_device("engine", device, lambda idx: VGGishEngine(load_vggish_weights(), idx))
        feats = eng.forward_pcm16(samples, rate)
        if feats.shape[0] == 0:
            raise RuntimeError(f'{video_path}: {samples.shape[0]} samples at {rate} Hz make no 0.96 s example '
                               f'(at least {audio.MIN_SAMPLES} samples at 16 kHz are needed)')
        return {self.feature_type: feats.cpu().numpy()}

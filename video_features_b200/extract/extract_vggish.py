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

import glob
import os
import pathlib
from typing import Dict

import numpy as np
import torch
from tqdm import tqdm

from .. import audio
from ..utils import AsyncSink, action_on_extraction, already_extracted, form_list_from_user_input
from ..vggish_engine import VGGishEngine
from .extract_resnet import checkpoint_dirs

_STATE_DICT: Dict[str, torch.Tensor] = {}


def load_vggish_weights() -> Dict[str, torch.Tensor]:
    """The first ``vggish-*.pth`` (torchvggish's hub file is vggish-10086976.pth) found in
    extract_resnet.checkpoint_dirs(); read from disk once per process."""
    if not _STATE_DICT:
        dirs = checkpoint_dirs()
        for d in dirs:
            found = sorted(glob.glob(os.path.join(d, "vggish-*.pth")))
            if found:
                _STATE_DICT.update(torch.load(found[0], map_location="cpu"))
                break
        else:
            raise FileNotFoundError(f"vggish-*.pth not found in {dirs} (set VF_CKPT_DIR or TORCH_HOME)")
    return _STATE_DICT


class ExtractVGGish(torch.nn.Module):

    def __init__(self, args):
        super(ExtractVGGish, self).__init__()
        self.feature_type = args.feature_type
        if self.feature_type != 'vggish_torch':
            raise NotImplementedError(f'{self.feature_type}: the TF1 VGGish (a TF .ckpt, PCA and 8-bit quantisation) is '
                                      'not built; use vggish_torch')
        self.path_list = form_list_from_user_input(args)
        others = [p for p in self.path_list if pathlib.Path(p).suffix != '.wav']
        if others:
            raise NotImplementedError(f'{self.feature_type}: only .wav input is read ({others[0]}); the reference '
                                      'extracts the audio of other files with ffmpeg, which this engine does not ship')
        self.keep_tmp_files = args.keep_tmp_files
        self.on_extraction = args.on_extraction
        self.tmp_path = os.path.join(args.tmp_path, self.feature_type)
        self.output_path = os.path.join(args.output_path, self.feature_type)
        self.output_direct = args.output_direct
        self.progress = tqdm(total=len(self.path_list))
        self.keep_features = False
        self._engines: Dict[int, VGGishEngine] = {}

    def forward(self, indices: torch.LongTensor):
        device = indices.device
        if device.type != 'cuda':
            raise RuntimeError("the H100 engine has no CPU path: pass indices on a CUDA device")
        feats_list = []
        sink = AsyncSink() if os.environ.get("VF_ASYNC_SINK") == "1" else None     # opt-in extras, see ExtractCLIP.forward
        resume = os.environ.get("VF_RESUME") == "1"
        try:
            for idx in indices:
                path = self.path_list[idx]
                try:                                      # per-file catch-print-continue (extract_vggish.py forward)
                    if resume and already_extracted([self.feature_type], path, self.output_path, self.on_extraction,
                                                    self.output_direct):
                        self.progress.update()
                        continue
                    feats = self.extract(device, path)
                    if self.keep_features:
                        feats_list.append(feats)
                    if sink is not None:
                        sink.submit(feats, path, self.output_path, self.on_extraction, self.output_direct)
                    else:
                        action_on_extraction(feats, path, self.output_path, self.on_extraction,
                                             output_direct=self.output_direct)
                except KeyboardInterrupt:
                    raise
                except Exception as err:
                    print(err)
                    print(f'Extraction failed at: {path}. Continuing extraction')
                self.progress.update()
        finally:
            if sink is not None:
                sink.close()
        return feats_list

    def _engine(self, device: torch.device) -> VGGishEngine:
        idx = device.index if device.index is not None else torch.cuda.current_device()
        if idx not in self._engines:
            self._engines[idx] = VGGishEngine(load_vggish_weights(), idx)
        return self._engines[idx]

    def extract(self, device: torch.device, video_path=None) -> Dict[str, np.ndarray]:
        samples, rate = audio.read_wav_pcm16(video_path)
        feats = self._engine(device).forward_pcm16(samples, rate)
        if feats.shape[0] == 0:
            raise RuntimeError(f'{video_path}: {samples.shape[0]} samples at {rate} Hz make no 0.96 s example '
                               f'(at least {audio.MIN_SAMPLES} samples at 16 kHz are needed)')
        return {self.feature_type: feats.cpu().numpy()}

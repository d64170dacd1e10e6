"""``ExtractDINOv2`` -- DINOv2 frame features (``--feature_type dinov2_vit{s,b,l,g}14[_reg]``) on the H100 engine, with
ExtractResNet's surface.

Not in the reference's list of extractors: the self-supervised ViTs of ``torch.hub.load('facebookresearch/dinov2',
name)``.  The output key is the feature type; rows are float32 ``(n_frames, D)``, D = 384 / 768 / 1024 / 1536 for
S / B / L / g, the hub model's output (the class token after the final norm), plus 'fps' and 'timestamps_ms', saved
under ``{output_path}/{feature_type}``.  Every frame is read sequentially with OpenCV (a failed FIRST read is skipped,
as ExtractResNet does).  Underneath, per chunk of FRAMES_PER_CALL frames:
  decoder frames (uint8 BGR) -> pinned host buffer -> device
  -> fused Resize(256, bicubic, Pillow-exact) + CenterCrop(224) + BGR->RGB + ToTensor + Normalize + ViT
     (vf_dinov2_encode_u8)
The engine call is asynchronous, so decoding the next chunk overlaps the network on the current one; the features stay
on the device until the video is finished (one device->host copy per video).  The hub checkpoints are backbones
without a classifier, so ``--show_pred`` is refused (utils.sanity_check).
"""
from __future__ import annotations

import glob
import os
from typing import Dict, List

import numpy as np
import torch
from tqdm import tqdm

from ..dinov2_engine import DINOv2Engine
from ..utils import AsyncSink, action_on_extraction, already_extracted, form_list_from_user_input
from .extract_resnet import checkpoint_dirs

TYPES = ("dinov2_vits14", "dinov2_vitb14", "dinov2_vitl14", "dinov2_vitg14", "dinov2_vits14_reg", "dinov2_vitb14_reg",
         "dinov2_vitl14_reg", "dinov2_vitg14_reg")
# frames per engine call: frames are independent, so this cannot change any feature
FRAMES_PER_CALL = 64
_STATE_DICTS: Dict[str, Dict[str, torch.Tensor]] = {}


def checkpoint_name(feature_type: str) -> str:
    """The hub's file name: dinov2_vits14_pretrain.pth, dinov2_vits14_reg4_pretrain.pth, ..."""
    if feature_type not in TYPES:
        raise NotImplementedError(feature_type)
    if feature_type.endswith("_reg"):
        return feature_type[:-4] + "_reg4_pretrain.pth"
    return feature_type + "_pretrain.pth"


def load_dinov2_weights(feature_type: str) -> Dict[str, torch.Tensor]:
    """The first checkpoint_name(feature_type) found in checkpoint_dirs() ($VF_CKPT_DIR, then
    $TORCH_HOME/hub/checkpoints, where torch.hub stores it); read from disk once per process."""
    if feature_type not in _STATE_DICTS:
        dirs, name = checkpoint_dirs(), checkpoint_name(feature_type)
        for d in dirs:
            path = os.path.join(d, name)
            if os.path.exists(path):
                _STATE_DICTS[feature_type] = torch.load(path, map_location="cpu")
                break
        else:
            raise FileNotFoundError(f"{name} not found in {dirs} (set VF_CKPT_DIR or TORCH_HOME)")
    return _STATE_DICTS[feature_type]


class ExtractDINOv2(torch.nn.Module):

    def __init__(self, args):
        super(ExtractDINOv2, self).__init__()
        self.feature_type = args.feature_type
        if self.feature_type not in TYPES:
            raise NotImplementedError(self.feature_type)
        self.path_list = form_list_from_user_input(args)
        self.central_crop_size = 224
        self.extraction_fps = args.extraction_fps
        if self.extraction_fps is not None:
            raise NotImplementedError("extraction_fps re-encodes with ffmpeg (outside the rebuilt path, SURVEY.md §2)")
        self.show_pred = args.show_pred
        self.keep_tmp_files = args.keep_tmp_files
        self.on_extraction = args.on_extraction
        self.tmp_path = os.path.join(args.tmp_path, self.feature_type)
        self.output_path = os.path.join(args.output_path, self.feature_type)
        self.progress = tqdm(total=len(self.path_list))
        self.keep_features = False
        self._engines: Dict[int, DINOv2Engine] = {}
        self._pinned: Dict[tuple, List[torch.Tensor]] = {}

    def forward(self, indices: torch.LongTensor):
        device = indices.device
        if device.type != 'cuda':
            raise RuntimeError("the H100 engine has no CPU path: pass indices on a CUDA device")
        feats_list = []
        sink = AsyncSink() if os.environ.get("VF_ASYNC_SINK") == "1" else None     # opt-in extras, see ExtractCLIP.forward
        resume = os.environ.get("VF_RESUME") == "1"
        try:
            for idx in indices:
                video = self.path_list[idx]
                try:                                      # per-video catch-print-continue
                    if resume and already_extracted([self.feature_type], video, self.output_path, self.on_extraction):
                        self.progress.update()
                        continue
                    feats = self.extract(device, None, None, video)
                    if self.keep_features:
                        feats_list.append(feats)
                    if sink is not None:
                        sink.submit(feats, video, self.output_path, self.on_extraction)
                    else:
                        action_on_extraction(feats, video, self.output_path, self.on_extraction)
                except KeyboardInterrupt:
                    raise
                except Exception as err:
                    print(err)
                    print(f'Extraction failed at: {video} with error (↑). Continuing extraction')
                self.progress.update()
        finally:
            if sink is not None:
                sink.close()
        return feats_list

    def _engine(self, device: torch.device) -> DINOv2Engine:
        idx = device.index if device.index is not None else torch.cuda.current_device()
        if idx not in self._engines:
            self._engines[idx] = DINOv2Engine(load_dinov2_weights(self.feature_type), idx, max_frames=FRAMES_PER_CALL)
        return self._engines[idx]

    def _staging(self, shape) -> List[torch.Tensor]:
        """Two pinned (FRAMES_PER_CALL, H, W, 3) uint8 staging buffers per frame size: one fills while the other's
        host->device copy runs."""
        if shape not in self._pinned:
            self._pinned = {shape: [torch.empty((FRAMES_PER_CALL,) + shape, dtype=torch.uint8).pin_memory()
                                    for _ in range(2)]}
        return self._pinned[shape]

    def extract(self, device: torch.device, model=None, classifier=None, video_path=None) -> Dict[str, np.ndarray]:
        import cv2
        eng = self._engine(device)
        cap = cv2.VideoCapture(video_path)
        fps = cap.get(cv2.CAP_PROP_FPS)
        timestamps_ms, outs = [], []
        bufs, copied = None, [None, None]           # copied[s]: event after the last host->device copy out of buffer s
        slot, k = 0, 0

        def submit(s: int, n: int):
            with torch.cuda.device(device):
                x = bufs[s][:n].to(device, non_blocking=True)
                copied[s] = torch.cuda.Event()
                copied[s].record()
                outs.append(eng.encode_u8(x))

        first_frame = True
        while cap.isOpened():
            frame_exists, bgr = cap.read()
            if first_frame:
                first_frame = False
                if frame_exists is False:
                    continue
            if not frame_exists:
                if k:
                    submit(slot, k)
                cap.release()
                break
            timestamps_ms.append(cap.get(cv2.CAP_PROP_POS_MSEC))
            if bufs is None:
                bufs = self._staging(tuple(bgr.shape))
            if k == 0 and copied[slot] is not None:
                copied[slot].synchronize()          # the previous copy out of this buffer has finished
            bufs[slot][k].copy_(torch.from_numpy(bgr))
            k += 1
            if k == FRAMES_PER_CALL:
                submit(slot, k)
                slot, k = slot ^ 1, 0
        # one device->host copy per video
        feats = torch.cat(outs).cpu().numpy() if outs else np.array([])
        return {self.feature_type: feats, 'fps': np.array(fps), 'timestamps_ms': np.array(timestamps_ms)}

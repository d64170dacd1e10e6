"""``ExtractResNet`` -- drop-in for the reference's models/resnet/extract_resnet.py on the H100 engine.

Same constructor attributes / ``forward(indices)`` / ``extract(...)`` surface; output key ``feature_type`` is a float64
``(n_frames, D)`` array (D = 512 for resnet18/34, 2048 for resnet50/101/152; the reference builds it with ``.tolist()``)
plus 'fps' and 'timestamps_ms', saved under ``{output_path}/{feature_type}``.  Every frame is read sequentially with
OpenCV (a failed FIRST read is skipped, extract_resnet.py:130-137).  Underneath, per chunk of FRAMES_PER_CALL frames:
  decoder frames (uint8 BGR) -> pinned host buffer -> GPU Pillow-exact bilinear resize to short side 256
  -> fused BGR->RGB swap + CenterCrop(224) + ToTensor + Normalize + ResNet trunk (vf_resnet_forward_u8)
The engine call is asynchronous, so decoding the next chunk overlaps the network on the current one; the features stay
on the device until the video is finished (one device->host copy per video).
``--show_pred``: after every engine call the checkpoint's ``fc`` runs on its device features (class_head.py) and the
ImageNet top-5 of each frame is printed in frame order, as the reference prints per batch (extract_resnet.py:105-114).
"""
from __future__ import annotations

import glob
import os
from typing import Dict, List

import numpy as np
import torch
from tqdm import tqdm

from .. import ops
from .._lib import VF_FILTER_BILINEAR
from ..class_head import FC_KEYS, ClassHead, TopKQueue
from ..resnet_engine import DEPTHS, ResNetEngine
from ..utils import AsyncSink, action_on_extraction, already_extracted, form_list_from_user_input, print_top_predictions

RESIZE_SIZE = 256
CENTER_CROP_SIZE = 224
# frames per engine call: frames are independent, so this cannot change any feature (the reference's --batch_size
# only groups frames for its own model calls).  Chosen by a sweep on one H100 (scripts/resnet_time.py, README).
FRAMES_PER_CALL = 64
_STATE_DICTS: Dict[int, Dict[str, torch.Tensor]] = {}


def checkpoint_dirs() -> List[str]:
    """Where the ImageNet weights are looked up, in order: $VF_CKPT_DIR, then torch hub's checkpoint cache
    ($TORCH_HOME/hub/checkpoints, default ~/.cache/torch/hub/checkpoints), where the reference's
    ``pretrained=True`` stores them."""
    dirs = [os.environ.get("VF_CKPT_DIR"), os.path.join(torch.hub.get_dir(), "checkpoints")]
    return [d for d in dirs if d]


def load_resnet_weights(depth: int) -> Dict[str, torch.Tensor]:
    """The first ``resnet{depth}-*.pth`` found in checkpoint_dirs(); read from disk once per process."""
    if depth not in _STATE_DICTS:
        dirs = checkpoint_dirs()
        for d in dirs:
            found = sorted(glob.glob(os.path.join(d, f"resnet{depth}-*.pth")))
            if found:
                _STATE_DICTS[depth] = torch.load(found[0], map_location="cpu")
                break
        else:
            raise FileNotFoundError(f"resnet{depth}-*.pth not found in {dirs} (set VF_CKPT_DIR or TORCH_HOME)")
    return _STATE_DICTS[depth]


class ExtractResNet(torch.nn.Module):

    def __init__(self, args):
        super(ExtractResNet, self).__init__()
        self.feature_type = args.feature_type
        self.path_list = form_list_from_user_input(args)
        self.batch_size = args.batch_size
        self.central_crop_size = CENTER_CROP_SIZE
        self.extraction_fps = args.extraction_fps
        self.show_pred = args.show_pred
        self.keep_tmp_files = args.keep_tmp_files
        self.on_extraction = args.on_extraction
        self.tmp_path = os.path.join(args.tmp_path, self.feature_type)
        self.output_path = os.path.join(args.output_path, self.feature_type)
        depth = int(self.feature_type[len("resnet"):]) if self.feature_type.startswith("resnet") else None
        if depth not in DEPTHS:
            raise NotImplementedError(self.feature_type)
        if self.extraction_fps is not None:
            raise NotImplementedError("extraction_fps re-encodes with ffmpeg (outside the rebuilt path, SURVEY.md §2)")
        self.depth = depth
        self.progress = tqdm(total=len(self.path_list))
        self.keep_features = False
        self._engines: Dict[int, ResNetEngine] = {}
        self._heads: Dict[int, ClassHead] = {}
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
                try:                                      # per-video catch-print-continue (extract_resnet.py:74-84)
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

    def _engine(self, device: torch.device) -> ResNetEngine:
        idx = device.index if device.index is not None else torch.cuda.current_device()
        if idx not in self._engines:
            self._engines[idx] = ResNetEngine(load_resnet_weights(self.depth), self.depth, idx, max_frames=FRAMES_PER_CALL)
        return self._engines[idx]

    def _head(self, device: torch.device) -> ClassHead:
        idx = device.index if device.index is not None else torch.cuda.current_device()
        if idx not in self._heads:
            self._heads[idx] = ClassHead.from_state_dict(load_resnet_weights(self.depth), FC_KEYS, idx,
                                                         f"resnet{self.depth} checkpoint")
        return self._heads[idx]

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
        head = self._head(device) if self.show_pred else None
        preds = TopKQueue() if self.show_pred else None
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
                h, w = x.shape[1:3]
                oh, ow = ops.resize_geometry(h, w, RESIZE_SIZE, True)
                if (oh, ow) != (h, w):
                    x = torch.ops.vfeat.resize_u8(x, oh, ow, VF_FILTER_BILINEAR)      # ToPILImage -> Resize(256)
                outs.append(eng.forward_u8(x))
                if head is not None:                # only the top-5 crosses to the host, printed one call later
                    preds.submit([(head, outs[-1])], lambda tops: print_top_predictions(*tops[0], 'imagenet'))

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
        if preds is not None:
            preds.flush()
        # one device->host copy per video; float64 like the reference's `.tolist()` -> np.array
        feats = torch.cat(outs).cpu().numpy().astype(np.float64) if outs else np.array([])
        return {self.feature_type: feats, 'fps': np.array(fps), 'timestamps_ms': np.array(timestamps_ms)}

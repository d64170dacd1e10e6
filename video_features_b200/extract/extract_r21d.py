"""``ExtractR21D`` -- drop-in for the reference's models/r21d/extract_r21d.py on the H100 engine.

Same constructor attributes / ``forward(indices)`` / ``extract(...)`` surface; output key ``r21d_rgb`` is a float64
``(n_stacks, 512)`` array (the reference builds it with ``.tolist()`` -> np.array), one row per full stack of
``form_slices(n_frames, stack_size, step_size)``; a video shorter than one stack gives ``np.array([])``.  No 'fps' /
'timestamps_ms' keys, as in the reference.  Saved under ``{output_path}/r21d_rgb``.

The reference decodes the whole video with torchvision's ``read_video`` (PyAV).  Here frames are read sequentially with
OpenCV and swapped BGR->RGB inside the engine; only frames some stack needs are kept, so host and device memory do not
grow with the video.  Per call of CLIPS_PER_CALL stacks:
  decoder frames (uint8 BGR, the stacks' frames once each) -> pinned host buffer -> device
  -> fused BGR->RGB + /255 + bilinear Resize((128, 171)) of the CenterCrop(112) window + Normalize + R(2+1)D trunk
     (vf_r21d_forward_u8)
The engine call is asynchronous, so decoding the next stacks overlaps the network on the current ones; the features
stay on the device until the video is finished (one device->host copy per video).
``--show_pred``: after every engine call the checkpoint's ``fc`` runs on its device features (class_head.py); per stack,
the header ``{video_path} @ frames ({start}, {end})`` and the Kinetics top-5 are printed (extract_r21d.py:113-121).
"""
from __future__ import annotations

import glob
import os
from collections import deque
from typing import Dict, List

import numpy as np
import torch
from tqdm import tqdm

from ..class_head import FC_KEYS, ClassHead, TopKQueue
from ..r21d_engine import R21DEngine
from ..utils import AsyncSink, action_on_extraction, already_extracted, form_list_from_user_input, print_top_predictions
from .extract_resnet import checkpoint_dirs

CENTRAL_CROP_MIN_SIDE_SIZE = 112
DEFAULT_R21D_STEP_SIZE = 16
DEFAULT_R21D_STACK_SIZE = 16
# stacks per engine call: stacks are independent, so this cannot change any feature
CLIPS_PER_CALL = 8
_STATE_DICT: Dict[str, torch.Tensor] = {}


def load_r21d_weights() -> Dict[str, torch.Tensor]:
    """The first ``r2plus1d_18-*.pth`` found in checkpoint_dirs() ($VF_CKPT_DIR, then $TORCH_HOME/hub/checkpoints,
    where the reference's ``pretrained=True`` stores it); read from disk once per process."""
    if not _STATE_DICT:
        dirs = checkpoint_dirs()
        for d in dirs:
            found = sorted(glob.glob(os.path.join(d, "r2plus1d_18-*.pth")))
            if found:
                _STATE_DICT.update(torch.load(found[0], map_location="cpu"))
                break
        else:
            raise FileNotFoundError(f"r2plus1d_18-*.pth not found in {dirs} (set VF_CKPT_DIR or TORCH_HOME)")
    return _STATE_DICT


class ExtractR21D(torch.nn.Module):

    def __init__(self, args):
        super(ExtractR21D, self).__init__()
        self.feature_type = args.feature_type
        if self.feature_type != "r21d_rgb":
            raise NotImplementedError(self.feature_type)
        self.path_list = form_list_from_user_input(args)
        self.central_crop_min_side_size = CENTRAL_CROP_MIN_SIDE_SIZE
        self.extraction_fps = args.extraction_fps
        self.step_size = args.step_size
        self.stack_size = args.stack_size
        if self.step_size is None:
            self.step_size = DEFAULT_R21D_STEP_SIZE
        if self.stack_size is None:
            self.stack_size = DEFAULT_R21D_STACK_SIZE
        if self.extraction_fps is not None:
            raise NotImplementedError("extraction_fps re-encodes with ffmpeg (outside the rebuilt path, SURVEY.md §2)")
        if self.stack_size < 1 or self.step_size < 1:
            raise ValueError(f"stack_size {self.stack_size} and step_size {self.step_size} must be >= 1")
        # the reference's Compose(ToFloatTensorInZeroOne, Resize, Normalize, CenterCrop) runs fused inside the engine
        self.transforms = None
        self.show_pred = args.show_pred
        self.keep_tmp_files = args.keep_tmp_files
        self.on_extraction = args.on_extraction
        self.tmp_path = os.path.join(args.tmp_path, self.feature_type)
        self.output_path = os.path.join(args.output_path, self.feature_type)
        self.progress = tqdm(total=len(self.path_list))
        self.keep_features = False
        self._engines: Dict[int, R21DEngine] = {}
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
                try:                                      # per-video catch-print-continue (extract_r21d.py)
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

    def _engine(self, device: torch.device) -> R21DEngine:
        idx = device.index if device.index is not None else torch.cuda.current_device()
        if idx not in self._engines:
            # a workspace of about CLIPS_PER_CALL 16-frame stacks whatever the stack size; the engine chunks larger calls
            T = self.stack_size
            self._engines[idx] = R21DEngine(load_r21d_weights(), idx, max_clips=max(1, CLIPS_PER_CALL * 18 // (T + 2)),
                                            max_T=T)
        return self._engines[idx]

    def _head(self, device: torch.device) -> ClassHead:
        idx = device.index if device.index is not None else torch.cuda.current_device()
        if idx not in self._heads:
            self._heads[idx] = ClassHead.from_state_dict(load_r21d_weights(), FC_KEYS, idx, "r2plus1d_18 checkpoint")
        return self._heads[idx]

    def _staging(self, shape) -> List[torch.Tensor]:
        """Two pinned uint8 staging buffers per frame size, each large enough for the frames of CLIPS_PER_CALL stacks:
        one fills while the other's host->device copy runs."""
        if shape not in self._pinned:
            T, step = self.stack_size, self.step_size
            cap = min(CLIPS_PER_CALL * T, (CLIPS_PER_CALL - 1) * step + T)
            self._pinned = {shape: [torch.empty((cap,) + shape, dtype=torch.uint8).pin_memory() for _ in range(2)]}
        return self._pinned[shape]

    def extract(self, device: torch.device, model=None, classifier=None, video_path=None) -> Dict[str, np.ndarray]:
        import cv2
        eng = self._engine(device)
        head = self._head(device) if self.show_pred else None
        preds = TopKQueue() if self.show_pred else None
        T, step = self.stack_size, self.step_size
        cap = cv2.VideoCapture(video_path)
        if not cap.isOpened():             # the reference's read_video raises on an unreadable file
            raise RuntimeError(f"cannot open {video_path} for decoding")
        outs = []
        kept = deque()                     # (frame index, BGR frame) of frames a pending stack needs
        bufs, copied = None, [None, None]  # copied[s]: event after the last host->device copy out of buffer s
        state = {"slot": 0, "next": 0}     # next: first stack not yet submitted

        def submit(last: int):
            """Stacks next..last (all complete) -> one engine call."""
            first, s = state["next"], state["slot"]
            if copied[s] is not None:
                copied[s].synchronize()    # the previous copy out of this buffer has finished
            idx = sorted({f for i in range(first, last + 1) for f in range(i * step, i * step + T)})
            pos = {f: j for j, f in enumerate(idx)}
            by_index = dict(kept)
            for j, f in enumerate(idx):
                bufs[s][j].copy_(torch.from_numpy(by_index[f]))
            with torch.cuda.device(device):
                x = bufs[s][:len(idx)].to(device, non_blocking=True)
                copied[s] = torch.cuda.Event()
                copied[s].record()
                outs.append(eng.forward_u8(x, [pos[i * step] for i in range(first, last + 1)], T))
                if head is not None:               # only the top-5 crosses to the host, printed one call later
                    def emit(tops, stacks=range(first, last + 1)):
                        for j, i in enumerate(stacks):
                            print(f'{video_path} @ frames ({i * step}, {i * step + T})')
                            print_top_predictions(*(t[j:j + 1] for t in tops[0]), 'kinetics')
                    preds.submit([(head, outs[-1])], emit)
            state["next"], state["slot"] = last + 1, s ^ 1
            while kept and kept[0][0] < state["next"] * step:
                kept.popleft()

        f = 0
        while cap.isOpened():
            frame_exists, bgr = cap.read()
            if not frame_exists:
                cap.release()
                break
            if bufs is None:
                bufs = self._staging(tuple(bgr.shape))
            if f >= state["next"] * step and f % step < T:
                kept.append((f, bgr))      # some stack >= next contains frame f
            # stacks ending at frame f are complete; call once CLIPS_PER_CALL of them are waiting
            if f + 1 >= T and (f + 1 - T) % step == 0 and (f + 1 - T) // step - state["next"] + 1 == CLIPS_PER_CALL:
                submit((f + 1 - T) // step)
            f += 1
        n_stacks = (f - T) // step + 1 if f >= T else 0
        if n_stacks > state["next"]:
            submit(n_stacks - 1)
        if preds is not None:
            preds.flush()
        # one device->host copy per video; float64 like the reference's `.tolist()` -> np.array
        feats = torch.cat(outs).cpu().numpy().astype(np.float64) if outs else np.array([])
        return {self.feature_type: feats}

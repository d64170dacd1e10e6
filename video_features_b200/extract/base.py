"""What the frame, stack, flow and audio extractors share: checkpoint lookup, the per-video loop, per-device engine and
head caches, and the two video feeders.

Frame extractors (ExtractResNet, ExtractDINOv2; FrameExtractor below) read every frame sequentially with OpenCV (a
failed FIRST read is skipped, as the reference's extract_resnet.py:130-137 does).  Per chunk of FRAMES_PER_CALL frames:
  decoder frames (uint8 BGR) -> pinned host buffer -> device -> the extractor's encode step
Stack extractors (ExtractR21D, ExtractS3D, ExtractSwin3D, ExtractMViT; StackExtractor below) read frames sequentially
with OpenCV and keep only frames some stack of ``form_slices(n_frames, stack_size, step_size)`` needs, so host and
device memory do not grow with the video.  Per call of ``clips_per_call`` stacks:
  decoder frames (uint8 BGR, the stacks' frames once each) -> pinned host buffer -> device
  -> ``forward_u8(x, starts, T)``: the model's fused transform and network
In both, two pinned buffers alternate (one fills while the other's host->device copy runs) and the engine call is
asynchronous, so decoding the next frames overlaps the network on the current ones; the features stay on the device
until the video is finished (one device->host copy per video).  ``--show_pred``: after every engine call the
checkpoint's classifier runs on its device features (class_head.py) and only the top-5 crosses to the host, printed one
call later.
"""
from __future__ import annotations

import glob
import os
from collections import deque
from typing import Callable, Dict, Iterable, Iterator, List, Optional, Sequence, Tuple

import numpy as np
import torch
from tqdm import tqdm

from ..class_head import ClassHead, TopKQueue
from ..utils import AsyncSink, action_on_extraction, already_extracted, form_list_from_user_input, print_top_predictions

# frames per engine call of the frame extractors: frames are independent, so this cannot change any feature (the
# reference's --batch_size only groups frames for its own model calls).  Chosen by a sweep on one H100
# (scripts/resnet_time.py, README).
FRAMES_PER_CALL = 64


def checkpoint_dirs() -> List[str]:
    """Where weights are looked up, in order: $VF_CKPT_DIR, then torch hub's checkpoint cache
    ($TORCH_HOME/hub/checkpoints, default ~/.cache/torch/hub/checkpoints), where the reference's ``pretrained=True``
    and torchvision store them."""
    dirs = [os.environ.get("VF_CKPT_DIR"), os.path.join(torch.hub.get_dir(), "checkpoints")]
    return [d for d in dirs if d]


def load_first(pattern: str) -> Dict[str, torch.Tensor]:
    """The first file matching the glob ``pattern`` in the first of checkpoint_dirs() that has one, on the CPU."""
    dirs = checkpoint_dirs()
    for d in dirs:
        found = sorted(glob.glob(os.path.join(d, pattern)))
        if found:
            return torch.load(found[0], map_location="cpu")
    raise FileNotFoundError(f"{pattern} not found in {dirs} (set VF_CKPT_DIR or TORCH_HOME)")


class Extractor(torch.nn.Module):
    """The reference extractors' constructor attributes and ``forward(indices)``: per video, resume check, extract,
    sink, and the reference's catch-print-continue."""
    video_args = True       # extraction_fps and show_pred are attributes, and extraction_fps is refused
    output_direct = False
    failed_at = "Extraction failed at: {} with error (↑). Continuing extraction"

    def __init__(self, args):
        super().__init__()
        self.feature_type = args.feature_type
        self.path_list = form_list_from_user_input(args)
        if self.video_args:
            self.extraction_fps = args.extraction_fps
            self.show_pred = args.show_pred
            if self.extraction_fps is not None:
                raise NotImplementedError("extraction_fps re-encodes with ffmpeg (outside the rebuilt path, "
                                          "SURVEY.md §2)")
        self.keep_tmp_files = args.keep_tmp_files
        self.on_extraction = args.on_extraction
        self.tmp_path = os.path.join(args.tmp_path, self.feature_type)
        self.output_path = os.path.join(args.output_path, self.feature_type)
        self.progress = tqdm(total=len(self.path_list))
        self.keep_features = False
        self._per_device: Dict[tuple, object] = {}
        self._pinned: Dict[tuple, List[torch.Tensor]] = {}

    def forward(self, indices: torch.LongTensor):
        return self._run(indices, self.keep_features)

    def extract_video(self, device: torch.device, video_path) -> Dict[str, np.ndarray]:
        """``extract`` with the reference's signature: (device, model, classifier, video_path) here."""
        return self.extract(device, None, None, video_path)

    def _run(self, indices, keep: bool) -> list:
        device = indices.device
        if device.type != 'cuda':
            raise RuntimeError("the H100 engine has no CPU path: pass indices on a CUDA device")
        feats_list = []
        sink = AsyncSink() if os.environ.get("VF_ASYNC_SINK") == "1" else None    # opt-in extras, see ExtractCLIP.forward
        resume = os.environ.get("VF_RESUME") == "1"
        try:
            for idx in indices:
                video = self.path_list[idx]
                try:
                    if resume and already_extracted([self.feature_type], video, self.output_path, self.on_extraction,
                                                    self.output_direct):
                        self.progress.update()
                        continue
                    feats = self.extract_video(device, video)
                    if keep:
                        feats_list.append(feats)
                    if sink is not None:
                        sink.submit(feats, video, self.output_path, self.on_extraction, self.output_direct)
                    else:
                        action_on_extraction(feats, video, self.output_path, self.on_extraction, self.output_direct)
                except KeyboardInterrupt:
                    raise
                except Exception as err:
                    print(err)
                    print(self.failed_at.format(video))
                self.progress.update()
        finally:
            if sink is not None:
                sink.close()
        return feats_list

    def per_device(self, kind: str, device: torch.device, make: Callable[[int], object]):
        """One ``make(device index)`` per (kind, device), kept for the extractor's life."""
        key = (kind, device_index(device))
        if key not in self._per_device:
            self._per_device[key] = make(key[1])
        return self._per_device[key]

    def _staging(self, n: int, shape: tuple) -> List[torch.Tensor]:
        """Two pinned (n,) + shape uint8 staging buffers, kept for the last frame size: one fills while the other's
        host->device copy runs."""
        if (n,) + shape not in self._pinned:
            self._pinned = {(n,) + shape: [torch.empty((n,) + shape, dtype=torch.uint8).pin_memory() for _ in range(2)]}
        return self._pinned[(n,) + shape]


def device_index(device: torch.device) -> int:
    return device.index if device.index is not None else torch.cuda.current_device()


def _to_host(outs: List[torch.Tensor], float64: bool) -> np.ndarray:
    """One device->host copy per video; float64 where the reference builds its rows with ``.tolist()`` -> np.array."""
    feats = torch.cat(outs).cpu().numpy() if outs else np.array([])
    return feats.astype(np.float64) if float64 else feats


class FrameExtractor(Extractor):
    """Every frame, FRAMES_PER_CALL per engine call; outputs the rows plus 'fps' and 'timestamps_ms'."""
    float64 = False

    def encoder(self, device: torch.device, preds) -> Callable[[torch.Tensor], torch.Tensor]:
        """For one video: (n, H, W, 3) uint8 BGR frames on the device -> (n, D) device features; with --show_pred it
        also submits their top-5 to ``preds``."""
        raise NotImplementedError

    def extract(self, device: torch.device, model=None, classifier=None, video_path=None) -> Dict[str, np.ndarray]:
        import cv2
        preds = TopKQueue() if self.show_pred else None
        encode = self.encoder(device, preds)
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
                outs.append(encode(x))

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
                bufs = self._staging(FRAMES_PER_CALL, tuple(bgr.shape))
            if k == 0 and copied[slot] is not None:
                copied[slot].synchronize()          # the previous copy out of this buffer has finished
            bufs[slot][k].copy_(torch.from_numpy(bgr))
            k += 1
            if k == FRAMES_PER_CALL:
                submit(slot, k)
                slot, k = slot ^ 1, 0
        if preds is not None:
            preds.flush()
        return {self.feature_type: _to_host(outs, self.float64), 'fps': np.array(fps),
                'timestamps_ms': np.array(timestamps_ms)}


def stack_calls(frames: Iterable, T: int, step: int, per_call: int) -> Iterator[Tuple[int, list, List[int]]]:
    """Group the full stacks of ``form_slices(len(frames), T, step)`` into engine calls of ``per_call`` stacks (the last
    call may hold fewer).  Yields, per call, (index of its first stack, the frames of its stacks in order, each frame
    once, the position in that list where each of its stacks starts).  Only frames a pending stack needs are held, so
    a call never holds more than min(per_call * T, (per_call - 1) * step + T) frames."""
    kept = deque()                     # (frame index, frame) of frames some stack >= first contains
    first, n = 0, 0                    # first: first stack not yet yielded

    def call(last: int):
        end = last * step + T
        # a stack's frames are contiguous; consecutive stacks start min(step, T) frames apart in the list
        return first, [fr for f, fr in kept if f < end], [j * min(step, T) for j in range(last - first + 1)]

    for f, frame in enumerate(frames):
        n = f + 1
        if f >= first * step and f % step < T:
            kept.append((f, frame))
        # stacks ending at frame f are complete; a call goes once per_call of them are waiting
        if f + 1 >= T and (f + 1 - T) % step == 0 and (f + 1 - T) // step - first + 1 == per_call:
            last = (f + 1 - T) // step
            yield call(last)
            first = last + 1
            while kept and kept[0][0] < first * step:
                kept.popleft()
    n_stacks = (n - T) // step + 1 if n >= T else 0
    if n_stacks > first:
        yield call(n_stacks - 1)


def read_frames(cap) -> Iterator[np.ndarray]:
    """The frames of an opened cv2.VideoCapture, in order, until the first failed read."""
    while cap.isOpened():
        ok, bgr = cap.read()
        if not ok:
            cap.release()
            break
        yield bgr


class StackExtractor(Extractor):
    """Stacks of ``stack_size`` frames every ``step_size`` frames, ``clips_per_call`` stacks per engine call; outputs
    one row per full stack.  A subclass names its checkpoints and classifier and builds its engine."""
    feature_types: Sequence[str] = ()
    head_keys: Sequence[str] = ()      # the classifier's weight and bias in the checkpoint
    default_stack = default_step = 0
    clips_per_call = 4
    float64 = False

    def __init__(self, args):
        if args.feature_type not in self.feature_types:
            raise NotImplementedError(args.feature_type)
        super().__init__(args)
        self.step_size = args.step_size
        self.stack_size = args.stack_size
        if self.step_size is None:
            self.step_size = self.default_step
        if self.stack_size is None:
            self.stack_size = self.default_stack
        self.check_sizes()
        # the model's transform runs fused inside the engine
        self.transforms = None

    def check_sizes(self):
        if self.stack_size < 1 or self.step_size < 1:
            raise ValueError(f"stack_size {self.stack_size} and step_size {self.step_size} must be >= 1")

    def load_weights(self) -> Dict[str, torch.Tensor]:
        raise NotImplementedError

    def new_engine(self, idx: int):
        raise NotImplementedError

    def class_names(self) -> Optional[List[str]]:
        """The --show_pred class names; None: the Kinetics-400 names."""
        return None

    def new_head(self, idx: int) -> ClassHead:
        return ClassHead.from_state_dict(self.load_weights(), self.head_keys, idx, f"{self.feature_type} checkpoint")

    def _engine(self, device: torch.device):
        return self.per_device("engine", device, self.new_engine)

    def _head(self, device: torch.device) -> ClassHead:
        return self.per_device("head", device, self.new_head)

    def extract(self, device: torch.device, model=None, classifier=None, video_path=None) -> Dict[str, np.ndarray]:
        import cv2
        eng = self._engine(device)
        head = self._head(device) if self.show_pred else None
        preds = TopKQueue() if self.show_pred else None
        T, step, per_call = self.stack_size, self.step_size, self.clips_per_call
        cap = cv2.VideoCapture(video_path)
        if not cap.isOpened():             # the reference's read_video raises on an unreadable file
            raise RuntimeError(f"cannot open {video_path} for decoding")
        outs, s = [], 0
        bufs, copied = None, [None, None]  # copied[s]: event after the last host->device copy out of buffer s
        for first, frames, starts in stack_calls(read_frames(cap), T, step, per_call):
            if bufs is None:
                bufs = self._staging(min(per_call * T, (per_call - 1) * step + T), frames[0].shape)
            if copied[s] is not None:
                copied[s].synchronize()    # the previous copy out of this buffer has finished
            for j, bgr in enumerate(frames):
                bufs[s][j].copy_(torch.from_numpy(bgr))
            n = len(frames)
            del frames                     # the decoded frames are not held while the next call's are read
            with torch.cuda.device(device):
                x = bufs[s][:n].to(device, non_blocking=True)
                copied[s] = torch.cuda.Event()
                copied[s].record()
                outs.append(eng.forward_u8(x, starts, T))
                if head is not None:
                    def emit(tops, stacks=range(first, first + len(starts))):
                        for j, i in enumerate(stacks):
                            print(f'{video_path} @ frames ({i * step}, {i * step + T})')
                            print_top_predictions(*(t[j:j + 1] for t in tops[0]), 'kinetics', self.class_names())
                    preds.submit([(head, outs[-1])], emit)
            s ^= 1
        if preds is not None:
            preds.flush()
        return {self.feature_type: _to_host(outs, self.float64)}

"""Host utilities of the hot path: path listing, frame sampler, output sink, decoder access.

Mirrors the reference's ``utils/utils.py`` for the rows SURVEY.md §8 marks in scope (S1, S2, O1) -- same function
names, argument meaning, printed messages and error behaviour.  The sampler's index arithmetic runs in
libvfeat.so (``vf_sample_indices``); decoding uses OpenCV exactly as ``mmcv.VideoReader`` does (mmcv is the
reference's thin wrapper over ``cv2.VideoCapture``; it is not installed here).
"""
from __future__ import annotations

import argparse
import functools
import os
import pathlib as plb
import pickle
import queue
import threading
from typing import Dict, List, Optional

import numpy as np

from . import ops


class VideoReader:
    """The subset of ``mmcv.VideoReader`` the reference touches (utils/utils.py:310-330, extract_i3d.py:232-259):
    ``fps``, ``frame_cnt``, ``get_frame(i)`` (seek with CAP_PROP_POS_FRAMES, frames come back BGR, None on failure)."""

    def __init__(self, path: str):
        import cv2
        self._cv2 = cv2
        self._cap = cv2.VideoCapture(str(path))
        if not self._cap.isOpened():
            raise FileNotFoundError(f"cannot open video: {path}")
        self.fps = self._cap.get(cv2.CAP_PROP_FPS)
        self.frame_cnt = int(self._cap.get(cv2.CAP_PROP_FRAME_COUNT))
        self.width = int(self._cap.get(cv2.CAP_PROP_FRAME_WIDTH))
        self.height = int(self._cap.get(cv2.CAP_PROP_FRAME_HEIGHT))
        self._pos = 0

    def get_frame(self, frame_id: int):
        if frame_id < 0 or frame_id >= self.frame_cnt:
            raise IndexError(f'"frame_id" must be between 0 and {self.frame_cnt - 1}')
        if frame_id != self._pos:
            self._cap.set(self._cv2.CAP_PROP_POS_FRAMES, frame_id)
            pos = int(self._cap.get(self._cv2.CAP_PROP_POS_FRAMES))
            for _ in range(max(frame_id - pos, 0)):      # decoder landed early: read forward (mmcv does the same)
                self._cap.read()
        ok, img = self._cap.read()
        self._pos = frame_id + 1 if ok else int(self._cap.get(self._cv2.CAP_PROP_POS_FRAMES))
        return img if ok else None

    def read(self):
        ok, img = self._cap.read()
        if ok:
            self._pos += 1
        return img if ok else None

    def get_frame_into(self, frame_id: int, out: np.ndarray) -> bool:
        """`get_frame(frame_id)` decoded straight into `out` ((H,W,3) uint8, C-contiguous -- e.g. a row of a pinned staging
        buffer): the decoder's colour conversion writes there, no intermediate array.  False when the read fails."""
        if frame_id < 0 or frame_id >= self.frame_cnt:
            raise IndexError(f'"frame_id" must be between 0 and {self.frame_cnt - 1}')
        if frame_id != self._pos:
            self._cap.set(self._cv2.CAP_PROP_POS_FRAMES, frame_id)
            pos = int(self._cap.get(self._cv2.CAP_PROP_POS_FRAMES))
            for _ in range(max(frame_id - pos, 0)):
                self._cap.read()
        ok, img = self._cap.read(out)
        self._pos = frame_id + 1 if ok else int(self._cap.get(self._cv2.CAP_PROP_POS_FRAMES))
        if ok and img is not out and not np.shares_memory(img, out):
            np.copyto(out, img)                       # OpenCV allocated its own array (shape / layout mismatch)
        return bool(ok)


def extract_frames(path: str, method: str):
    """utils/utils.py:297-333.  method: ``uni_N`` (N frames uniformly) or ``fix_N`` (N frames per second).
    Returns (frames: list of HxWx3 uint8 BGR arrays or None, fps, timestamps_ms)."""
    kind, *params = method.split('_')
    if kind not in ('fix', 'uni'):
        raise NotImplementedError(f'{kind} are not supported')
    reader = VideoReader(str(path))
    indices = ops.sample_indices(kind, int(params[0]), reader.frame_cnt, reader.fps)
    per_frame = 0.001 / reader.fps                       # (sic) the reference's unit, utils/utils.py:312
    return [reader.get_frame(int(i)) for i in indices], reader.fps, [i * per_frame for i in indices]


class FrameStream:
    """`extract_frames` in two steps, for callers that own the destination memory: construction opens the video and fixes
    the sampled indices (so `count`, `hw`, `fps`, `timestamps_ms` are known), `read_into(dst)` then decodes the frames
    into `dst[(0..count)]`.  Frames whose read fails are dropped and later ones move up, as the reference drops its
    `None` frames (models/CLIP/extract_clip.py:122); the number of frames written is returned."""

    def __init__(self, path: str, method: str):
        kind, *params = method.split('_')
        if kind not in ('fix', 'uni'):
            raise NotImplementedError(f'{kind} are not supported')
        self._reader = VideoReader(str(path))
        self._indices = [int(i) for i in ops.sample_indices(kind, int(params[0]), self._reader.frame_cnt, self._reader.fps)]
        self.count = len(self._indices)
        self.hw = (self._reader.height, self._reader.width)
        self.fps = self._reader.fps
        per_frame = 0.001 / self._reader.fps              # (sic) utils/utils.py:312
        self.timestamps_ms = [i * per_frame for i in self._indices]

    def read_into(self, dst: np.ndarray) -> int:
        k = 0
        for i in self._indices:
            if self._reader.get_frame_into(i, dst[k]):
                k += 1
        return k


_SINK_EXT = {'save_numpy': 'npy', 'save_pickle': 'pkl'}
_NOT_FEATURES = ('fps', 'timestamps_ms')


def _sink_path(video_path, key: str, output_path: str, on_extraction: str, output_direct: bool) -> str:
    """<output_path>/<stem>.<ext> when output_direct, else <stem>_<key>.<ext> (utils/utils.py:83-88)."""
    stem = plb.Path(video_path).stem
    base = stem if output_direct is True else f'{stem}_{key}'
    return os.path.join(output_path, f'{base}.{_SINK_EXT[on_extraction]}')


def action_on_extraction(feats_dict: Dict[str, np.ndarray], video_path, output_path, on_extraction: str,
                         output_direct: bool = False):
    """utils/utils.py:50-114: print / save_numpy / save_pickle; 'fps' and 'timestamps_ms' are never saved."""
    if on_extraction != 'print' and on_extraction not in _SINK_EXT:
        if any(k not in _NOT_FEATURES for k in feats_dict):
            raise NotImplementedError(f'on_extraction: {on_extraction} is not implemented')
        return
    if isinstance(video_path, (list, tuple)):            # (video, flow) pairs: named after the video
        video_path = video_path[0]
    for key, value in feats_dict.items():
        if key in _NOT_FEATURES:
            continue
        if on_extraction == 'print':
            print(key)
            print(value)
            print(f'max: {value.max():.8f}; mean: {value.mean():.8f}; min: {value.min():.8f}')
            print()
            continue
        os.makedirs(output_path, exist_ok=True)
        target = _sink_path(video_path, key, output_path, on_extraction, output_direct)
        if len(value) == 0:
            print(f'Warning: the value is empty for {key} @ {target}')
        # written under a scratch name and renamed into place: an output file that exists is a complete file (the
        # resume check relies on it; a job killed mid-write leaves only `<target>.tmp`)
        scratch = target + '.tmp'
        with open(scratch, 'wb') as f:
            if on_extraction == 'save_numpy':
                np.save(f, value)
            else:
                pickle.dump(value, f)
        os.replace(scratch, target)


def sink_targets(feats_keys, video_path, output_path, on_extraction: str, output_direct: bool = False) -> List[str]:
    """Files `action_on_extraction` would write for these feature keys ([] for 'print')."""
    if on_extraction not in _SINK_EXT:
        return []
    if isinstance(video_path, (list, tuple)):
        video_path = video_path[0]
    return [_sink_path(video_path, k, output_path, on_extraction, output_direct) for k in feats_keys if k not in _NOT_FEATURES]


def already_extracted(feats_keys, video_path, output_path, on_extraction: str, output_direct: bool = False) -> bool:
    """Resume check (SURVEY 8(f) rank 2; the reference has none): every output file of this video exists and is
    non-empty.  Only meaningful for the saving sinks."""
    targets = sink_targets(feats_keys, video_path, output_path, on_extraction, output_direct)
    return bool(targets) and all(os.path.isfile(t) and os.path.getsize(t) > 0 for t in targets)


class AsyncSink:
    """Writer thread behind `action_on_extraction` (SURVEY 8(f) rank 2): the extractor hands a finished feature dict
    over and goes on with the next video while `np.save` / `pickle.dump` run here.  Same files, same names, same
    printed warnings; a failed write is reported like a failed extraction (message + continue) and counted in
    ``errors``.  ``close()`` drains the queue; use as a context manager."""

    def __init__(self, max_pending: int = 8):
        self._q: "queue.Queue[Optional[tuple]]" = queue.Queue(maxsize=max_pending)
        self.errors: List[tuple] = []
        self.written = 0
        self._t = threading.Thread(target=self._run, name="vf-sink", daemon=True)
        self._t.start()

    def _run(self):
        while True:
            item = self._q.get()
            if item is None:
                return
            feats, video_path, rest = item
            try:
                action_on_extraction(feats, video_path, *rest)
                self.written += 1
            except Exception as err:                     # mirror the extractors' per-video catch-print-continue
                self.errors.append((video_path, err))
                print(err)
                print(f'Saving failed at: {video_path}. Continuing extraction')

    def submit(self, feats_dict, video_path, output_path, on_extraction, output_direct: bool = False):
        if not self._t.is_alive():
            raise RuntimeError("AsyncSink is closed")
        self._q.put((feats_dict, video_path, (output_path, on_extraction, output_direct)))   # blocks when max_pending wait

    def close(self):
        if self._t.is_alive():
            self._q.put(None)
            self._t.join()

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()
        return False


@functools.lru_cache(maxsize=None)
def _class_names(dataset: str):
    if dataset == 'kinetics':
        from torchvision.models.video import R2Plus1D_18_Weights
        return tuple(R2Plus1D_18_Weights.KINETICS400_V1.meta["categories"])
    if dataset == 'imagenet':
        from torchvision.models import ResNet50_Weights
        return tuple(ResNet50_Weights.IMAGENET1K_V1.meta["categories"])
    raise NotImplementedError


def class_names(dataset: str) -> List[str]:
    """Class names of 'imagenet' (1000) or 'kinetics' (400), from the metadata torchvision ships with its weight enums
    (no download).  The Kinetics list equals the reference's K400_label_map.txt; the ImageNet names are the first name
    of each IN_label_map.txt line (two differ in spelling: 'crane bird', 'maillot tank suit')."""
    return list(_class_names(dataset))


def print_top_predictions(top_idx, top_logit, top_prob, dataset: str, classes: Optional[List[str]] = None):
    """Per row, the reference's lines `{logit:.3f} {softmax:.3f} {class}` for each of the k entries, then an empty
    line (utils/utils.py:44-47); top_* are (n, k) host tensors, as ClassHead.top_k_host returns them."""
    classes = _class_names(dataset) if classes is None else classes
    for idx, lg, pr in zip(top_idx.tolist(), top_logit.tolist(), top_prob.tolist()):
        for i, logit, smax in zip(idx, lg, pr):
            print(f'{logit:.3f} {smax:.3f} {classes[i]}')
        print()


def show_predictions_on_dataset(logits, dataset: str, classes: Optional[List[str]] = None):
    """utils/utils.py:19-47 on (B, classes) logits that are already at hand: softmax, sorted descending (equal
    probabilities by the lower class index), the top 5 printed per row.  The extractors do not come through here:
    they print the top-k the classifier-head kernel returns (print_top_predictions)."""
    import torch
    import torch.nn.functional as F
    if dataset not in ('imagenet', 'kinetics'):
        raise NotImplementedError
    logits = torch.as_tensor(logits)
    softmaxes = F.softmax(logits, dim=-1)
    _, top_idx = torch.sort(softmaxes, dim=-1, descending=True, stable=True)
    k = 5
    top_idx = top_idx[:, :k]
    print_top_predictions(top_idx, logits.gather(1, top_idx), softmaxes.gather(1, top_idx), dataset, classes)


def form_slices(size: int, stack_size: int, step_size: int):
    """utils/utils.py:117-126: (start, end) of every full stack."""
    n_full = (size - stack_size) // step_size + 1
    return [(k * step_size, k * step_size + stack_size) for k in range(n_full)]


def sanity_check(args: argparse.Namespace):
    """utils/utils.py:129-150 (the checks that concern CLIP / I3D / RAFT)."""
    if os.path.relpath(args.output_path) == os.path.relpath(args.tmp_path):
        raise AssertionError('The same path for out & tmp')
    if args.feature_type.startswith('dinov2_'):
        if args.show_pred:
            raise AssertionError(f'--show_pred: the {args.feature_type} checkpoint is a backbone without a classifier')
        if args.stack_size is not None:
            raise AssertionError(f'--stack_size: {args.feature_type} gives one feature per frame; stacks do not apply')
    if args.feature_type.startswith('videomae_') and args.stack_size is not None and args.stack_size != 16:
        raise AssertionError(f'--stack_size: {args.feature_type} takes stacks of 16 frames (its positional table is '
                             f'built for 16 frames); got {args.stack_size}')
    if args.show_pred:
        print('--show_pred: only the first of the listed GPUs is used')
        args.device_ids = args.device_ids[:1]
    if args.feature_type == 'i3d' and args.stack_size is not None and args.stack_size < 10:
        raise AssertionError(f'I3D model does not support inputs shorter than 10 timestamps. You have: {args.stack_size}')
    if getattr(args, 'model_name', None) is not None and args.feature_type != 'r21d_rgb':
        raise AssertionError(f'--model_name selects the r21d_rgb network; it does not apply to {args.feature_type}')
    if getattr(args, 'pred_texts', None) is not None:
        if not args.feature_type.startswith('CLIP'):
            raise AssertionError(f'--pred_texts are zero-shot prompts of the CLIP feature types; they do not apply to '
                                 f'{args.feature_type}')
        if not args.show_pred:
            raise AssertionError('--pred_texts only takes effect with --show_pred')


def _paired(videos, flows):
    """(video, flow) pairs whose file stems agree, in the given order."""
    return [(str(v), str(f)) for v, f in zip(videos, flows) if plb.Path(v).stem == plb.Path(f).stem]


def form_list_from_user_input(args: argparse.Namespace) -> list:
    """utils/utils.py:153-204: file with paths / directory glob / explicit list; ValueError when nothing is given or
    a path is missing."""
    listing, vdir, vpaths = (getattr(args, k, None) for k in ('file_with_video_paths', 'video_dir', 'video_paths'))
    fdir, fpaths = getattr(args, 'flow_dir', None), getattr(args, 'flow_paths', None)
    if listing is not None:
        with open(listing) as f:
            paths = [ln.replace('\n', '') for ln in f]
        paths = [p for p in paths if p]
    elif vdir is not None:
        found = list(plb.Path(vdir).glob('*'))               # unsorted, as the reference (utils/utils.py:173)
        if fdir is None:
            paths = [str(p) for p in found]
        else:
            by_stem = lambda x: x.stem
            paths = _paired(sorted(found, key=by_stem), sorted(plb.Path(fdir).glob('*'), key=by_stem))
    elif vpaths is not None:
        paths = vpaths if fpaths is None else _paired(vpaths, fpaths)
    else:
        raise ValueError('no video provided')

    for entry in paths:
        if isinstance(entry, tuple):
            assert os.path.exists(entry[0])
            assert os.path.exists(entry[1])
        elif not os.path.exists(entry):
            print(f'The path does not exist: {entry}')
            raise ValueError('path not exist')
    return paths

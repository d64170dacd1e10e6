"""``ExtractI3D`` -- drop-in for the reference's models/i3d/extract_i3d.py on the H100 engine.

Same constructor / attributes / ``forward(indices)`` / ``extract(...)`` surface, dict keys ('rgb', 'flow', 'fps',
'timestamps_ms'), stack / step logic (stack_size+1 frames per stack, one overlap frame when step == stack) and
float64 ``(n_stacks, 1024)`` outputs.  Underneath, per group of up to ``VF_I3D_STACKS`` (default 8) stacks:
  decoder frames (uint8, BGR kept as the reference does) -> GPU Pillow-exact bilinear resize to min side 256
  -> rgb stream : fused crop + 2x/255-1 + phase packing -> I3D on all stacks of the group (vf_i3d_forward_u8_strided)
  -> flow stream: PWC-Net (``--flow_type pwc``, the CLI default) on the stack's 65 resized BGR frames, as the reference
     passes them (extract_i3d.py:175), at the frame size; or RAFT on the 64 consecutive pairs of each stack, padded
     and NOT unpadded (extract_i3d.py:172)
     -> fused crop + clamp + 8-bit quantisation + scaling -> I3D (vf_i3d_forward_flow)
Features stay on the device until the video is finished: one device->host copy per stream per video instead of the
reference's ``.tolist()`` per stack (extract_i3d.py:188).
``--flow_type flow`` (pre-computed ``flow_x_*.jpg`` / ``flow_y_*.jpg`` pairs, extract_i3d.py:195-229,266-278) feeds
the same fused flow transform.
``--show_pred``: the checkpoint's conv3d_0c_1x1 runs on each group's device features (I3DEngine.head); per stack and
per stream, the header ``{video_path} @ stack {i} ({stream} stream)`` and the Kinetics top-5 are printed, stack-major as
the reference loops (extract_i3d.py:180-229); with ``--flow_type flow`` only the flow stream prints, as there.
"""
from __future__ import annotations

import os
import pathlib
import traceback
from typing import Dict, List

import numpy as np
import torch
from tqdm import tqdm

from .. import ops
from .._lib import VF_FILTER_BILINEAR
from ..class_head import TopKQueue
from ..i3d_engine import I3DEngine
from ..pwc_engine import PWCEngine
from ..raft_engine import RAFTEngine
from ..utils import (AsyncSink, already_extracted, VideoReader, action_on_extraction, form_list_from_user_input,
                     print_top_predictions)

PRE_CENTRAL_CROP_MIN_SIDE_SIZE = 256
CENTRAL_CROP_MIN_SIDE_SIZE = 224
DEFAULT_I3D_STEP_SIZE = 64
DEFAULT_I3D_STACK_SIZE = 64
_HERE = pathlib.Path(__file__).resolve().parent
_CKPT_DIRS = [os.environ.get("VF_CKPT_DIR"), str(_HERE / "checkpoints"), str(_HERE.parents[1] / "checkpoints")]
_CKPT = {'rgb': 'i3d_rgb.pt', 'flow': 'i3d_flow.pt', 'raft': 'raft-sintel.pth', 'pwc': 'pwc_net_sintel.pt'}
_STATE_DICTS: Dict[str, Dict[str, torch.Tensor]] = {}


def load_checkpoint(kind: str) -> Dict[str, torch.Tensor]:
    """The reference's vendored weights (models/i3d/checkpoints/i3d_{rgb,flow}.pt, models/raft/checkpoints/
    raft-sintel.pth, models/pwc/checkpoints/pwc_net_sintel.pt), looked up in $VF_CKPT_DIR or ./checkpoints; read from disk once per process."""
    if kind not in _STATE_DICTS:
        for d in _CKPT_DIRS:
            if d and os.path.exists(os.path.join(d, _CKPT[kind])):
                _STATE_DICTS[kind] = torch.load(os.path.join(d, _CKPT[kind]), map_location="cpu")
                break
        else:
            raise FileNotFoundError(f"{_CKPT[kind]} not found in {[d for d in _CKPT_DIRS if d]} (set VF_CKPT_DIR)")
    return _STATE_DICTS[kind]


def stack_windows(n_frames: int, stack_size: int, step_size: int, extra: int = 1) -> List[range]:
    """Frame index ranges of the stacks the reference's feeding loop produces (extract_i3d.py:266-296): frames are
    appended one at a time, a stack fires when it holds ``stack_size + extra`` frames and then drops its first
    ``step_size`` entries (``extra`` = 1: B+1 frames give B flow fields; 0 in the pre-computed-flow branch)."""
    out, held = [], []
    for i in range(n_frames):
        held.append(i)
        if len(held) - extra == stack_size:
            out.append(range(held[0], held[-1] + 1))
            held = held[step_size:]
    return out


class ExtractI3D(torch.nn.Module):

    def __init__(self, args, external_call=False):
        super(ExtractI3D, self).__init__()
        self.feature_type = args.feature_type
        self.streams = ['rgb', 'flow'] if args.streams is None else args.streams
        self.path_list = form_list_from_user_input(args)
        self.flow_type = args.flow_type
        self.min_side_size = PRE_CENTRAL_CROP_MIN_SIDE_SIZE
        self.central_crop_size = CENTRAL_CROP_MIN_SIDE_SIZE
        self.extraction_fps = args.extraction_fps
        self.step_size = args.step_size if args.step_size is not None else DEFAULT_I3D_STEP_SIZE
        self.stack_size = args.stack_size if args.stack_size is not None else DEFAULT_I3D_STACK_SIZE
        self.show_pred = args.show_pred
        self.keep_tmp_files = args.keep_tmp_files
        self.on_extraction = args.on_extraction
        self.tmp_path = os.path.join(args.tmp_path, self.feature_type)
        self.external_call = external_call
        if external_call is False:
            self.output_direct = args.output_direct
            self.output_path = args.output_path if self.output_direct is True else os.path.join(args.output_path, self.feature_type)
        if 'flow' in self.streams and self.flow_type not in ('pwc', 'raft', 'flow'):
            raise NotImplementedError(f"flow_type '{self.flow_type}': the PWC, RAFT and pre-computed flow branches are "
                                      "built on the H100 engine")
        self.progress = tqdm(total=len(self.path_list))
        self.group_stacks = max(1, int(os.environ.get("VF_I3D_STACKS", "8")))     # stacks per engine call
        self.keep_features = False
        self._models: Dict[int, dict] = {}

    def _load(self, device: torch.device) -> dict:
        if device.type != 'cuda':
            raise RuntimeError("the H100 engine has no CPU path: pass indices on a CUDA device")
        idx = device.index if device.index is not None else torch.cuda.current_device()
        if idx not in self._models:
            m = {s: I3DEngine(load_checkpoint(s), s, idx, max_stacks=self.group_stacks, max_T=max(self.stack_size, 16))
                 for s in self.streams}
            self._models[idx] = {'i3d': m, 'raft': None, 'raft_cap': (0, 0, 0), 'pwc': None, 'pwc_cap': (0, 0, 0),
                                 'device_index': idx}
        return self._models[idx]

    @staticmethod
    def _raft(models: dict, frames: int, h: int, w: int) -> RAFTEngine:
        """The RAFT engine of this device, re-created (the old one closed) whenever a video needs more frames per call
        or a larger frame than its workspace holds -- a list may mix aspect ratios."""
        cf, ch, cw = models['raft_cap']
        if models['raft'] is None or frames > cf or h > ch or w > cw:
            if models['raft'] is not None:
                models['raft'].close()
            cap = (max(cf, frames), max(ch, h), max(cw, w))
            models['raft'] = RAFTEngine(load_checkpoint('raft'), models['device_index'], max_frames=cap[0], max_h=cap[1],
                                        max_w=cap[2])
            models['raft_cap'] = cap
        return models['raft']

    @staticmethod
    def _pwc(models: dict, frames: int, h: int, w: int) -> PWCEngine:
        """The PWC-Net engine of this device, re-created like the RAFT engine (_raft) when a video outgrows it."""
        cf, ch, cw = models['pwc_cap']
        if models['pwc'] is None or frames > cf or h > ch or w > cw:
            if models['pwc'] is not None:
                models['pwc'].close()
            cap = (max(cf, frames), max(ch, h), max(cw, w))
            models['pwc'] = PWCEngine(load_checkpoint('pwc'), models['device_index'], max_frames=cap[0], max_h=cap[1],
                                      max_w=cap[2])
            models['pwc_cap'] = cap
        return models['pwc']

    def forward(self, indices: torch.LongTensor):
        device = indices.device
        models = self._load(device)
        feats_list = []
        saving = self.external_call is False           # opt-in extras (SURVEY 8(f) rank 2), see ExtractCLIP.forward
        sink = AsyncSink() if saving and os.environ.get("VF_ASYNC_SINK") == "1" else None
        resume = saving and os.environ.get("VF_RESUME") == "1"
        try:
            for idx in indices:
                try:
                    if resume and already_extracted(self.streams, self.path_list[idx], self.output_path, self.on_extraction):
                        self.progress.update()
                        continue
                    feats_dict = self.extract(device, None, models, self.path_list[idx])
                    if self.external_call is not False or self.keep_features:
                        feats_list.append(feats_dict)
                    if self.external_call is not False:
                        pass
                    elif sink is not None:
                        sink.submit(feats_dict, self.path_list[idx], self.output_path, self.on_extraction)
                    else:
                        action_on_extraction(feats_dict, self.path_list[idx], self.output_path, self.on_extraction)
                except KeyboardInterrupt:
                    raise KeyboardInterrupt
                except Exception as e:
                    print(e)
                    print(f'Extraction failed at: {self.path_list[idx]}. Continuing extraction')
                    traceback.print_exc()
                self.progress.update()
        finally:
            if sink is not None:
                sink.close()
        return feats_list

    # ------------------------------------------------------------------ one group of stacks on the device
    def _resized(self, frames: List[np.ndarray], device: torch.device) -> torch.Tensor:
        x = torch.from_numpy(np.stack(frames)).to(device, non_blocking=True)
        h, w = x.shape[1:3]
        oh, ow = ops.resize_geometry(h, w, self.min_side_size, True)
        if (oh, ow) != (h, w):
            x = torch.ops.vfeat.resize_u8(x, oh, ow, VF_FILTER_BILINEAR)          # ToPILImage -> ResizeImproved(256)
        return x

    def _run_group(self, feats: Dict[str, list], x: torch.Tensor, first: int, windows: List[range], models: dict,
                   flow_stacks=None):
        """x: resized uint8 frames [first, first + len(x)) of the video on the device; windows: the stacks of this group.
        Appends one (len(windows), 1024) device tensor per stream (extract_i3d.py:160-193)."""
        n = len(windows)
        span = len(windows[0])
        fsz = x.shape[1] * x.shape[2] * 3
        starts = [w.start - first for w in windows]
        for stream in self.streams:
            if stream == 'rgb':
                T = span - 1                                                       # rgb_stack[:-1]
                step = starts[1] - starts[0] if n > 1 else span
                if n == 1 or all(b - a == step for a, b in zip(starts, starts[1:])):
                    v = x[starts[0]:].as_strided((n, T, x.shape[1], x.shape[2], 3), (step * fsz, fsz, x.shape[2] * 3, 3, 1))
                else:
                    v = torch.stack([x[s:s + T] for s in starts])
                feats['rgb'].append(models['i3d']['rgb'].forward_frames_u8(v))      # crop / scale fused
            elif stream == 'flow':
                if flow_stacks is not None:                                        # --flow_type flow: jpg pairs
                    flow = flow_stacks
                elif self.flow_type == 'pwc':
                    # the stack's BGR frames as the reference passes them (extract_i3d.py:175), flow at the frame size
                    pwc = self._pwc(models, span, x.shape[1], x.shape[2])
                    flow = torch.stack([pwc.flow(x[s:s + span]) for s in starts])
                else:
                    raft = self._raft(models, span, x.shape[1], x.shape[2])
                    # padded flow, never unpadded, as the reference feeds it (extract_i3d.py:172)
                    flow = torch.stack([raft.flow(x[s:s + span], iters=20, unpad=False) for s in starts])
                feats['flow'].append(models['i3d']['flow'].forward_flow(flow))
            else:
                raise NotImplementedError

    def _show_group(self, preds: TopKQueue, feats: Dict[str, list], g0: int, n: int, models: dict, video_path):
        """Queues the Kinetics top-5 of the group's last feature block per stream, printed stack-major once they are
        on the host; only the top-5 crosses to the host."""
        shown = [s for s in self.streams if not (self.flow_type == 'flow' and s != 'flow')]   # extract_i3d.py:226

        def emit(tops):
            for j in range(n):
                for s, top in zip(shown, tops):
                    print(f'{video_path} @ stack {g0 + j} ({s} stream)')
                    print_top_predictions(*(t[j:j + 1] for t in top), 'kinetics')
        preds.submit([(models['i3d'][s].head(), feats[s][-1]) for s in shown], emit)

    @staticmethod
    def _read_flow_pair(fx, fy) -> torch.Tensor:
        import cv2                                        # mmcv.imread(flag='grayscale') is cv2.imread(IMREAD_GRAYSCALE)
        a, b = cv2.imread(str(fx), cv2.IMREAD_GRAYSCALE), cv2.imread(str(fy), cv2.IMREAD_GRAYSCALE)
        if a is None or b is None:
            raise FileNotFoundError(f"cannot read flow images {fx} / {fy}")
        return torch.from_numpy(np.stack([a, b]))

    def extract(self, device, flow_xtr_model, models, video_path=None):
        flows = None
        if self.flow_type == 'flow':                         # path_list entries are (video, flow image folder) pairs
            video = VideoReader(str(video_path[0]))
            by_number = lambda p: p.stem[7:]                 # (sic) string order, extract_i3d.py:233-236
            fxs = sorted(pathlib.Path(video_path[1]).glob("flow_x*.jpg"), key=by_number)
            fys = sorted(pathlib.Path(video_path[1]).glob("flow_y*.jpg"), key=by_number)
            flows = list(zip(fxs, fys))
        else:
            video = VideoReader(str(video_path[0] if isinstance(video_path, (tuple, list)) else video_path))
        fps, frame_cnt = video.fps, video.frame_cnt
        mspf = 0.001 / fps                                   # (sic) extract_i3d.py:241
        if self.extraction_fps is not None:
            samples_num = int(frame_cnt / fps * self.extraction_fps)
            samples_ix = np.linspace(1, frame_cnt - 1, samples_num).astype(int)
        elif frame_cnt < DEFAULT_I3D_STACK_SIZE + 1:          # short video: resampled up to 65 frames
            samples_ix = np.linspace(1, frame_cnt - 1, DEFAULT_I3D_STACK_SIZE + 1).astype(int)
        else:
            samples_ix = np.arange(frame_cnt)
        frames, timestamps_ms = [], [i * mspf for i in samples_ix]
        for i in samples_ix:
            f = video.get_frame(int(i)) if int(i) < frame_cnt else None
            if f is not None:
                frames.append(f)
        feats: Dict[str, list] = {stream: [] for stream in self.streams}
        if flows is not None:
            # pre-computed flow: frame k is paired with flow image k; a stack fires at stack_size entries, the rgb stream
            # still drops its last frame (extract_i3d.py:195-229,268-278)
            n = min(len(frames), len(flows))
            windows = stack_windows(n, self.stack_size, self.step_size, extra=0)
        else:
            windows = stack_windows(len(frames), self.stack_size, self.step_size, extra=1)
        preds = TopKQueue() if self.show_pred else None
        for g0 in range(0, len(windows), self.group_stacks):
            group = windows[g0:g0 + self.group_stacks]
            first, last = group[0].start, group[-1].stop
            x = self._resized(frames[first:last], device)
            fl = None
            if flows is not None and 'flow' in self.streams:
                fl = torch.stack([torch.stack([self._read_flow_pair(*flows[i]) for i in w]) for w in group])
                fl = fl.to(device, non_blocking=True).float()                      # uint8 grey levels, as the reference reads them
            self._run_group(feats, x, first, group, models, fl)
            if preds is not None:
                self._show_group(preds, feats, g0, len(group), models, video_path)
        if preds is not None:
            preds.flush()
        # one device->host copy per stream; float64 like the reference's `.tolist()` -> np.array
        feats_dict = {s: (torch.cat(v).cpu().numpy().astype(np.float64) if v else np.array([])) for s, v in feats.items()}
        feats_dict['fps'] = np.array(fps)
        feats_dict['timestamps_ms'] = np.array(timestamps_ms)
        return feats_dict

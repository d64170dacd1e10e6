"""``ExtractRAFT`` -- drop-in for the reference's models/raft/extract_raft.py on the H100 engine.

Same constructor / attributes / ``forward`` (returns None) / ``extract`` surface; output key 'raft' is a float64
``(T-1, 2, H, W)`` array (the reference builds it with ``.tolist()``), saved under ``{output_path}/raft``.  Frames are
read sequentially with OpenCV, converted BGR->RGB (extract_raft.py:133 -- the stand-alone extractor does swap),
optionally resized (``--side_size``, Pillow-exact bilinear on the GPU), and processed in windows of max(batch_size, 16)+1 frames
with the last frame carried over; padding to /8 and unpadding happen inside the engine.
"""
from __future__ import annotations

import os
from typing import Dict

import numpy as np
import torch
from tqdm import tqdm

from .. import ops
from .._lib import VF_FILTER_BILINEAR
from ..raft_engine import RAFTEngine
from ..utils import AsyncSink, action_on_extraction, already_extracted, form_list_from_user_input
from .extract_i3d import load_checkpoint


# attributes the reference's constructor copies from `args` unchanged (extract_raft.py:24-36)
_ARG_ATTRS = ('feature_type', 'batch_size', 'extraction_fps', 'resize_to_smaller_edge', 'side_size', 'show_pred',
              'keep_tmp_files', 'on_extraction')


class ExtractRAFT(torch.nn.Module):

    def __init__(self, args):
        super().__init__()
        for name in _ARG_ATTRS:
            setattr(self, name, getattr(args, name))
        self.path_list = form_list_from_user_input(args)
        # per-feature sub-folders of the scratch and output roots, as the reference lays them out
        self.tmp_path, self.output_path = (os.path.join(root, self.feature_type) for root in (args.tmp_path, args.output_path))
        self.progress = tqdm(total=len(self.path_list))
        if self.extraction_fps is not None:
            raise NotImplementedError("extraction_fps re-encodes with ffmpeg (outside the rebuilt path, SURVEY.md §2)")
        self._engines: Dict[int, tuple] = {}              # device index -> (engine, (frames, h, w) capacity)
        # pairs per engine call: frame pairs are independent, so how many share a call does not change any value; the
        # reference's default of one pair per call (--batch_size 1) would leave the GPU idle between launches
        self.pairs_per_call = max(self.batch_size, int(os.environ.get("VF_RAFT_PAIRS", "16")))

    def forward(self, indices: torch.LongTensor):
        device = indices.device
        if device.type != 'cuda':
            raise RuntimeError("the H100 engine has no CPU path: pass indices on a CUDA device")
        sink = AsyncSink() if os.environ.get("VF_ASYNC_SINK") == "1" else None     # opt-in extras, see ExtractCLIP.forward
        resume = os.environ.get("VF_RESUME") == "1"
        try:
            for idx in indices:
                video = self.path_list[idx]
                try:                                      # per-video catch-print-continue (extract_raft.py:60-75)
                    if resume and already_extracted([self.feature_type], video, self.output_path, self.on_extraction):
                        self.progress.update()
                        continue
                    feats = self.extract(device, None, video)
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

    def _engine(self, device: torch.device, h: int, w: int) -> RAFTEngine:
        """One engine per device.  Its workspace is sized for the largest frame seen so far; a larger frame closes it
        and creates a bigger one (a list of many resolutions must not accumulate engines until cudaMalloc fails)."""
        idx = device.index if device.index is not None else torch.cuda.current_device()
        eng, cap = self._engines.get(idx, (None, (0, 0, 0)))
        if eng is None or h > cap[1] or w > cap[2]:
            if eng is not None:
                eng.close()
            cap = (self.pairs_per_call + 1, max(cap[1], h), max(cap[2], w))
            eng = self._new_engine(idx, cap)
            self._engines[idx] = (eng, cap)
        return eng

    def _new_engine(self, idx: int, cap: tuple):
        return RAFTEngine(load_checkpoint('raft'), idx, max_frames=cap[0], max_h=cap[1], max_w=cap[2])

    def _flow_of_frames(self, x: torch.Tensor, device) -> torch.Tensor:
        """x: (n+1, H, W, 3) uint8 RGB frames on the device -> (n, 2, H, W) fp32 flow."""
        return self._engine(device, x.shape[1], x.shape[2]).flow(x, iters=20, unpad=True)

    def _flow_of_window(self, window, device) -> list:
        """window: n+1 RGB frames (H, W, 3) uint8 -> [one (n, 2, H, W) float64 array]."""
        x = torch.from_numpy(np.stack(window)).to(device)
        if self.side_size is not None:
            oh, ow = ops.resize_geometry(x.shape[1], x.shape[2], self.side_size, self.resize_to_smaller_edge)
            if (oh, ow) != tuple(x.shape[1:3]):
                x = torch.ops.vfeat.resize_u8(x, oh, ow, VF_FILTER_BILINEAR)
        # float64 (T, 2, H, W) on the host: the same values `.tolist()` -> np.array gives the reference, without
        # materialising 8 bytes + a Python float object per flow component
        return [self._flow_of_frames(x, device).cpu().numpy().astype(np.float64)]

    def extract(self, device, model, video_path=None) -> Dict[str, np.ndarray]:
        import cv2
        cap = cv2.VideoCapture(video_path)
        fps = cap.get(cv2.CAP_PROP_FPS)
        stamps, window, flows = [], [], []
        seen_first = False
        while cap.isOpened():
            ok, bgr = cap.read()
            if not seen_first:                            # a failed FIRST read is retried (extract_raft.py:124-128)
                seen_first = True
                if ok is False:
                    continue
            if not ok:                                    # end of stream: flush the partial window
                if len(window) > 1:
                    flows.extend(self._flow_of_window(window, device))
                cap.release()
                break
            stamps.append(cap.get(cv2.CAP_PROP_POS_MSEC))
            window.append(cv2.cvtColor(bgr, cv2.COLOR_BGR2RGB))      # the stand-alone extractor swaps to RGB
            if len(window) == self.pairs_per_call + 1:
                flows.extend(self._flow_of_window(window, device))
                window = window[-1:]                      # the last frame opens the next window
        flows = np.concatenate(flows) if flows else np.array(flows)
        return {self.feature_type: flows, 'fps': np.array(fps), 'timestamps_ms': np.array(stamps)}

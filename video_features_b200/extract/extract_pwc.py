"""``ExtractPWC`` -- drop-in for the reference's models/pwc/extract_pwc.py on the H100 engine.

Same constructor / attributes / ``forward`` (returns None) / ``extract`` surface; output key 'pwc' is a float64
``(T-1, 2, H, W)`` array (the reference builds it with ``.tolist()``), saved under ``{output_path}/pwc``.  The read
loop is ExtractRAFT's, as the two reference extractors share it line for line (extract_pwc.py:104-156,
extract_raft.py:108-160): frames read with OpenCV and converted BGR->RGB (extract_pwc.py:129), optionally resized
(``--side_size``, Pillow-exact bilinear on the GPU), processed in windows of max(batch_size, 16)+1 frames with the
last frame carried over.  The /64 resize and the channel swap the model does itself happen inside the engine.
"""
from __future__ import annotations

import torch

from ..pwc_engine import PWCEngine
from .extract_i3d import load_checkpoint
from .extract_raft import ExtractRAFT


class ExtractPWC(ExtractRAFT):

    def _new_engine(self, idx: int, cap: tuple) -> PWCEngine:
        return PWCEngine(load_checkpoint('pwc'), idx, max_frames=cap[0], max_h=cap[1], max_w=cap[2])

    def _flow_of_frames(self, x: torch.Tensor, device) -> torch.Tensor:
        return self._engine(device, x.shape[1], x.shape[2]).flow(x)

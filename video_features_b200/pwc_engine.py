"""PWC-Net optical-flow handle: stands where the reference keeps ``PWCNet()`` with pwc_net_sintel.pt loaded
(models/pwc/extract_pwc.py:57-60, models/i3d/extract_i3d.py:97-102)."""
from __future__ import annotations

import ctypes as C
from typing import Dict

import numpy as np
import torch

from ._lib import NamedTensor, check, lib, read_split_conv

# debug_read ids (include/vfeat.h vf_pwc_debug_read)
FEATURES, VOLUME, UPFLOW, UPFEAT, FLOW, REFINE, MASK = range(7)


class PWCEngine:
    """``state_dict``: the reference checkpoint (keys with or without a ``module.`` prefix)."""

    def __init__(self, state_dict: Dict[str, torch.Tensor], device: int = 0, max_frames: int = 17, max_h: int = 256,
                 max_w: int = 384):
        if not torch.cuda.is_available():
            raise RuntimeError("PWCEngine needs a CUDA device (sm_90a); there is no CPU fallback")
        self.device = torch.device("cuda", device)
        keep = []
        items = [(k[7:] if k.startswith("module.") else k, v) for k, v in state_dict.items()
                 if torch.is_tensor(v) and v.dtype.is_floating_point]
        arr = (NamedTensor * len(items))()
        for i, (k, v) in enumerate(items):
            a = np.ascontiguousarray(v.detach().to("cpu", torch.float32).numpy())
            nm = k.encode()
            keep.append((a, nm))
            arr[i].name = nm
            arr[i].data = a.ctypes.data_as(C.POINTER(C.c_float))
            arr[i].numel = a.size
        h = C.c_void_p()
        check(lib().vf_pwc_create(C.byref(h), arr, len(items), device, max_frames, max_h, max_w))
        self._h = h
        del keep

    def flow(self, frames: torch.Tensor) -> torch.Tensor:
        """frames: (N, 3, H, W) float in [0,255] or (N, H, W, 3) uint8, on this device, N >= 2, in the channel order the
        reference's caller passes (the model swaps channels 0 and 2 itself).  Returns (N-1, 2, H, W) fp32 ==
        PWCNet()(frames[:-1], frames[1:])."""
        if not frames.is_cuda:
            raise RuntimeError("PWCEngine expects CUDA frames (no CPU fallback)")
        frames = frames.contiguous()
        if frames.dtype == torch.uint8:
            assert frames.dim() == 4 and frames.shape[3] == 3
            n, hs, ws, is_u8, chw = frames.shape[0], frames.shape[1], frames.shape[2], 1, 0
        else:
            frames = frames.to(torch.float32)
            assert frames.dim() == 4 and frames.shape[1] == 3
            n, hs, ws, is_u8, chw = frames.shape[0], frames.shape[2], frames.shape[3], 0, 1
        out = torch.empty((n - 1, 2, hs, ws), device=frames.device, dtype=torch.float32)
        with torch.cuda.device(self.device):
            check(lib().vf_pwc_flow(self._h, frames.data_ptr(), is_u8, chw, n, hs, ws, out.data_ptr(),
                                    torch.cuda.current_stream().cuda_stream))
        return out

    def debug_read(self, what: int, level: int = 2) -> torch.Tensor:
        """An internal tensor of the last call (ids above, include/vfeat.h vf_pwc_debug_read) as fp32 NCHW."""
        dims = (C.c_int * 4)()
        check(lib().vf_pwc_debug_read(self._h, what, level, None, 0, dims, None))
        out = torch.empty(tuple(dims), device=self.device, dtype=torch.float32)
        with torch.cuda.device(self.device):
            check(lib().vf_pwc_debug_read(self._h, what, level, out.data_ptr(), out.numel(), dims,
                                          torch.cuda.current_stream().cuda_stream))
        return out

    def conv(self, index: int) -> dict:
        """Diagnostics: conv ``index`` as uploaded (include/vfeat.h vf_pwc_conv gives the order); see
        _lib.read_split_conv."""
        with torch.cuda.device(self.device):
            return read_split_conv(lib().vf_pwc_conv, self._h, index, self.device)

    @property
    def launch_count(self) -> int:
        return int(lib().vf_pwc_launch_count(self._h))

    def close(self):
        if getattr(self, "_h", None):
            lib().vf_pwc_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

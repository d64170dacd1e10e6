"""RAFT optical-flow handle: stands where the reference keeps ``DataParallel(RAFT())`` with raft-sintel.pth loaded
(models/raft/extract_raft.py:58-61, models/i3d/extract_i3d.py:104-108)."""
from __future__ import annotations

import ctypes as C
from typing import Dict

import numpy as np
import torch

from ._lib import NamedTensor, check, lib


class RAFTEngine:
    """``state_dict``: the reference checkpoint (keys with or without the ``module.`` prefix)."""

    def __init__(self, state_dict: Dict[str, torch.Tensor], device: int = 0, max_frames: int = 65, max_h: int = 272,
                 max_w: int = 480):
        if not torch.cuda.is_available():
            raise RuntimeError("RAFTEngine needs a CUDA device (sm_90a); there is no CPU fallback")
        self.device = torch.device("cuda", device)
        keep, names = [], []
        items = [(k[7:] if k.startswith("module.") else k, v) for k, v in state_dict.items()
                 if torch.is_tensor(v) and v.dtype.is_floating_point]
        arr = (NamedTensor * len(items))()
        for i, (k, v) in enumerate(items):
            a = np.ascontiguousarray(v.detach().to("cpu", torch.float32).numpy())
            nm = k.encode()
            keep.append(a); names.append(nm)
            arr[i].name = nm
            arr[i].data = a.ctypes.data_as(C.POINTER(C.c_float))
            arr[i].numel = a.size
        h = C.c_void_p()
        check(lib().vf_raft_create(C.byref(h), arr, len(items), device, max_frames, max_h, max_w))
        self._h = h
        del keep, names

    @staticmethod
    def padded_size(h: int, w: int):
        H, W = C.c_int(), C.c_int()
        check(lib().vf_raft_padded_size(h, w, C.byref(H), C.byref(W)))
        return H.value, W.value

    def flow(self, frames: torch.Tensor, iters: int = 20, unpad: bool = True) -> torch.Tensor:
        """frames: (N, 3, H, W) float in [0,255] or (N, H, W, 3) uint8, on this device, N >= 2.
        Returns (N-1, 2, H', W') fp32 == model(pad(frames)[:-1], pad(frames)[1:]) (unpadded if ``unpad``)."""
        if not frames.is_cuda:
            raise RuntimeError("RAFTEngine expects CUDA frames (no CPU fallback)")
        frames = frames.contiguous()
        if frames.dtype == torch.uint8:
            assert frames.dim() == 4 and frames.shape[3] == 3
            n, hs, ws, is_u8, chw = frames.shape[0], frames.shape[1], frames.shape[2], 1, 0
        else:
            frames = frames.to(torch.float32)
            assert frames.dim() == 4 and frames.shape[1] == 3
            n, hs, ws, is_u8, chw = frames.shape[0], frames.shape[2], frames.shape[3], 0, 1
        ho, wo = (hs, ws) if unpad else self.padded_size(hs, ws)
        out = torch.empty((n - 1, 2, ho, wo), device=frames.device, dtype=torch.float32)
        with torch.cuda.device(self.device):
            check(lib().vf_raft_flow(self._h, frames.data_ptr(), is_u8, chw, n, hs, ws, iters, int(unpad),
                                     out.data_ptr(), torch.cuda.current_stream().cuda_stream))
        return out

    def debug_read(self, what: int) -> torch.Tensor:
        dims = (C.c_int * 4)()
        check(lib().vf_raft_debug_read(self._h, what, None, 0, dims, None))
        out = torch.empty(tuple(dims), device=self.device, dtype=torch.float32)
        with torch.cuda.device(self.device):
            check(lib().vf_raft_debug_read(self._h, what, out.data_ptr(), out.numel(), dims,
                                           torch.cuda.current_stream().cuda_stream))
        return out

    @property
    def launch_count(self) -> int:
        return int(lib().vf_raft_launch_count(self._h))

    def close(self):
        if getattr(self, "_h", None):
            lib().vf_raft_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

"""ResNet frame-feature handle: stands where the reference keeps torchvision ``models.resnetXX(pretrained=True)`` with
``fc = Identity()`` in eval mode (models/resnet/extract_resnet.py:52-72)."""
from __future__ import annotations

import ctypes as C
from typing import Dict

import numpy as np
import torch

from ._lib import NamedTensor, check, lib

DEPTHS = (18, 34, 50, 101, 152)


class ResNetEngine:
    """``state_dict``: torchvision's resnet{depth} keys (with or without the ``module.`` prefix), any float dtype.
    ``max_frames``: frames per internal chunk (the workspace); larger calls are chunked inside the call."""

    def __init__(self, state_dict: Dict[str, torch.Tensor], depth: int, device: int = 0, max_frames: int = 64):
        if not torch.cuda.is_available():
            raise RuntimeError("ResNetEngine needs a CUDA device (sm_90a); there is no CPU fallback")
        self.device = torch.device("cuda", device)
        self.depth = depth
        self.out_dim = 512 if depth in (18, 34) else 2048
        keep = []
        items = [(k, v) for k, v in state_dict.items() if torch.is_tensor(v) and v.dtype.is_floating_point]
        arr = (NamedTensor * max(len(items), 1))()
        for i, (k, v) in enumerate(items):
            a = np.ascontiguousarray(v.detach().to("cpu", torch.float32).numpy())
            nm = k.encode()
            keep.append((a, nm))
            arr[i].name = nm
            arr[i].data = a.ctypes.data_as(C.POINTER(C.c_float))
            arr[i].numel = a.size
        h = C.c_void_p()
        check(lib().vf_resnet_create(C.byref(h), arr, len(items), depth, device, max_frames))
        self._h = h
        del keep

    def forward_f32(self, x: torch.Tensor) -> torch.Tensor:
        """x: (n, 3, 224, 224) fp32, already transformed, on this device -> (n, D) fp32 (``model(x)``)."""
        if not x.is_cuda:
            raise RuntimeError("ResNetEngine expects CUDA input (no CPU fallback)")
        x = x.to(torch.float32).contiguous()
        assert x.dim() == 4 and tuple(x.shape[1:]) == (3, 224, 224), x.shape
        out = torch.empty((x.shape[0], self.out_dim), device=x.device, dtype=torch.float32)
        with torch.cuda.device(self.device):
            check(lib().vf_resnet_forward_f32(self._h, x.data_ptr(), x.shape[0], out.data_ptr(),
                                              torch.cuda.current_stream().cuda_stream))
        return out

    def forward_u8(self, frames: torch.Tensor, out: torch.Tensor = None) -> torch.Tensor:
        """frames: (n, Hr, Wr, 3) uint8 BGR on this device, resized to short side 256 -> (n, D) fp32; the BGR->RGB swap,
        CenterCrop(224), ToTensor and Normalize are fused.  Asynchronous on the current stream.  ``out``: an optional
        (n, D) fp32 device tensor to write into."""
        if not frames.is_cuda:
            raise RuntimeError("ResNetEngine expects CUDA frames (no CPU fallback)")
        assert frames.dtype == torch.uint8 and frames.dim() == 4 and frames.shape[3] == 3, frames.shape
        frames = frames.contiguous()
        n, hr, wr, _ = frames.shape
        if out is None:
            out = torch.empty((n, self.out_dim), device=frames.device, dtype=torch.float32)
        assert out.is_contiguous() and tuple(out.shape) == (n, self.out_dim) and out.dtype == torch.float32
        with torch.cuda.device(self.device):
            check(lib().vf_resnet_forward_u8(self._h, frames.data_ptr(), n, hr, wr, out.data_ptr(),
                                             torch.cuda.current_stream().cuda_stream))
        return out

    def read_stage(self, stage: int) -> torch.Tensor:
        """Diagnostics: stage 0 stem, 1 maxpool, 2..5 layer1..4 of the last chunk of the last call, fp32 (n, C, H, W)."""
        dims = (C.c_int * 4)()
        check(lib().vf_resnet_read_stage(self._h, stage, None, 0, dims, None))
        out = torch.empty(tuple(dims), device=self.device, dtype=torch.float32)
        with torch.cuda.device(self.device):
            check(lib().vf_resnet_read_stage(self._h, stage, out.data_ptr(), out.numel(), dims,
                                             torch.cuda.current_stream().cuda_stream))
        return out

    @property
    def launch_count(self) -> int:
        return int(lib().vf_resnet_launch_count(self._h))

    def close(self):
        if getattr(self, "_h", None):
            lib().vf_resnet_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

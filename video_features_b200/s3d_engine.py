"""S3D clip-feature handle: torchvision ``s3d()`` in eval mode, the 1024-d ``avgpool(features(x)).mean((2, 3, 4))``,
with the ``S3D_Weights.KINETICS400_V1`` clip transform fused into the u8 entry."""
from __future__ import annotations

import ctypes as C
from typing import Dict, Sequence

import torch

from ._lib import check, debug_mixed, lib, named_tensors, read_conv

OUT_DIM = 1024
MIN_T = 13


class S3DEngine:
    """``state_dict``: torchvision's s3d keys (with or without the ``module.`` prefix), any float dtype.
    ``max_clips`` x ``max_T``: the workspace (about 1 GB per 64-frame clip); a call runs in chunks of as many clips of
    its T as the workspace holds."""

    def __init__(self, state_dict: Dict[str, torch.Tensor], device: int = 0, max_clips: int = 2, max_T: int = 64):
        if not torch.cuda.is_available():
            raise RuntimeError("S3DEngine needs a CUDA device (sm_90a); there is no CPU fallback")
        self.device = torch.device("cuda", device)
        self.out_dim = OUT_DIM
        arr, n, keep = named_tensors(state_dict)
        h = C.c_void_p()
        check(lib().vf_s3d_create(C.byref(h), arr, n, device, max_clips, max_T))
        self._h = h
        del keep

    def forward_f32(self, x: torch.Tensor) -> torch.Tensor:
        """x: (n, 3, T, 224, 224) fp32, already transformed, T >= 13, on this device -> (n, 1024) fp32."""
        if not x.is_cuda:
            raise RuntimeError("S3DEngine expects CUDA input (no CPU fallback)")
        x = x.to(torch.float32).contiguous()
        assert x.dim() == 5 and x.shape[1] == 3 and tuple(x.shape[3:]) == (224, 224), x.shape
        out = torch.empty((x.shape[0], self.out_dim), device=x.device, dtype=torch.float32)
        with torch.cuda.device(self.device):
            check(lib().vf_s3d_forward_f32(self._h, x.data_ptr(), x.shape[0], x.shape[2], out.data_ptr(),
                                            torch.cuda.current_stream().cuda_stream))
        return out

    def forward_u8(self, frames: torch.Tensor, starts: Sequence[int], T: int, out: torch.Tensor = None) -> torch.Tensor:
        """frames: (F, H, W, 3) uint8 BGR decoded frames of any size on this device; clip i is frames
        ``starts[i] .. starts[i] + T - 1`` -> (len(starts), 1024) fp32.  The BGR->RGB swap, Resize((256, 256)) on uint8,
        CenterCrop(224), /255 and Normalize are fused.  Asynchronous on the current stream.  ``out``: an optional
        (len(starts), 1024) fp32 device tensor to write into."""
        if not frames.is_cuda:
            raise RuntimeError("S3DEngine expects CUDA frames (no CPU fallback)")
        assert frames.dtype == torch.uint8 and frames.dim() == 4 and frames.shape[3] == 3, frames.shape
        frames = frames.contiguous()
        nf, hh, ww, _ = frames.shape
        n = len(starts)
        st = (C.c_int * max(n, 1))(*[int(s) for s in starts])
        if out is None:
            out = torch.empty((n, self.out_dim), device=frames.device, dtype=torch.float32)
        assert out.is_contiguous() and tuple(out.shape) == (n, self.out_dim) and out.dtype == torch.float32
        with torch.cuda.device(self.device):
            check(lib().vf_s3d_forward_u8(self._h, frames.data_ptr(), nf, hh, ww, st, n, T, out.data_ptr(),
                                           torch.cuda.current_stream().cuda_stream))
        return out

    def read_stage(self, stage: int) -> torch.Tensor:
        """Diagnostics: stage 0 stem, 1 features.3, 2 Mixed 3c, 3 Mixed 4f, 4 Mixed 5c of the last chunk of the last
        call, fp32 (n, C, T, H, W)."""
        dims = (C.c_int * 5)()
        check(lib().vf_s3d_read_stage(self._h, stage, None, 0, dims, None))
        out = torch.empty(tuple(dims), device=self.device, dtype=torch.float32)
        with torch.cuda.device(self.device):
            check(lib().vf_s3d_read_stage(self._h, stage, out.data_ptr(), out.numel(), dims,
                                           torch.cuda.current_stream().cuda_stream))
        return out

    def conv(self, index: int) -> dict:
        """Diagnostics: conv ``index`` as uploaded, in execution order (include/vfeat.h vf_s3d_conv); see _lib.read_conv."""
        with torch.cuda.device(self.device):
            return read_conv(lib().vf_s3d_conv, self._h, index, self.device)

    def debug_mixed(self, block: int, x: torch.Tensor) -> torch.Tensor:
        """Diagnostics: Mixed block ``block`` (0 .. 8: features.5, 6, 8 .. 12, 14, 15) on the fp16 pair volume x
        (n, T + 2, S + 2, S + 2, 2 cin), S = 28 / 14 / 7, zero border -> its concat pair volume (n, T + 2, S + 2, S + 2,
        2 ctot) (include/vfeat.h vf_s3d_debug_mixed).  read_stage then fails until the next forward."""
        return debug_mixed(lib().vf_s3d_debug_mixed, self._h, block, x, self.device)

    @property
    def launch_count(self) -> int:
        return int(lib().vf_s3d_launch_count(self._h))

    def close(self):
        if getattr(self, "_h", None):
            lib().vf_s3d_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

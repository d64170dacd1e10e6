"""R(2+1)D clip-feature handle: stands where the reference keeps torchvision ``r2plus1d_18(pretrained=True)`` with
``fc = Identity()`` in eval mode (models/r21d/extract_r21d.py), and runs the IG65M R(2+1)D-34 models on the same
engine."""
from __future__ import annotations

import ctypes as C
from typing import Dict, Sequence

import torch

from ._lib import check, lib, named_tensors, read_conv

OUT_DIM = 512


class R21DEngine:
    """``state_dict``: torchvision's VideoResNet keys (with or without the ``module.`` prefix), any float dtype; the
    depth, the mid widths and the downsamples are read from it (r2plus1d_18, or R(2+1)D-34 with 3, 4, 6, 3 blocks).
    ``bn_eps``: every BatchNorm's eps (1e-5 for r2plus1d_18, 1e-3 for the IG65M R(2+1)D-34 models).
    ``max_clips`` x ``max_T``: the workspace; a call of T-frame clips runs in chunks of
    max_clips * (max_T + 2) // (T + 2) clips inside the call."""

    def __init__(self, state_dict: Dict[str, torch.Tensor], device: int = 0, max_clips: int = 4, max_T: int = 16,
                 bn_eps: float = 1e-5):
        if not torch.cuda.is_available():
            raise RuntimeError("R21DEngine needs a CUDA device (sm_90a); there is no CPU fallback")
        self.device = torch.device("cuda", device)
        self.out_dim = OUT_DIM
        arr, n, keep = named_tensors(state_dict)
        h = C.c_void_p()
        check(lib().vf_r21d_create2(C.byref(h), arr, n, device, max_clips, max_T, float(bn_eps)))
        self._h = h
        del keep

    def forward_f32(self, x: torch.Tensor) -> torch.Tensor:
        """x: (n, 3, T, 112, 112) fp32, already transformed, on this device -> (n, 512) fp32 (``model(x)``)."""
        if not x.is_cuda:
            raise RuntimeError("R21DEngine expects CUDA input (no CPU fallback)")
        x = x.to(torch.float32).contiguous()
        assert x.dim() == 5 and x.shape[1] == 3 and tuple(x.shape[3:]) == (112, 112), x.shape
        out = torch.empty((x.shape[0], self.out_dim), device=x.device, dtype=torch.float32)
        with torch.cuda.device(self.device):
            check(lib().vf_r21d_forward_f32(self._h, x.data_ptr(), x.shape[0], x.shape[2], out.data_ptr(),
                                            torch.cuda.current_stream().cuda_stream))
        return out

    def forward_u8(self, frames: torch.Tensor, starts: Sequence[int], T: int, out: torch.Tensor = None) -> torch.Tensor:
        """frames: (F, H, W, 3) uint8 BGR decoded frames of any size on this device; clip i is frames
        ``starts[i] .. starts[i] + T - 1`` -> (len(starts), 512) fp32.  The BGR->RGB swap, /255, Resize((128, 171)),
        Normalize and CenterCrop(112) are fused.  Asynchronous on the current stream.  ``out``: an optional
        (len(starts), 512) fp32 device tensor to write into."""
        if not frames.is_cuda:
            raise RuntimeError("R21DEngine expects CUDA frames (no CPU fallback)")
        assert frames.dtype == torch.uint8 and frames.dim() == 4 and frames.shape[3] == 3, frames.shape
        frames = frames.contiguous()
        nf, hh, ww, _ = frames.shape
        n = len(starts)
        st = (C.c_int * max(n, 1))(*[int(s) for s in starts])
        if out is None:
            out = torch.empty((n, self.out_dim), device=frames.device, dtype=torch.float32)
        assert out.is_contiguous() and tuple(out.shape) == (n, self.out_dim) and out.dtype == torch.float32
        with torch.cuda.device(self.device):
            check(lib().vf_r21d_forward_u8(self._h, frames.data_ptr(), nf, hh, ww, st, n, T, out.data_ptr(),
                                           torch.cuda.current_stream().cuda_stream))
        return out

    def read_stage(self, stage: int) -> torch.Tensor:
        """Diagnostics: stage 0 stem, 1..4 layer1..4 of the last chunk of the last call, fp32 (n, C, T, H, W)."""
        dims = (C.c_int * 5)()
        check(lib().vf_r21d_read_stage(self._h, stage, None, 0, dims, None))
        out = torch.empty(tuple(dims), device=self.device, dtype=torch.float32)
        with torch.cuda.device(self.device):
            check(lib().vf_r21d_read_stage(self._h, stage, out.data_ptr(), out.numel(), dims,
                                           torch.cuda.current_stream().cuda_stream))
        return out

    def conv(self, index: int) -> dict:
        """Diagnostics: conv ``index`` as uploaded, in execution order (include/vfeat.h vf_r21d_conv); see _lib.read_conv."""
        with torch.cuda.device(self.device):
            return read_conv(lib().vf_r21d_conv, self._h, index, self.device)

    @property
    def launch_count(self) -> int:
        return int(lib().vf_r21d_launch_count(self._h))

    def close(self):
        if getattr(self, "_h", None):
            lib().vf_r21d_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

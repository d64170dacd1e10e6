"""Swin3D clip-feature handle: torchvision ``swin3d_t`` / ``swin3d_s`` / ``swin3d_b`` in eval mode, the feature
``flatten(avgpool(norm(features(patch_embed(x)))))``, with the ``Swin3D_*_Weights.KINETICS400_V1`` clip transform fused
into the u8 entry."""
from __future__ import annotations

import ctypes as C
from typing import Dict, Sequence

import torch

from ._lib import check, lib, named_tensors

STAGES = ("embed", "stage1", "stage2", "stage3", "stage4", "norm")     # read_stage ids 0..5


class Swin3DEngine:
    """``state_dict``: torchvision's swin3d keys (with or without the ``module.`` prefix), any float dtype; the shape
    (t, s or b) is read from it.  ``max_clips`` x ``max_T``: the workspace, 192 + 34 C bytes per stage-1 row (C the embed
    dim) and 16 x 3136 such rows per 32-frame clip: about 173 MB per clip for t / s, 228 MB for b; a call runs in chunks
    of as many clips of its T as the workspace holds."""

    def __init__(self, state_dict: Dict[str, torch.Tensor], device: int = 0, max_clips: int = 4, max_T: int = 32):
        if not torch.cuda.is_available():
            raise RuntimeError("Swin3DEngine needs a CUDA device (sm_90a); there is no CPU fallback")
        self.device = torch.device("cuda", device)
        arr, n, keep = named_tensors(state_dict)
        h = C.c_void_p()
        check(lib().vf_swin3d_create(C.byref(h), arr, n, device, max_clips, max_T))
        self._h = h
        del keep
        info = (C.c_int * 8)()
        check(lib().vf_swin3d_info(self._h, info))
        self.out_dim, self.embed_dim, self.depths = info[0], info[1], tuple(info[2:6])

    def forward_f32(self, x: torch.Tensor) -> torch.Tensor:
        """x: (n, 3, T, 224, 224) fp32, already transformed, on this device -> (n, out_dim) fp32."""
        if not x.is_cuda:
            raise RuntimeError("Swin3DEngine expects CUDA input (no CPU fallback)")
        x = x.to(torch.float32).contiguous()
        assert x.dim() == 5 and x.shape[1] == 3 and tuple(x.shape[3:]) == (224, 224), x.shape
        out = torch.empty((x.shape[0], self.out_dim), device=x.device, dtype=torch.float32)
        with torch.cuda.device(self.device):
            check(lib().vf_swin3d_forward_f32(self._h, x.data_ptr(), x.shape[0], x.shape[2], out.data_ptr(),
                                               torch.cuda.current_stream().cuda_stream))
        return out

    def forward_u8(self, frames: torch.Tensor, starts: Sequence[int], T: int, out: torch.Tensor = None) -> torch.Tensor:
        """frames: (F, H, W, 3) uint8 BGR decoded frames of any size on this device; clip i is frames
        ``starts[i] .. starts[i] + T - 1`` -> (len(starts), out_dim) fp32.  The BGR->RGB swap, Resize([256]) on uint8,
        CenterCrop(224), /255 and Normalize are fused.  Asynchronous on the current stream.  ``out``: an optional
        (len(starts), out_dim) fp32 device tensor to write into."""
        if not frames.is_cuda:
            raise RuntimeError("Swin3DEngine expects CUDA frames (no CPU fallback)")
        assert frames.dtype == torch.uint8 and frames.dim() == 4 and frames.shape[3] == 3, frames.shape
        frames = frames.contiguous()
        nf, hh, ww, _ = frames.shape
        n = len(starts)
        st = (C.c_int * max(n, 1))(*[int(s) for s in starts])
        if out is None:
            out = torch.empty((n, self.out_dim), device=frames.device, dtype=torch.float32)
        assert out.is_contiguous() and tuple(out.shape) == (n, self.out_dim) and out.dtype == torch.float32
        with torch.cuda.device(self.device):
            check(lib().vf_swin3d_forward_u8(self._h, frames.data_ptr(), nf, hh, ww, st, n, T, out.data_ptr(),
                                              torch.cuda.current_stream().cuda_stream))
        return out

    def read_stage(self, stage: int) -> torch.Tensor:
        """Diagnostics: STAGES[stage] of the last chunk of the last call, fp32 (n, T', H', W', C)."""
        dims = (C.c_int * 5)()
        check(lib().vf_swin3d_read_stage(self._h, stage, None, 0, dims, None))
        out = torch.empty(tuple(dims), device=self.device, dtype=torch.float32)
        with torch.cuda.device(self.device):
            check(lib().vf_swin3d_read_stage(self._h, stage, out.data_ptr(), out.numel(), dims,
                                              torch.cuda.current_stream().cuda_stream))
        return out

    @property
    def launch_count(self) -> int:
        return int(lib().vf_swin3d_launch_count(self._h))

    def close(self):
        if getattr(self, "_h", None):
            lib().vf_swin3d_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def window_attention(qkv: torch.Tensor, bias_qkv: torch.Tensor, table: torch.Tensor, shifted: bool) -> torch.Tensor:
    """Diagnostics: the engine's window attention alone (include/vfeat.h vf_swin3d_attention).  qkv: (n, T', H, W, 3C)
    fp16, bias_qkv: (3C,) fp32, table: (2535, C / 32) fp32, all on one device -> (n, T', H, W, C) fp16."""
    assert qkv.is_cuda and qkv.dtype == torch.float16 and qkv.dim() == 5 and qkv.shape[-1] % 96 == 0, qkv.shape
    n, tq, hh, ww, c3 = qkv.shape
    c = c3 // 3
    qkv = qkv.contiguous()
    bias_qkv = bias_qkv.to(qkv.device, torch.float32).contiguous()
    table = table.to(qkv.device, torch.float32).contiguous()
    assert bias_qkv.numel() == c3 and tuple(table.shape) == (2535, c // 32), (bias_qkv.shape, table.shape)
    out = torch.empty((n, tq, hh, ww, c), device=qkv.device, dtype=torch.float16)
    with torch.cuda.device(qkv.device):
        check(lib().vf_swin3d_attention(qkv.data_ptr(), bias_qkv.data_ptr(), table.data_ptr(), n, tq, hh, ww, c,
                                         int(shifted), out.data_ptr(), torch.cuda.current_stream().cuda_stream))
    return out

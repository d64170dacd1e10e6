"""MViT clip-feature handle: torchvision ``mvit_v1_b`` / ``mvit_v2_s`` in eval mode, the feature ``norm(x)[:, 0]`` (the
class token after the final norm), with the ``MViT_*_Weights.KINETICS400_V1`` clip transform fused into the u8 entry."""
from __future__ import annotations

import ctypes as C
from typing import Dict, Sequence

import torch

from ._lib import check, lib, named_tensors

STAGES = ("embed", "stage1", "stage2", "stage3", "stage4", "norm")     # read_stage ids 0..5
T = 16                                                                 # fixed by the position tables


class MViTEngine:
    """``state_dict``: torchvision's mvit_v1_b / mvit_v2_s keys (with or without the ``module.`` prefix), any float
    dtype; the variant is read from it.  ``max_clips``: the workspace, about 190 MB per 16-frame clip; a call runs in
    chunks of as many clips as it holds."""

    def __init__(self, state_dict: Dict[str, torch.Tensor], device: int = 0, max_clips: int = 4):
        if not torch.cuda.is_available():
            raise RuntimeError("MViTEngine needs a CUDA device (sm_90a); there is no CPU fallback")
        self.device = torch.device("cuda", device)
        arr, n, keep = named_tensors(state_dict)
        h = C.c_void_p()
        check(lib().vf_mvit_create(C.byref(h), arr, n, device, max_clips))
        self._h = h
        del keep
        info = (C.c_int * 4)()
        check(lib().vf_mvit_info(self._h, info))
        self.out_dim, self.version, self.T, self.max_clips = info[0], info[1], info[2], info[3]
        self.name = "mvit_v1_b" if self.version == 1 else "mvit_v2_s"

    def forward_f32(self, x: torch.Tensor) -> torch.Tensor:
        """x: (n, 3, 16, 224, 224) fp32, already transformed, on this device -> (n, 768) fp32."""
        if not x.is_cuda:
            raise RuntimeError("MViTEngine expects CUDA input (no CPU fallback)")
        x = x.to(torch.float32).contiguous()
        assert x.dim() == 5 and x.shape[1] == 3 and tuple(x.shape[3:]) == (224, 224), x.shape
        out = torch.empty((x.shape[0], self.out_dim), device=x.device, dtype=torch.float32)
        with torch.cuda.device(self.device):
            check(lib().vf_mvit_forward_f32(self._h, x.data_ptr(), x.shape[0], x.shape[2], out.data_ptr(),
                                             torch.cuda.current_stream().cuda_stream))
        return out

    def forward_u8(self, frames: torch.Tensor, starts: Sequence[int], T: int = T, out: torch.Tensor = None) -> torch.Tensor:
        """frames: (F, H, W, 3) uint8 BGR decoded frames of any size on this device; clip i is frames
        ``starts[i] .. starts[i] + 15`` -> (len(starts), 768) fp32.  The BGR->RGB swap, Resize([256]) on uint8,
        CenterCrop(224), /255 and Normalize(0.45, 0.225) are fused.  Asynchronous on the current stream.  ``out``: an
        optional (len(starts), 768) fp32 device tensor to write into."""
        if not frames.is_cuda:
            raise RuntimeError("MViTEngine expects CUDA frames (no CPU fallback)")
        assert frames.dtype == torch.uint8 and frames.dim() == 4 and frames.shape[3] == 3, frames.shape
        frames = frames.contiguous()
        nf, hh, ww, _ = frames.shape
        n = len(starts)
        st = (C.c_int * max(n, 1))(*[int(s) for s in starts])
        if out is None:
            out = torch.empty((n, self.out_dim), device=frames.device, dtype=torch.float32)
        assert out.is_contiguous() and tuple(out.shape) == (n, self.out_dim) and out.dtype == torch.float32
        with torch.cuda.device(self.device):
            check(lib().vf_mvit_forward_u8(self._h, frames.data_ptr(), nf, hh, ww, st, n, T, out.data_ptr(),
                                            torch.cuda.current_stream().cuda_stream))
        return out

    def read_stage(self, stage: int) -> torch.Tensor:
        """Diagnostics: STAGES[stage] of the last chunk of the last call, fp32 (n, tokens, C), class token first."""
        dims = (C.c_int * 3)()
        check(lib().vf_mvit_read_stage(self._h, stage, None, 0, dims, None))
        out = torch.empty(tuple(dims), device=self.device, dtype=torch.float32)
        with torch.cuda.device(self.device):
            check(lib().vf_mvit_read_stage(self._h, stage, out.data_ptr(), out.numel(), dims,
                                            torch.cuda.current_stream().cuda_stream))
        return out

    @property
    def launch_count(self) -> int:
        return int(lib().vf_mvit_launch_count(self._h))

    def close(self):
        if getattr(self, "_h", None):
            lib().vf_mvit_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def _thw(n_rows: int, thw: Sequence[int]):
    assert len(thw) == 3 and 1 + thw[0] * thw[1] * thw[2] == n_rows, (n_rows, thw)
    return (C.c_int * 3)(*[int(v) for v in thw])


def pool_attention(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, q_thw, k_thw, rel=None,
                   resid: bool = False) -> torch.Tensor:
    """Diagnostics: the engine's pooling attention alone (include/vfeat.h vf_mvit_attention).  q: (n, 1 + Nq, heads * 96)
    fp16 (any row pitch: a column slice of the qkv rows is fine), k / v: (n, 1 + Nk, heads * 96) fp16, all on one
    device; rel: (rel_h, rel_w, rel_t) fp32 tables of torchvision's sizes, or None -> (n, 1 + Nq, heads * 96) fp16."""
    assert q.is_cuda and q.dtype == k.dtype == v.dtype == torch.float16 and q.dim() == k.dim() == 3
    n, nq, c = q.shape
    assert c % 96 == 0 and q.stride(2) == 1 and q.stride(0) == nq * q.stride(1), q.stride()
    k, v = k.contiguous(), v.contiguous()
    assert k.shape == v.shape and k.shape[0] == n and k.shape[2] == c, (k.shape, v.shape)
    qa, ka = _thw(nq, q_thw), _thw(k.shape[1], k_thw)
    ptrs = [None, None, None]
    keep = []
    if rel is not None:
        for i, (tab, a, b) in enumerate(zip(rel, (q_thw[1], q_thw[2], q_thw[0]), (k_thw[1], k_thw[2], k_thw[0]))):
            tab = tab.to(q.device, torch.float32).contiguous()
            assert tuple(tab.shape) == (2 * max(a, b) - 1, 96), tab.shape
            keep.append(tab)
            ptrs[i] = tab.data_ptr()
    out = torch.empty((n, nq, c), device=q.device, dtype=torch.float16)
    with torch.cuda.device(q.device):
        check(lib().vf_mvit_attention(q.data_ptr(), q.stride(1), k.data_ptr(), v.data_ptr(), ptrs[0], ptrs[1], ptrs[2],
                                       n, c // 96, qa, ka, int(rel is not None), int(resid), out.data_ptr(),
                                       torch.cuda.current_stream().cuda_stream))
    return out


def head_pool(src: torch.Tensor, thw, stride: int, weight: torch.Tensor, gamma: torch.Tensor,
              beta: torch.Tensor) -> torch.Tensor:
    """Diagnostics: the engine's head pooling alone (vf_mvit_head_pool).  src: (n, 1 + T H W, heads * 96) fp16 (any row
    pitch), weight: (96, 1, 3, 3, 3), gamma / beta: (96,) -> (n, 1 + T Ho Wo, heads * 96) fp16."""
    assert src.is_cuda and src.dtype == torch.float16 and src.dim() == 3 and src.stride(2) == 1
    n, rows, c = src.shape
    assert c % 96 == 0 and src.stride(0) == rows * src.stride(1), src.stride()
    _thw(rows, thw)
    w = weight.to(src.device, torch.float32).contiguous()
    gm, bt = gamma.to(src.device, torch.float32).contiguous(), beta.to(src.device, torch.float32).contiguous()
    assert w.numel() == 96 * 27 and gm.numel() == bt.numel() == 96
    ho, wo = (thw[1] - 1) // stride + 1, (thw[2] - 1) // stride + 1
    out = torch.empty((n, 1 + thw[0] * ho * wo, c), device=src.device, dtype=torch.float16)
    with torch.cuda.device(src.device):
        check(lib().vf_mvit_head_pool(src.data_ptr(), src.stride(1), n, c // 96, thw[0], thw[1], thw[2], stride,
                                       w.data_ptr(), gm.data_ptr(), bt.data_ptr(), out.data_ptr(),
                                       torch.cuda.current_stream().cuda_stream))
    return out


def skip_pool(x: torch.Tensor, thw) -> torch.Tensor:
    """Diagnostics: the engine's skip max-pool alone (vf_mvit_skip_pool).  x: (n, 1 + T H W, C) fp32 ->
    (n, 1 + T Ho Wo, C) fp32."""
    assert x.is_cuda and x.dtype == torch.float32 and x.dim() == 3
    x = x.contiguous()
    n, rows, c = x.shape
    _thw(rows, thw)
    out = torch.empty((n, 1 + thw[0] * ((thw[1] - 1) // 2 + 1) * ((thw[2] - 1) // 2 + 1), c), device=x.device,
                      dtype=torch.float32)
    with torch.cuda.device(x.device):
        check(lib().vf_mvit_skip_pool(x.data_ptr(), n, c, thw[0], thw[1], thw[2], out.data_ptr(),
                                       torch.cuda.current_stream().cuda_stream))
    return out

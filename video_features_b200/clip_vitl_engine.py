"""CLIP ViT-L/14 image tower handle (``CLIP-ViT-L/14`` at 224 px, ``CLIP-ViT-L/14@336px``): stands where the reference
would keep the result of ``clip.load("ViT-L/14" | "ViT-L/14@336px", device)``, ``preprocess`` and ``encode_image``
included.  It offers the methods ``ExtractCLIP`` calls on its model."""
from __future__ import annotations

import ctypes as C
from typing import Dict, Optional

import numpy as np
import torch

from ._lib import check, lib, named_tensors

LAYERS = 24


class ClipViTLEngine:
    """``state_dict``: openai's ``visual.*`` keys (a full CLIP state dict or a JIT archive's ``state_dict()``; other keys
    are ignored), any float dtype.  The configuration is inferred from the sizes.  ``max_frames``: frames per internal
    chunk (0: the tower's default, about 2.5 GB of workspace); larger calls are chunked inside the call."""

    def __init__(self, state_dict: Dict[str, torch.Tensor], device: int = 0, max_frames: int = 0):
        if not torch.cuda.is_available():
            raise RuntimeError("ClipViTLEngine needs a CUDA device (sm_90a); there is no CPU fallback")
        self.device = torch.device("cuda", device)
        arr, n, keep = named_tensors({k: v for k, v in state_dict.items() if k.startswith("visual.")})
        h = C.c_void_p()
        check(lib().vf_clip_vitl_create(C.byref(h), arr, n, device, max_frames))
        self._h = h
        del keep
        info = (C.c_int * 8)()
        check(lib().vf_clip_vitl_info(self._h, info))
        (self.out_dim, self.n_px, self.width, self.layers, self.heads, self.patch, self.tokens,
         self.max_frames) = list(info)
        self._events = {}
        self._next_ticket = 0

    def _stream(self) -> int:
        return torch.cuda.current_stream(self.device).cuda_stream

    def _out(self, n: int, out: Optional[torch.Tensor]) -> torch.Tensor:
        if out is None:
            return torch.empty((n, self.out_dim), device=self.device, dtype=torch.float32)
        assert out.is_cuda and out.is_contiguous() and tuple(out.shape) == (n, self.out_dim) and out.dtype == torch.float32
        return out

    def encode_image(self, frames: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """frames: (n, 3, n_px, n_px), already transformed, on this device -> (n, 768) fp32 on this device."""
        if not frames.is_cuda:
            raise RuntimeError("ClipViTLEngine expects CUDA input (no CPU fallback)")
        frames = frames.to(torch.float32).contiguous()
        assert frames.dim() == 4 and tuple(frames.shape[1:]) == (3, self.n_px, self.n_px), frames.shape
        n = frames.shape[0]
        out = self._out(n, out)
        with torch.cuda.device(self.device):
            check(lib().vf_clip_vitl_encode_f32(self._h, frames.data_ptr(), n, out.data_ptr(), self._stream()))
        return out

    def encode_frames_u8(self, frames: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """frames: (n, H, W, 3) uint8 on this device, any size, decoder channel order -> (n, 768) fp32 on this device;
        the bicubic resize, centre crop and normalisation are fused.  Asynchronous on the current stream."""
        if not frames.is_cuda:
            raise RuntimeError("ClipViTLEngine expects CUDA frames (no CPU fallback)")
        assert frames.dtype == torch.uint8 and frames.dim() == 4 and frames.shape[3] == 3, frames.shape
        frames = frames.contiguous()
        n, hh, ww, _ = frames.shape
        out = self._out(n, out)
        with torch.cuda.device(self.device):
            check(lib().vf_clip_vitl_encode_u8(self._h, frames.data_ptr(), n, hh, ww, out.data_ptr(), self._stream()))
        return out

    def encode_frames_u8_host(self, frames, out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Host uint8 frames (numpy or CPU tensor, (n, H, W, 3)) -> (n, 768) fp32 on the host, synchronous."""
        if isinstance(frames, np.ndarray):
            frames = torch.from_numpy(np.ascontiguousarray(frames))
        assert (not frames.is_cuda) and frames.dtype == torch.uint8 and frames.dim() == 4 and frames.shape[3] == 3
        with torch.cuda.device(self.device):
            dev = self.encode_frames_u8(frames.contiguous().to(self.device))
            if out is None:
                return dev.cpu()
            out.copy_(dev)
        return out

    def encode_frames_u8_host_async(self, frames: torch.Tensor, out_host: Optional[torch.Tensor] = None,
                                    out_dev: bool = False):
        """Pinned host frames in; features to ``out_host`` (pinned) and / or a new device tensor (``out_dev=True``).
        Returns ``(ticket, device tensor or None)``; ``frames`` and ``out_host`` belong to the engine until
        ``wait(ticket)``.  The copies and the tower are enqueued on the current stream."""
        assert (not frames.is_cuda) and frames.dtype == torch.uint8 and frames.dim() == 4 and frames.shape[3] == 3
        assert frames.is_contiguous() and frames.is_pinned(), "asynchronous calls need pinned, contiguous host frames"
        n = frames.shape[0]
        if out_host is not None:
            assert out_host.dtype == torch.float32 and out_host.is_contiguous() and tuple(out_host.shape) == (n, self.out_dim)
            assert out_host.is_pinned(), "asynchronous calls need a pinned host output"
        assert out_host is not None or out_dev
        with torch.cuda.device(self.device):
            dev = self.encode_frames_u8(frames.to(self.device, non_blocking=True))
            if out_host is not None:
                out_host.copy_(dev, non_blocking=True)
            ev = torch.cuda.Event()
            ev.record()
        ticket = self._next_ticket
        self._next_ticket += 1
        self._events[ticket] = ev
        return ticket, (dev if out_dev else None)

    def wait(self, ticket: int) -> None:
        """Block until the asynchronous call `ticket` has finished with its host buffers."""
        self._events.pop(int(ticket)).synchronize()

    # ---- diagnostics: the tower's pieces one at a time (n <= max_frames), eager, on the current stream
    def debug_embed(self, frames: torch.Tensor) -> torch.Tensor:
        """Patch embedding, tokens and ln_pre -> (n, tokens, 1024) fp32.  frames: fp32 (n, 3, n_px, n_px) transformed,
        or uint8 (n, H, W, 3) through the fused transform."""
        assert frames.is_cuda
        frames = frames.contiguous()
        n = frames.shape[0]
        x = torch.empty((n, self.tokens, self.width), device=self.device, dtype=torch.float32)
        with torch.cuda.device(self.device):
            if frames.dtype == torch.uint8:
                check(lib().vf_clip_vitl_debug_embed_u8(self._h, frames.data_ptr(), n, frames.shape[1], frames.shape[2],
                                                        x.data_ptr(), self._stream()))
            else:
                assert frames.dtype == torch.float32 and tuple(frames.shape[1:]) == (3, self.n_px, self.n_px)
                check(lib().vf_clip_vitl_debug_embed_f32(self._h, frames.data_ptr(), n, x.data_ptr(), self._stream()))
        return x

    def debug_blocks(self, x: torch.Tensor, begin: int, end: int) -> torch.Tensor:
        """Resblocks [begin, end) on a copy of the residual stream x (n, tokens, 1024) fp32.  Block 23 updates the class
        rows only."""
        y = x.to(torch.float32).contiguous().clone()
        with torch.cuda.device(self.device):
            check(lib().vf_clip_vitl_debug_blocks(self._h, y.data_ptr(), y.shape[0], begin, end, self._stream()))
        return y

    def debug_head(self, x: torch.Tensor) -> torch.Tensor:
        """ln_post + proj on the class rows of x (n, tokens, 1024) fp32 -> (n, 768)."""
        x = x.to(torch.float32).contiguous()
        out = torch.empty((x.shape[0], self.out_dim), device=self.device, dtype=torch.float32)
        with torch.cuda.device(self.device):
            check(lib().vf_clip_vitl_debug_head(self._h, x.data_ptr(), x.shape[0], out.data_ptr(), self._stream()))
        return out

    def attention(self, qkv: torch.Tensor) -> torch.Tensor:
        """The tower's attention kernel on caller rows: qkv (n, S, 3072) fp16, q | k | v after the bias, S <= 577 ->
        (n, S, 1024) fp16."""
        assert qkv.is_cuda and qkv.dtype == torch.float16 and qkv.dim() == 3 and qkv.shape[2] == 3 * self.width
        qkv = qkv.contiguous()
        n, s, _ = qkv.shape
        out = torch.empty((n, s, self.width), device=self.device, dtype=torch.float16)
        with torch.cuda.device(self.device):
            check(lib().vf_clip_vitl_attention(self._h, qkv.data_ptr(), n, s, out.data_ptr(), self._stream()))
        return out

    @property
    def launch_count(self) -> int:
        return int(lib().vf_clip_vitl_launch_count(self._h))

    def close(self):
        if getattr(self, "_h", None):
            lib().vf_clip_vitl_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

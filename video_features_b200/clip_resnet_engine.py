"""CLIP ResNet image tower handle (RN50, RN101, RN50x4, RN50x16): stands where the reference keeps the result of
``clip.load("RN50" | "RN101" | "RN50x4" | "RN50x16", device)`` (models/CLIP/extract_clip.py:45-64), ``preprocess`` and
``encode_image`` included.  It offers the methods ``ExtractCLIP`` calls on its model."""
from __future__ import annotations

import ctypes as C
from typing import Dict, Optional

import numpy as np
import torch

from ._lib import check, lib, named_tensors, read_conv

STAGES = ("stem", "layer1", "layer2", "layer3", "layer4", "tokens", "pre_cproj")     # vf_clip_rn_read_stage ids


class ClipResNetEngine:
    """``state_dict``: openai's ``visual.*`` keys (a full CLIP state dict or a JIT archive's ``state_dict()``; other keys
    are ignored), any float dtype.  The configuration is inferred from the sizes.  ``max_frames``: frames per internal
    chunk (0: the tower's default); larger calls are chunked inside the call."""

    def __init__(self, state_dict: Dict[str, torch.Tensor], device: int = 0, max_frames: int = 0):
        if not torch.cuda.is_available():
            raise RuntimeError("ClipResNetEngine needs a CUDA device (sm_90a); there is no CPU fallback")
        self.device = torch.device("cuda", device)
        arr, n, keep = named_tensors({k: v for k, v in state_dict.items() if k.startswith("visual.")})
        h = C.c_void_p()
        check(lib().vf_clip_rn_create(C.byref(h), arr, n, device, max_frames))
        self._h = h
        del keep
        info = (C.c_int * 11)()
        check(lib().vf_clip_rn_info(self._h, info))
        (self.out_dim, self.n_px, self.width, self.embed, self.heads, self.tokens,
         self.max_frames) = list(info)[:7]
        self.layers = tuple(info[7:11])
        self._events = {}
        self._next_ticket = 0

    def _stream(self) -> int:
        return torch.cuda.current_stream(self.device).cuda_stream

    def encode_image(self, frames: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """frames: (n, 3, n_px, n_px), already transformed, on this device -> (n, out_dim) fp32 on this device."""
        if not frames.is_cuda:
            raise RuntimeError("ClipResNetEngine expects CUDA input (no CPU fallback)")
        frames = frames.to(torch.float32).contiguous()
        assert frames.dim() == 4 and tuple(frames.shape[1:]) == (3, self.n_px, self.n_px), frames.shape
        n = frames.shape[0]
        if out is None:
            out = torch.empty((n, self.out_dim), device=self.device, dtype=torch.float32)
        with torch.cuda.device(self.device):
            check(lib().vf_clip_rn_encode_f32(self._h, frames.data_ptr(), n, out.data_ptr(), self._stream()))
        return out

    def encode_frames_u8(self, frames: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """frames: (n, H, W, 3) uint8 on this device, any size, decoder channel order -> (n, out_dim) fp32 on this
        device; the bicubic resize, centre crop and normalisation are fused.  Asynchronous on the current stream."""
        if not frames.is_cuda:
            raise RuntimeError("ClipResNetEngine expects CUDA frames (no CPU fallback)")
        assert frames.dtype == torch.uint8 and frames.dim() == 4 and frames.shape[3] == 3, frames.shape
        frames = frames.contiguous()
        n, hh, ww, _ = frames.shape
        if out is None:
            out = torch.empty((n, self.out_dim), device=self.device, dtype=torch.float32)
        assert out.is_cuda and out.is_contiguous() and tuple(out.shape) == (n, self.out_dim) and out.dtype == torch.float32
        with torch.cuda.device(self.device):
            check(lib().vf_clip_rn_encode_u8(self._h, frames.data_ptr(), n, hh, ww, out.data_ptr(), self._stream()))
        return out

    def encode_frames_u8_host(self, frames, out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Host uint8 frames (numpy or CPU tensor, (n, H, W, 3)) -> (n, out_dim) fp32 on the host, synchronous."""
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

    def read_stage(self, stage: int) -> torch.Tensor:
        """Diagnostics: of the last chunk of the last call, fp32: 0 stem, 1..4 layer1..4 (n, C, H, W), 5 the
        attention-pool tokens (n, T, E), 6 the attention output before c_proj (n, E)."""
        dims = (C.c_int * 4)()
        check(lib().vf_clip_rn_read_stage(self._h, stage, None, 0, dims, None))
        out = torch.empty(tuple(dims), device=self.device, dtype=torch.float32)
        with torch.cuda.device(self.device):
            check(lib().vf_clip_rn_read_stage(self._h, stage, out.data_ptr(), out.numel(), dims, self._stream()))
        if stage == 5:
            return out[..., 0].transpose(1, 2).contiguous()
        if stage == 6:
            return out[:, :, 0, 0]
        return out

    def read_pairs(self, stage: int) -> torch.Tensor:
        """Diagnostics: stage 0 .. 4 of read_stage as held, the pair volume (n, S + 2, S + 2, 2C) fp16, border
        included (the form debug_block takes)."""
        dims = (C.c_int * 4)()
        check(lib().vf_clip_rn_read_stage(self._h, stage, None, 0, dims, None))
        if not 0 <= stage <= 4:
            raise ValueError(f"stage {stage}: read_pairs takes 0 .. 4")
        n, c, s, _ = dims
        out = torch.empty((n, s + 2, s + 2, 2 * c), dtype=torch.float16, device=self.device)
        with torch.cuda.device(self.device):
            check(lib().vf_clip_rn_read_pairs(self._h, stage, out.data_ptr(), out.numel(), self._stream()))
        return out

    def conv(self, index: int) -> dict:
        """Diagnostics: conv ``index`` as uploaded, in execution order (include/vfeat.h vf_clip_rn_conv)."""
        with torch.cuda.device(self.device):
            return read_conv(lib().vf_clip_rn_conv, self._h, index, self.device)

    def block_geometry(self, block: int):
        """(side of the input, cin, side of the output, cout) of Bottleneck ``block`` as debug_block takes it."""
        if not 0 <= block < sum(self.layers):
            raise ValueError(f"block {block} outside 0 .. {sum(self.layers) - 1}")
        L, b = 0, block
        while b >= self.layers[L]:
            b -= self.layers[L]
            L += 1
        s_out, cout = self.n_px // (4 << L), 4 * (self.width << L)
        if b > 0:
            return s_out, cout, s_out, cout
        if L == 0:
            return self.n_px // 2, self.width, s_out, cout
        return 2 * s_out, cout // 2, s_out, cout

    def _check_pairs(self, x: torch.Tensor, side: int, c: int, what: str) -> torch.Tensor:
        # the entries copy n (side + 2)^2 rows of 2c halves from x: a wrong shape must not reach them
        if x.dtype != torch.float16 or x.dim() != 4 or tuple(x.shape[1:]) != (side + 2, side + 2, 2 * c):
            raise ValueError(f"{what} takes an fp16 pair volume (n, {side + 2}, {side + 2}, {2 * c}); "
                             f"got {x.dtype} {tuple(x.shape)}")
        if x.device != self.device:
            raise ValueError(f"the volume is on {x.device}, the engine on {self.device}")
        if not 1 <= x.shape[0] <= self.max_frames:
            raise ValueError(f"{x.shape[0]} frames; {what} takes 1 .. {self.max_frames}")
        return x.contiguous()

    def debug_block(self, block: int, x: torch.Tensor):
        """Diagnostics: Bottleneck ``block`` (execution order) once through the trunk's kernels (include/vfeat.h
        vf_clip_rn_debug_block).  x: zero-bordered pair volume (n, S_in + 2, S_in + 2, 2 cin) on the device (block 0:
        the unpooled stem output).  Returns (output, branch, shortcut or None) pair volumes (n, S_out + 2, S_out + 2,
        2 cout), border rows included.  read_stage then fails until the next encode."""
        s_in, cin, s_out, cout = self.block_geometry(block)
        x = self._check_pairs(x, s_in, cin, f"block {block}")
        shape = (x.shape[0], s_out + 2, s_out + 2, 2 * cout)
        out, branch, short = (torch.empty(shape, dtype=torch.float16, device=self.device) for _ in range(3))
        has_down = block in {sum(self.layers[:L]) for L in range(4)}
        with torch.cuda.device(self.device):
            check(lib().vf_clip_rn_debug_block(self._h, block, x.data_ptr(), x.shape[0], out.data_ptr(),
                                               branch.data_ptr(), short.data_ptr() if has_down else None,
                                               self._stream()))
        return out, branch, (short if has_down else None)

    def debug_attnpool(self, x: torch.Tensor):
        """Diagnostics: the attention pool as the encode runs it on a layer4 pair volume x (n, S4 + 2, S4 + 2, 2E)
        (include/vfeat.h vf_clip_rn_debug_attnpool).  Returns dict features (n, out_dim) fp32, tokens (n, T, 2E) fp16
        pairs, kv (n, T, 2E) fp32 ([k | v]), q (n, E) fp32 (unscaled), att (n, 2E) fp16 pairs."""
        s4 = self.n_px // 32
        x = self._check_pairs(x, s4, self.embed, "the attention pool")
        n, T, E = x.shape[0], self.tokens, self.embed
        feats = torch.empty((n, self.out_dim), dtype=torch.float32, device=self.device)
        out = dict(features=feats, tokens=torch.empty((n, T, 2 * E), dtype=torch.float16, device=self.device),
                   kv=torch.empty((n, T, 2 * E), dtype=torch.float32, device=self.device),
                   q=torch.empty((n, E), dtype=torch.float32, device=self.device),
                   att=torch.empty((n, 2 * E), dtype=torch.float16, device=self.device))
        with torch.cuda.device(self.device):
            check(lib().vf_clip_rn_debug_attnpool(self._h, x.data_ptr(), n, feats.data_ptr(), self._stream()))
            for what, key in enumerate(("tokens", "kv", "q", "att")):
                t = out[key]
                check(lib().vf_clip_rn_debug_attnpool_read(self._h, what, t.data_ptr(), t.numel(), self._stream()))
        return out

    @property
    def launch_count(self) -> int:
        return int(lib().vf_clip_rn_launch_count(self._h))

    def close(self):
        if getattr(self, "_h", None):
            lib().vf_clip_rn_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

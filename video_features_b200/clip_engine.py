"""CLIP ViT-B image tower handle (patch 32 or 16): the object that stands where the reference keeps the result of
``clip.load("ViT-B/32", device)`` (models/CLIP/extract_clip.py:47) -- ``encode_image`` included.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, Optional

import numpy as np
import torch

from . import _lib, ops  # noqa: F401  (ops registers torch.ops.vfeat.*)
from ._lib import ClipWeights, check, lib

_LAYER_KEYS = {
    "ln_1_w": "ln_1.weight", "ln_1_b": "ln_1.bias",
    "in_proj_w": "attn.in_proj_weight", "in_proj_b": "attn.in_proj_bias",
    "out_proj_w": "attn.out_proj.weight", "out_proj_b": "attn.out_proj.bias",
    "ln_2_w": "ln_2.weight", "ln_2_b": "ln_2.bias",
    "c_fc_w": "mlp.c_fc.weight", "c_fc_b": "mlp.c_fc.bias",
    "c_proj_w": "mlp.c_proj.weight", "c_proj_b": "mlp.c_proj.bias",
}
_TOP_KEYS = {
    "conv1_w": "conv1.weight", "class_embedding": "class_embedding",
    "positional_embedding": "positional_embedding", "ln_pre_w": "ln_pre.weight", "ln_pre_b": "ln_pre.bias",
    "ln_post_w": "ln_post.weight", "ln_post_b": "ln_post.bias", "proj": "proj",
}


def _shapes(patch: int):
    tokens = (224 // patch) ** 2 + 1
    return {"conv1_w": (768, 3, patch, patch), "class_embedding": (768,), "positional_embedding": (tokens, 768),
            "proj": (768, 512)}


class ClipEngine:
    """Owns device weights + workspace of one GPU.  ``state_dict`` uses openai's ``visual.*`` keys (a full CLIP
    state dict or a JIT archive's ``state_dict()`` works unchanged; text-tower keys are ignored)."""

    def __init__(self, state_dict: Dict[str, torch.Tensor], device: int = 0, chunk_frames: int = 0):
        if not torch.cuda.is_available():
            raise RuntimeError("ClipEngine needs a CUDA device (sm_90a); there is no CPU fallback")
        self.device = torch.device("cuda", device)
        self.out_dim = 512
        keep = []     # keep numpy arrays alive across the create call
        if "visual.conv1.weight" not in state_dict:
            raise KeyError("CLIP checkpoint is missing 'visual.conv1.weight'")
        patch = int(state_dict["visual.conv1.weight"].shape[-1])
        if patch not in (32, 16):
            raise ValueError(f"patch size {patch}: the ViT-B/32 and ViT-B/16 image towers are built")
        n_blocks = len({k.split(".")[3] for k in state_dict if k.startswith("visual.transformer.resblocks.")})
        if n_blocks != 12:
            raise ValueError(f"{n_blocks} transformer blocks: only the 12-block, 768-wide ViT-B towers are built")
        self.patch = patch
        self.tokens = (224 // patch) ** 2 + 1
        shapes = _shapes(patch)

        def arr(key: str, shape=None) -> C.POINTER(C.c_float):
            full = "visual." + key
            if full not in state_dict:
                raise KeyError(f"CLIP checkpoint is missing '{full}'")
            a = np.ascontiguousarray(state_dict[full].detach().to("cpu", torch.float32).numpy())
            if shape is not None and tuple(a.shape) != tuple(shape):
                raise ValueError(f"'{full}' has shape {a.shape}, ViT-B/{patch} needs {shape}")
            keep.append(a)
            return a.ctypes.data_as(C.POINTER(C.c_float))

        w = ClipWeights()
        for f, k in _TOP_KEYS.items():
            setattr(w, f, arr(k, shapes.get(f)))
        for i in range(12):
            for f, k in _LAYER_KEYS.items():
                setattr(w.layers[i], f, arr(f"transformer.resblocks.{i}.{k}"))
        h = C.c_void_p()
        check(lib().vf_clip_create_vit(C.byref(h), C.byref(w), device, chunk_frames, patch))
        self._h = h
        del keep

    @property
    def handle(self) -> int:
        """The vf_clip_t* as an integer: what the torch.ops.vfeat.clip_* custom ops take."""
        return int(self._h.value)

    # ---- model.encode_image(frames) : frames (T,3,224,224) float on this device
    def encode_image(self, frames: torch.Tensor) -> torch.Tensor:
        if not frames.is_cuda:
            raise RuntimeError("encode_image expects CUDA frames (no CPU fallback)")
        frames = frames.to(torch.float32).contiguous()
        assert frames.dim() == 4 and tuple(frames.shape[1:]) == (3, 224, 224), frames.shape
        return torch.ops.vfeat.clip_encode_image(self.handle, frames)          # PyTorch custom op over vf_clip_encode_f32

    # ---- fused preprocess + encode_image on raw decoder output: (T,H,W,3) uint8 on this device
    def encode_frames_u8(self, frames: torch.Tensor) -> torch.Tensor:
        assert frames.is_cuda and frames.dtype == torch.uint8 and frames.dim() == 4 and frames.shape[3] == 3
        return torch.ops.vfeat.clip_encode_u8(self.handle, frames.contiguous())  # custom op over vf_clip_encode_u8

    # ---- same with host buffers (numpy / CPU tensors): H2D + tower + D2H, synchronous
    def encode_frames_u8_host(self, frames, out: Optional[torch.Tensor] = None) -> torch.Tensor:
        if isinstance(frames, np.ndarray):
            frames = torch.from_numpy(np.ascontiguousarray(frames))
        assert (not frames.is_cuda) and frames.dtype == torch.uint8 and frames.dim() == 4 and frames.shape[3] == 3
        frames = frames.contiguous()
        n, hh, ww, _ = frames.shape
        if out is None:
            out = torch.empty((n, 512), dtype=torch.float32)
        assert out.dtype == torch.float32 and out.is_contiguous() and tuple(out.shape) == (n, 512)
        with torch.cuda.device(self.device):
            check(lib().vf_clip_encode_u8_host(self._h, frames.data_ptr(), n, hh, ww, out.data_ptr(),
                                               torch.cuda.current_stream().cuda_stream))
        return out

    # ---- host frames in, features on the DEVICE (for an all-gather), optionally on the host as well
    def encode_frames_u8_host_dev(self, frames: torch.Tensor, out_host: Optional[torch.Tensor] = None) -> torch.Tensor:
        assert (not frames.is_cuda) and frames.dtype == torch.uint8 and frames.dim() == 4 and frames.shape[3] == 3
        frames = frames.contiguous()
        n, hh, ww, _ = frames.shape
        out = torch.empty((n, 512), device=self.device, dtype=torch.float32)
        if out_host is not None:
            assert out_host.dtype == torch.float32 and out_host.is_contiguous() and tuple(out_host.shape) == (n, 512)
        with torch.cuda.device(self.device):
            check(lib().vf_clip_encode_u8_host_dev(self._h, frames.data_ptr(), n, hh, ww, out.data_ptr(),
                                                   None if out_host is None else out_host.data_ptr(),
                                                   torch.cuda.current_stream().cuda_stream))
        return out

    # ---- asynchronous form: enqueue and return; `wait(ticket)` before touching the host buffers
    def encode_frames_u8_host_async(self, frames: torch.Tensor, out_host: Optional[torch.Tensor] = None,
                                    out_dev: bool = False):
        """Pinned host frames in; features to ``out_host`` (pinned) and / or a new device tensor (``out_dev=True``).
        Returns ``(ticket, device tensor or None)``.  The H2D copies of this call overlap the tower of the call before
        it (vf_clip_encode_u8_host_async); ``frames`` and ``out_host`` belong to the engine until ``wait(ticket)``."""
        assert (not frames.is_cuda) and frames.dtype == torch.uint8 and frames.dim() == 4 and frames.shape[3] == 3
        assert frames.is_contiguous() and frames.is_pinned(), "asynchronous calls need pinned, contiguous host frames"
        n, hh, ww, _ = frames.shape
        if out_host is not None:
            assert out_host.dtype == torch.float32 and out_host.is_contiguous() and tuple(out_host.shape) == (n, 512)
            assert out_host.is_pinned(), "asynchronous calls need a pinned host output"
        assert out_host is not None or out_dev
        dev = torch.empty((n, 512), device=self.device, dtype=torch.float32) if out_dev else None
        ticket = C.c_int64(-1)
        with torch.cuda.device(self.device):
            check(lib().vf_clip_encode_u8_host_async(self._h, frames.data_ptr(), n, hh, ww,
                                                     None if dev is None else dev.data_ptr(),
                                                     None if out_host is None else out_host.data_ptr(),
                                                     torch.cuda.current_stream().cuda_stream, C.byref(ticket)))
        return int(ticket.value), dev

    def wait(self, ticket: int) -> None:
        """Block until the asynchronous call `ticket` has finished with its host buffers."""
        check(lib().vf_clip_wait(self._h, int(ticket)))

    def block_attention(self, layer: int, x: torch.Tensor, fused: bool = True) -> torch.Tensor:
        """Diagnostics: the attention half of resblock `layer` on x (n_frames*50, 768) fp16 -> (n_frames*50, 768) fp16,
        before the out-projection; fused=False runs the QKV GEMM + stand-alone attention kernel instead."""
        t = self.tokens
        assert x.is_cuda and x.dtype == torch.float16 and x.dim() == 2 and x.shape[1] == 768 and x.shape[0] % t == 0
        x = x.contiguous()
        out = torch.empty_like(x)
        with torch.cuda.device(self.device):
            check(lib().vf_clip_block_attention(self._h, layer, x.data_ptr(), x.shape[0] // t, out.data_ptr(), int(fused),
                                                torch.cuda.current_stream().cuda_stream))
        return out

    # ---- diagnostics: the tower's three pieces one at a time (vf_clip_debug_*); at most one chunk of frames per call
    def debug_embed(self, frames: torch.Tensor) -> torch.Tensor:
        """Patchify + patch embedding + ln_pre: (n,3,224,224) float32 or (n,H,W,3) uint8 on this device -> the fp32
        residual stream (n*tokens, 768)."""
        assert frames.is_cuda and frames.dim() == 4
        frames = frames.contiguous()
        n = frames.shape[0]
        x = torch.empty((n * self.tokens, 768), device=self.device, dtype=torch.float32)
        with torch.cuda.device(self.device):
            stream = torch.cuda.current_stream().cuda_stream
            if frames.dtype == torch.uint8:
                assert frames.shape[3] == 3, frames.shape
                check(lib().vf_clip_debug_embed_u8(self._h, frames.data_ptr(), n, frames.shape[1], frames.shape[2],
                                                   x.data_ptr(), stream))
            else:
                assert frames.dtype == torch.float32 and tuple(frames.shape[1:]) == (3, 224, 224), frames.shape
                check(lib().vf_clip_debug_embed_f32(self._h, frames.data_ptr(), n, x.data_ptr(), stream))
        return x

    def debug_blocks(self, x: torch.Tensor, begin: int, end: int) -> torch.Tensor:
        """Resblocks [begin, end) on a copy of the residual stream x (n*tokens, 768) float32.  end == 12: only the
        class-token rows (frame * tokens) of the result are defined."""
        t = self.tokens
        assert x.is_cuda and x.dtype == torch.float32 and x.dim() == 2 and x.shape[1] == 768 and x.shape[0] % t == 0
        x = x.contiguous().clone()
        with torch.cuda.device(self.device):
            check(lib().vf_clip_debug_blocks(self._h, x.data_ptr(), x.shape[0] // t, begin, end,
                                             torch.cuda.current_stream().cuda_stream))
        return x

    def debug_head(self, x: torch.Tensor) -> torch.Tensor:
        """ln_post on the class-token rows of x (n*tokens, 768) float32 + the projection -> (n, 512)."""
        t = self.tokens
        assert x.is_cuda and x.dtype == torch.float32 and x.dim() == 2 and x.shape[1] == 768 and x.shape[0] % t == 0
        x = x.contiguous()
        out = torch.empty((x.shape[0] // t, 512), device=self.device, dtype=torch.float32)
        with torch.cuda.device(self.device):
            check(lib().vf_clip_debug_head(self._h, x.data_ptr(), x.shape[0] // t, out.data_ptr(),
                                           torch.cuda.current_stream().cuda_stream))
        return out

    @property
    def launch_count(self) -> int:
        return int(lib().vf_clip_launch_count(self._h))

    def profile(self, enable: bool) -> None:
        check(lib().vf_clip_profile(self._h, int(enable)))

    def profile_read(self):
        """-> (gemm device ms, gemm launches, gemm algorithmic FLOPs) since the last read."""
        ms, n, fl = C.c_double(), C.c_int64(), C.c_double()
        check(lib().vf_clip_profile_read(self._h, C.byref(ms), C.byref(n), C.byref(fl)))
        return ms.value, n.value, fl.value

    def profile_categories(self):
        """device ms of the last profile_read window: {gemm, layernorm, attention, transform}."""
        ms = (C.c_double * 4)()
        check(lib().vf_clip_profile_categories(self._h, ms))
        return dict(zip(("gemm", "layernorm", "attention", "transform"), list(ms)))

    def close(self) -> None:
        if getattr(self, "_h", None):
            lib().vf_clip_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

"""DINOv2 frame-feature handle: ``torch.hub.load('facebookresearch/dinov2', name)(x)`` at 224 px for
``dinov2_vit{s,b,l,g}14`` and their ``_reg`` variants, the class token after the final norm, with the hub's eval
transform fused into the u8 entry."""
from __future__ import annotations

import ctypes as C
from typing import Dict

import torch
import torch.nn.functional as F

from ._lib import check, lib, named_tensors

GRID, HUB_GRID = 16, 37         # 224 / 14 patches a side; the checkpoints' grid (518 px)


def pos_table_224(pos_embed: torch.Tensor, registers: bool) -> torch.Tensor:
    """The hub's ``interpolate_pos_encoding`` for a 224 x 224 input, once, in fp32 on the host: (1, 1 + 37 * 37, D)
    -> (257, D).  The plain models scale the grid by (16 + 0.1) / 37 (DINOv2's interpolate_offset) without
    antialiasing; the _reg models ask for size (16, 16) with antialiasing.  Row 0 (the class position) is kept.
    tests/test_dinov2_oracle_cpu.py holds it equal to the oracle's restatement."""
    pe = pos_embed.detach().to("cpu", torch.float32).reshape(1, -1, pos_embed.shape[-1])
    d = pe.shape[-1]
    if pe.shape[1] != 1 + HUB_GRID * HUB_GRID:
        raise ValueError(f"pos_embed has {pe.shape[1]} rows, not 1 + 37 x 37")
    grid = pe[:, 1:].reshape(1, HUB_GRID, HUB_GRID, d).permute(0, 3, 1, 2)
    if registers:
        grid = F.interpolate(grid, mode="bicubic", antialias=True, size=(GRID, GRID))
    else:
        s = (GRID + 0.1) / HUB_GRID
        grid = F.interpolate(grid, mode="bicubic", antialias=False, scale_factor=(s, s))
    return torch.cat([pe[0, :1], grid.permute(0, 2, 3, 1).reshape(GRID * GRID, d)]).contiguous()


class DINOv2Engine:
    """``state_dict``: the hub checkpoint's keys (with or without the ``module.`` prefix), any float dtype; the shape is
    read from it.  The positional table for 224 px is interpolated once (``pos_table_224``) and handed to the
    engine as "pos_embed_224".  ``max_frames``: the workspace (0: about 2.5 GB, vf_dinov2_create); a larger call runs
    in chunks."""

    def __init__(self, state_dict: Dict[str, torch.Tensor], device: int = 0, max_frames: int = 0):
        if not torch.cuda.is_available():
            raise RuntimeError("DINOv2Engine needs a CUDA device (sm_90a); there is no CPU fallback")
        self.device = torch.device("cuda", device)
        arr, n, keep = named_tensors(state_dict_with_table(state_dict))
        h = C.c_void_p()
        check(lib().vf_dinov2_create(C.byref(h), arr, n, device, max_frames))
        self._h = h
        del keep
        info = (C.c_int * 7)()
        check(lib().vf_dinov2_info(self._h, info))
        self.out_dim, self.depth, self.heads, self.tokens, self.registers, swiglu, self.max_frames = tuple(info)
        self.ffn = "swiglu" if swiglu else "mlp"

    def _stream(self) -> int:
        return torch.cuda.current_stream(self.device).cuda_stream

    def encode_f32(self, x: torch.Tensor) -> torch.Tensor:
        """x: (n, 3, 224, 224) fp32, already transformed, on this device -> (n, out_dim) fp32."""
        if not x.is_cuda:
            raise RuntimeError("DINOv2Engine expects CUDA input (no CPU fallback)")
        x = x.to(torch.float32).contiguous()
        assert x.dim() == 4 and tuple(x.shape[1:]) == (3, 224, 224), x.shape
        out = torch.empty((x.shape[0], self.out_dim), device=x.device, dtype=torch.float32)
        with torch.cuda.device(self.device):
            check(lib().vf_dinov2_encode_f32(self._h, x.data_ptr(), x.shape[0], out.data_ptr(), self._stream()))
        return out

    def encode_u8(self, frames: torch.Tensor, out: torch.Tensor = None) -> torch.Tensor:
        """frames: (n, H, W, 3) uint8 BGR decoded frames of any size on this device -> (n, out_dim) fp32.  Resize(256,
        bicubic, Pillow-exact), CenterCrop(224), BGR->RGB, ToTensor and Normalize are fused.  Asynchronous on the
        current stream.  ``out``: an optional (n, out_dim) fp32 device tensor to write into."""
        if not frames.is_cuda:
            raise RuntimeError("DINOv2Engine expects CUDA frames (no CPU fallback)")
        assert frames.dtype == torch.uint8 and frames.dim() == 4 and frames.shape[3] == 3, frames.shape
        frames = frames.contiguous()
        n, hh, ww, _ = frames.shape
        if out is None:
            out = torch.empty((n, self.out_dim), device=frames.device, dtype=torch.float32)
        assert out.is_contiguous() and tuple(out.shape) == (n, self.out_dim) and out.dtype == torch.float32
        with torch.cuda.device(self.device):
            check(lib().vf_dinov2_encode_u8(self._h, frames.data_ptr(), n, hh, ww, out.data_ptr(), self._stream()))
        return out

    # ---- diagnostics: the pieces of the tower one at a time, eagerly, n <= max_frames
    def debug_embed_f32(self, x: torch.Tensor) -> torch.Tensor:
        """(n, 3, 224, 224) fp32 transformed frames -> the residual stream before block 0, (n, tokens, D) fp32."""
        x = x.to(self.device, torch.float32).contiguous()
        out = torch.empty((x.shape[0], self.tokens, self.out_dim), device=self.device, dtype=torch.float32)
        with torch.cuda.device(self.device):
            check(lib().vf_dinov2_debug_embed_f32(self._h, x.data_ptr(), x.shape[0], out.data_ptr(), self._stream()))
        return out

    def debug_embed_u8(self, frames: torch.Tensor) -> torch.Tensor:
        """(n, H, W, 3) uint8 BGR frames -> the residual stream before block 0, (n, tokens, D) fp32."""
        frames = frames.to(self.device).contiguous()
        n, hh, ww, _ = frames.shape
        out = torch.empty((n, self.tokens, self.out_dim), device=self.device, dtype=torch.float32)
        with torch.cuda.device(self.device):
            check(lib().vf_dinov2_debug_embed_u8(self._h, frames.data_ptr(), n, hh, ww, out.data_ptr(), self._stream()))
        return out

    def debug_blocks(self, x: torch.Tensor, first: int, last: int) -> torch.Tensor:
        """Blocks first .. last - 1 on a copy of x (n, tokens, D) fp32; the model's last block updates the class
        rows only."""
        assert tuple(x.shape[1:]) == (self.tokens, self.out_dim), x.shape
        y = x.to(self.device, torch.float32).clone().contiguous()
        with torch.cuda.device(self.device):
            check(lib().vf_dinov2_debug_blocks(self._h, y.data_ptr(), y.shape[0], first, last, self._stream()))
        return y

    def debug_head(self, x: torch.Tensor) -> torch.Tensor:
        """The final norm of the class rows of x (n, tokens, D) -> (n, D) fp32."""
        assert tuple(x.shape[1:]) == (self.tokens, self.out_dim), x.shape
        x = x.to(self.device, torch.float32).contiguous()
        out = torch.empty((x.shape[0], self.out_dim), device=self.device, dtype=torch.float32)
        with torch.cuda.device(self.device):
            check(lib().vf_dinov2_debug_head(self._h, x.data_ptr(), x.shape[0], out.data_ptr(), self._stream()))
        return out

    @property
    def launch_count(self) -> int:
        return int(lib().vf_dinov2_launch_count(self._h))

    def close(self):
        if getattr(self, "_h", None):
            lib().vf_dinov2_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def state_dict_with_table(state_dict):
    """The checkpoint's tensors plus "pos_embed_224", the table ``pos_table_224`` interpolates from its pos_embed."""
    sd = dict(state_dict)
    key = "pos_embed" if "pos_embed" in sd else "module.pos_embed"
    if key not in sd:
        raise KeyError("pos_embed: the DINOv2 checkpoint has no positional embedding")
    reg = "register_tokens" in sd or "module.register_tokens" in sd
    sd["pos_embed_224"] = pos_table_224(sd[key], reg)
    return sd


def swiglu(ab: torch.Tensor) -> torch.Tensor:
    """Diagnostics: the SwiGLU kernel alone.  ab (rows, 2 hidden) fp32 [a | b] on a device -> (rows, hidden) fp16
    silu(a) * b."""
    assert ab.is_cuda and ab.dtype == torch.float32 and ab.dim() == 2 and ab.shape[1] % 8 == 0, ab.shape
    ab = ab.contiguous()
    out = torch.empty((ab.shape[0], ab.shape[1] // 2), device=ab.device, dtype=torch.float16)
    with torch.cuda.device(ab.device):
        check(lib().vf_dinov2_swiglu(ab.data_ptr(), ab.shape[0], ab.shape[1] // 2, out.data_ptr(),
                                     torch.cuda.current_stream().cuda_stream))
    return out


def attention(qkv: torch.Tensor, heads: int) -> torch.Tensor:
    """Diagnostics: the blocks' attention alone.  qkv (n, S, 3 heads 64) fp16 -> (n, S, heads 64) fp16."""
    assert qkv.is_cuda and qkv.dtype == torch.float16 and qkv.dim() == 3 and qkv.shape[2] == 3 * heads * 64, qkv.shape
    qkv = qkv.contiguous()
    n, S, _ = qkv.shape
    out = torch.empty((n, S, heads * 64), device=qkv.device, dtype=torch.float16)
    with torch.cuda.device(qkv.device):
        check(lib().vf_dinov2_attention(qkv.data_ptr(), n, S, heads, out.data_ptr(),
                                        torch.cuda.current_stream().cuda_stream))
    return out

"""I3D feature extractor handle: stands where the reference keeps ``I3D(num_classes=400, modality=...)`` with its
checkpoint loaded (models/i3d/extract_i3d.py:109-118); ``engine(x, features=True)`` mirrors ``model(x, features=True)``.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict

import numpy as np
import torch

from . import ops  # noqa: F401  (registers torch.ops.vfeat.*)
from ._lib import I3D_UNITS, I3DWeights, check, lib

_MIXED = ["mixed_3b", "mixed_3c", "mixed_4b", "mixed_4c", "mixed_4d", "mixed_4e", "mixed_4f", "mixed_5b", "mixed_5c"]


def unit_names():
    names = ["conv3d_1a_7x7", "conv3d_2b_1x1", "conv3d_2c_3x3"]
    for m in _MIXED:
        names += [f"{m}.branch_0", f"{m}.branch_1.0", f"{m}.branch_1.1", f"{m}.branch_2.0", f"{m}.branch_2.1",
                  f"{m}.branch_3.1"]
    return names


class I3DEngine:
    """``state_dict``: the reference checkpoint layout (i3d_rgb.pt / i3d_flow.pt keys)."""

    def __init__(self, state_dict: Dict[str, torch.Tensor], modality: str = "rgb", device: int = 0,
                 max_stacks: int = 4, max_T: int = 64):
        if not torch.cuda.is_available():
            raise RuntimeError("I3DEngine needs a CUDA device (sm_90a); there is no CPU fallback")
        self.modality = modality
        self.cin = 3 if modality == "rgb" else 2
        self.device = torch.device("cuda", device)
        keep = []

        def arr(key):
            if key not in state_dict:
                raise KeyError(f"I3D checkpoint is missing '{key}'")
            a = np.ascontiguousarray(state_dict[key].detach().to("cpu", torch.float32).numpy())
            keep.append(a)
            return a, a.ctypes.data_as(C.POINTER(C.c_float))

        w = I3DWeights()
        names = unit_names()
        assert len(names) == I3D_UNITS
        for i, n in enumerate(names):
            wa, wp = arr(f"{n}.conv3d.weight")
            u = w.units[i]
            u.w = wp
            u.cout, u.cin, u.k = int(wa.shape[0]), int(wa.shape[1]), int(wa.shape[2])
            u.bn_w = arr(f"{n}.batch3d.weight")[1]
            u.bn_b = arr(f"{n}.batch3d.bias")[1]
            u.bn_mean = arr(f"{n}.batch3d.running_mean")[1]
            u.bn_var = arr(f"{n}.batch3d.running_var")[1]
        h = C.c_void_p()
        check(lib().vf_i3d_create(C.byref(h), C.byref(w), self.cin, device, max_stacks, max_T))
        self._h = h
        del keep

    def __call__(self, x: torch.Tensor, features: bool = True) -> torch.Tensor:
        """x (B, C, T, 224, 224) float on this device, values in [-1, 1] -> (B, 1024) float32."""
        if not features:
            raise NotImplementedError("only features=True (the extraction path) is built")
        if not x.is_cuda:
            raise RuntimeError("I3DEngine expects CUDA input (no CPU fallback)")
        x = x.to(torch.float32).contiguous()
        assert x.dim() == 5 and x.shape[1] == self.cin and tuple(x.shape[3:]) == (224, 224), x.shape
        return torch.ops.vfeat.i3d_forward(int(self._h.value), x)             # PyTorch custom op over vf_i3d_forward_f32

    def forward_frames_u8(self, frames: torch.Tensor) -> torch.Tensor:
        """rgb stream from resized uint8 frames (n, T, Hr, Wr, 3) on this device; crop/scale/permute fused."""
        assert frames.is_cuda and frames.dtype == torch.uint8 and frames.dim() == 5 and frames.shape[4] == 3
        n, T, Hr, Wr, _ = frames.shape
        fsz = Hr * Wr * 3
        # a window `stacks[:, :T]` of longer stacks (the reference's rgb_stack[:-1]) is read in place
        windowed = (n > 0 and frames.stride()[1:] == (fsz, Wr * 3, 3, 1) and frames.stride(0) % fsz == 0
                    and frames.stride(0) >= T * fsz)
        if not windowed:
            frames = frames.contiguous()
        stride = frames.stride(0) // fsz if n > 0 else T
        out = torch.empty((n, 1024), device=frames.device, dtype=torch.float32)
        with torch.cuda.device(self.device):
            check(lib().vf_i3d_forward_u8_strided(self._h, frames.data_ptr(), n, T, stride, Hr, Wr, out.data_ptr(),
                                                  torch.cuda.current_stream().cuda_stream))
        return out

    def forward_frames_u8_host(self, frames: torch.Tensor, T: int, group: int = 8, wait: bool = True):
        """rgb stream from HOST stacks (n, >=T, Hr, Wr, 3) uint8 (pinned memory for asynchronous copies): the first T
        frames of every stack are used; the host->device copy of stack group k+1 runs on a copy stream while group k is
        in the network.  Returns (n, 1024) float32 on the host.  ``wait=False`` returns ``(features, event)`` as soon as
        everything is enqueued -- the features (pinned) are valid after ``event.synchronize()``, and the copies of the
        NEXT call overlap the network of this one (``frames`` must stay untouched until then)."""
        assert not frames.is_cuda and frames.dtype == torch.uint8 and frames.dim() == 5 and frames.shape[4] == 3
        n = frames.shape[0]
        out = torch.empty((n, 1024), dtype=torch.float32).pin_memory()
        if n == 0:
            return out
        with torch.cuda.device(self.device):
            main = torch.cuda.current_stream()
            copy = getattr(self, "_copy_stream", None)
            if copy is None:
                copy = self._copy_stream = torch.cuda.Stream(device=self.device)
            bufs, ready, freed = [None, None], [None, None], [None, None]
            groups = [(a, min(n, a + group)) for a in range(0, n, group)]

            def stage(k):
                a, b = groups[k]
                with torch.cuda.stream(copy):
                    if freed[k & 1] is not None:
                        copy.wait_event(freed[k & 1])          # the network has finished reading this buffer
                    bufs[k & 1] = frames[a:b].to(self.device, non_blocking=True)
                    ready[k & 1] = torch.cuda.Event()
                    ready[k & 1].record(copy)

            stage(0)
            for k, (a, b) in enumerate(groups):
                if k + 1 < len(groups):
                    stage(k + 1)
                main.wait_event(ready[k & 1])
                y = self.forward_frames_u8(bufs[k & 1][:, :T])
                bufs[k & 1].record_stream(main)
                freed[k & 1] = torch.cuda.Event()
                freed[k & 1].record(main)
                out[a:b].copy_(y, non_blocking=True)
            if not wait:
                done = torch.cuda.Event(blocking=True)
                done.record(main)
                return out, done
            main.synchronize()
        return out

    def forward_flow(self, flow: torch.Tensor) -> torch.Tensor:
        """flow stream from raw optical flow (n, T, 2, H, W) fp32 on this device; T3 transform fused."""
        assert flow.is_cuda and flow.dtype == torch.float32 and flow.dim() == 5 and flow.shape[2] == 2
        flow = flow.contiguous()
        n, T, _, H, W = flow.shape
        out = torch.empty((n, 1024), device=flow.device, dtype=torch.float32)
        with torch.cuda.device(self.device):
            check(lib().vf_i3d_forward_flow(self._h, flow.data_ptr(), n, T, H, W, out.data_ptr(),
                                            torch.cuda.current_stream().cuda_stream))
        return out

    def read_stage(self, stage: int) -> torch.Tensor:
        """Diagnostics: a retained internal activation of the last forward as fp32 (n, C, T, H, W)."""
        dims = (C.c_int * 5)()
        check(lib().vf_i3d_read_stage(self._h, stage, None, 0, dims, None))
        out = torch.empty(tuple(dims), device=self.device, dtype=torch.float32)
        with torch.cuda.device(self.device):
            check(lib().vf_i3d_read_stage(self._h, stage, out.data_ptr(), out.numel(), dims,
                                          torch.cuda.current_stream().cuda_stream))
        return out

    @property
    def launch_count(self) -> int:
        return int(lib().vf_i3d_launch_count(self._h))

    def close(self):
        if getattr(self, "_h", None):
            lib().vf_i3d_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

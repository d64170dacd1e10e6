"""VGGish audio embedding handle: stands where the reference keeps ``VGGish(urls, postprocess=False)``
(models/vggish_torch/extract_vggish.py) and its ``forward(wav_path)``: 16-bit PCM samples in, raw 128-d embeddings
after the final ReLU out (no PCA).  Front end and trunk run on the GPU (include/vfeat.h vf_vggish_*)."""
from __future__ import annotations

import ctypes as C
from typing import Dict, Optional

import numpy as np
import torch

from . import audio
from ._lib import check, lib, named_tensors, read_conv

KEYS = tuple(f"features.{i}.{p}" for i in (0, 3, 6, 8, 11, 13) for p in ("weight", "bias")) + \
    tuple(f"embeddings.{i}.{p}" for i in (0, 2, 4) for p in ("weight", "bias"))
STAGES = ("waveform", "logmel", "pool1", "pool2", "pool3", "pool4", "fc1", "fc2", "fc3")   # vf_vggish_read_stage ids


class VGGishEngine:
    """``state_dict``: torchvggish keys (``features.{0,3,6,8,11,13}``, ``embeddings.{0,2,4}``; other keys, e.g. a PCA
    postprocessor's, are ignored), any float dtype.  ``max_examples``: 0.96 s examples per internal chunk (0: 64);
    longer inputs are chunked inside the call with the same features."""

    def __init__(self, state_dict: Dict[str, torch.Tensor], device: int = 0, max_examples: int = 0):
        if not torch.cuda.is_available():
            raise RuntimeError("VGGishEngine needs a CUDA device (sm_90a); there is no CPU fallback")
        self.device = torch.device("cuda", device)
        items = [(k[7:] if k.startswith("module.") else k, v) for k, v in state_dict.items()]
        items = [(k, v) for k, v in items if k in KEYS]
        arr, n, keep = named_tensors(items)
        hann = np.ascontiguousarray(audio.periodic_hann())
        mel = np.ascontiguousarray(audio.mel_matrix())
        win, num_table = audio.kaiser_best()
        win = np.ascontiguousarray(win)
        h = C.c_void_p()
        check(lib().vf_vggish_create(C.byref(h), arr, max(n, 1), hann.ctypes.data, mel.ctypes.data,
                                     win.ctypes.data, win.shape[0], num_table, device, max_examples))
        self._h = h
        del keep
        self.max_examples = max_examples or 64

    def _stream(self) -> int:
        return torch.cuda.current_stream(self.device).cuda_stream

    def forward_pcm16(self, samples, sample_rate: int) -> torch.Tensor:
        """int16 samples, (n,) mono or (n, channels) interleaved, numpy or a tensor on the host or this device ->
        (n_examples, 128) fp32 on this device (0 rows when the audio is shorter than 0.975 s)."""
        if isinstance(samples, np.ndarray):
            samples = torch.from_numpy(np.ascontiguousarray(samples))
        assert samples.dtype == torch.int16 and samples.dim() in (1, 2), (samples.dtype, samples.shape)
        n, ch = samples.shape[0], (samples.shape[1] if samples.dim() == 2 else 1)
        n_ex = audio.num_examples(audio.resampled_length(n, int(sample_rate)))
        out = torch.empty((n_ex, 128), device=self.device, dtype=torch.float32)
        got = C.c_int64()
        with torch.cuda.device(self.device):
            x = samples.contiguous().to(self.device)
            check(lib().vf_vggish_forward_pcm16(self._h, x.data_ptr(), n, ch, int(sample_rate), out.data_ptr(),
                                                out.numel(), C.byref(got), self._stream()))
        assert got.value == n_ex, (got.value, n_ex)
        return out

    def forward_logmel(self, examples: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """(n, 96, 64) fp32 log-mel examples (the network input) -> (n, 128) fp32 on this device."""
        x = torch.as_tensor(examples).to(self.device, torch.float32).contiguous()
        assert x.dim() == 3 and tuple(x.shape[1:]) == (audio.EXAMPLE_FRAMES, audio.MEL_BANDS), x.shape
        n = x.shape[0]
        if out is None:
            out = torch.empty((n, 128), device=self.device, dtype=torch.float32)
        with torch.cuda.device(self.device):
            check(lib().vf_vggish_forward_logmel_f32(self._h, x.data_ptr(), n, out.data_ptr(), self._stream()))
        return out

    def read_stage(self, stage: int) -> torch.Tensor:
        """Diagnostics, of the last chunk of the last call: 0 the resampled 16 kHz waveform (float64, (count,)), 1 the
        log-mel (n, 96, 64), 2..5 max-pools 1..4 (n, C, H, W), 6..8 fc1..fc3 after ReLU (n, D); fp32 from stage 1."""
        dims = (C.c_int * 4)()
        check(lib().vf_vggish_read_stage(self._h, stage, None, 0, dims, None))
        out = torch.empty(tuple(dims), device=self.device, dtype=torch.float64 if stage == 0 else torch.float32)
        with torch.cuda.device(self.device):
            check(lib().vf_vggish_read_stage(self._h, stage, out.data_ptr(), out.numel(), dims, self._stream()))
        if stage == 0:
            return out.flatten()
        if stage == 1:
            return out[:, 0]
        return out[:, :, 0, 0] if stage >= 6 else out

    def conv(self, index: int) -> dict:
        """Diagnostics: conv ``index`` as uploaded, 0..5 conv1..conv6, 6..8 fc1..fc3 (include/vfeat.h vf_vggish_conv)."""
        with torch.cuda.device(self.device):
            return read_conv(lib().vf_vggish_conv, self._h, index, self.device)

    @property
    def launch_count(self) -> int:
        return int(lib().vf_vggish_launch_count(self._h))

    def close(self):
        if getattr(self, "_h", None):
            lib().vf_vggish_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def time_register(sample_rate: int, t0: int, count: int) -> np.ndarray:
    """resampy's time register of outputs [t0, t0 + count) as the resampling kernel computes it (host code)."""
    out = np.empty(count, dtype=np.float64)
    check(lib().vf_vggish_time_register(int(sample_rate), t0, count, out.ctypes.data))
    return out

"""CLIP text tower handle (include/vfeat.h vf_clip_text_*) and the zero-shot head of ``--show_pred`` on the CLIP
feature types: prompts are encoded once, and every frame's image feature is compared with them by the classifier-head
kernel (class_head.py) with W = exp(logit_scale) * normalised text features and zero bias."""
from __future__ import annotations

import ctypes as C
import math
from typing import Dict

import numpy as np
import torch

from . import clip_tokenizer
from ._lib import check, lib, named_tensors
from .class_head import ClassHead

TEXT_PREFIXES = ("token_embedding.", "positional_embedding", "transformer.", "ln_final.", "text_projection",
                 "logit_scale")


def text_state_dict(state_dict: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
    """The text tower's entries of a full CLIP state dict (``read_clip_checkpoint``'s keys)."""
    return {k: v for k, v in state_dict.items() if k.startswith(TEXT_PREFIXES)}


class ClipTextEngine:
    """openai's ``encode_text`` followed by L2 normalisation on the GPU.  ``state_dict``: the text keys of a CLIP
    checkpoint, any float dtype.  ``max_rows``: the workspace in token rows (0: 8192, about 160 MB at width 768)."""

    def __init__(self, state_dict: Dict[str, torch.Tensor], device: int = 0, max_rows: int = 0):
        if not torch.cuda.is_available():
            raise RuntimeError("ClipTextEngine needs a CUDA device (sm_90a); there is no CPU fallback")
        self.device = torch.device("cuda", device)
        arr, n, keep = named_tensors(text_state_dict(state_dict))
        h = C.c_void_p()
        check(lib().vf_clip_text_create(C.byref(h), arr, n, device, max_rows))
        self._h = h
        del keep
        info = (C.c_int * 7)()
        check(lib().vf_clip_text_info(self._h, info))
        self.width, self.heads, self.layers, self.context, self.embed, self.vocab, self.max_rows = list(info)

    def encode(self, tokens) -> torch.Tensor:
        """tokens: (n, context) int ids (``clip_tokenizer`` rows) -> (n, embed) fp32 normalised text features on this
        device, asynchronous on the current stream."""
        t = np.ascontiguousarray(np.asarray(tokens, dtype=np.int32))
        assert t.ndim == 2 and t.shape[1] == self.context, (t.shape, self.context)
        out = torch.empty((t.shape[0], self.embed), device=self.device, dtype=torch.float32)
        with torch.cuda.device(self.device):
            check(lib().vf_clip_text_encode(self._h, t.ctypes.data, t.shape[0], out.data_ptr(),
                                            torch.cuda.current_stream().cuda_stream))
        return out

    def blocks(self, x: torch.Tensor, first: int, count: int) -> torch.Tensor:
        """Diagnostics: blocks first .. first + count - 1 on a copy of the residual stream x (n, L, width) fp32."""
        assert x.is_cuda and x.dim() == 3 and x.shape[2] == self.width
        y = x.to(torch.float32).contiguous().clone()
        with torch.cuda.device(self.device):
            check(lib().vf_clip_text_blocks(self._h, y.data_ptr(), y.shape[0], y.shape[1], first, count,
                                            torch.cuda.current_stream().cuda_stream))
        return y

    @property
    def launch_count(self) -> int:
        return int(lib().vf_clip_text_launch_count(self._h))

    def close(self):
        if getattr(self, "_h", None):
            lib().vf_clip_text_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def attention(qkv: torch.Tensor, heads: int) -> torch.Tensor:
    """The causal attention kernel alone: qkv (n, L, 3 * heads * 64) fp16 -> (n, L, heads * 64) fp16."""
    assert qkv.is_cuda and qkv.dtype == torch.float16 and qkv.dim() == 3 and qkv.shape[2] == 3 * heads * 64
    qkv = qkv.contiguous()
    out = torch.empty(qkv.shape[0], qkv.shape[1], heads * 64, device=qkv.device, dtype=torch.float16)
    with torch.cuda.device(qkv.device):
        check(lib().vf_clip_text_attention(qkv.data_ptr(), qkv.shape[0], qkv.shape[1], heads, out.data_ptr(),
                                           torch.cuda.current_stream().cuda_stream))
    return out


def l2_normalize_rows(x: torch.Tensor) -> torch.Tensor:
    """(n, C) fp32 device rows -> a new tensor of the rows over their L2 norms."""
    assert x.is_cuda and x.dtype == torch.float32 and x.dim() == 2
    x = x.contiguous()
    out = torch.empty_like(x)
    with torch.cuda.device(x.device):
        check(lib().vf_l2_normalize_rows(x.data_ptr(), x.shape[0], x.shape[1], out.data_ptr(),
                                         torch.cuda.current_stream().cuda_stream))
    return out


def check_vocabulary(state_dict: Dict[str, torch.Tensor], tokenizer: clip_tokenizer.SimpleTokenizer) -> None:
    """ValueError when the checkpoint has no text tower or its token embedding does not match the vocabulary."""
    emb = state_dict.get("token_embedding.weight")
    if emb is None or "logit_scale" not in state_dict:
        raise ValueError("--show_pred on CLIP needs the checkpoint's text tower ('token_embedding.weight', "
                         "'logit_scale', ...), and this checkpoint has none")
    if emb.shape[0] != tokenizer.vocab_size:
        raise ValueError(f"the BPE vocabulary has {tokenizer.vocab_size} entries but the checkpoint's "
                         f"token_embedding.weight has {emb.shape[0]} rows")


class ZeroShotHead:
    """CLIP's ``logits_per_image`` for a fixed list of prompts: ``forward`` L2-normalises the image features into
    scratch (the caller's tensor is not touched) and runs the classifier head on them; its interface is ClassHead's, so
    TopKQueue takes it as well."""

    def __init__(self, state_dict: Dict[str, torch.Tensor], tokens, device: int = 0):
        eng = ClipTextEngine(state_dict, device)
        try:
            text = eng.encode(tokens)
            scale = math.exp(float(state_dict["logit_scale"]))
            weight = (text.double() * scale).float().cpu()
        finally:
            eng.close()
        self.head = ClassHead(weight, torch.zeros(weight.shape[0]), device)
        self.n_classes, self.n_features = self.head.n_classes, self.head.n_features

    def forward(self, feats: torch.Tensor, k: int = 5):
        """feats (n, embed) on the device -> ClassHead.forward of the normalised rows (k clamped to the prompts)."""
        return self.head.forward(l2_normalize_rows(feats.to(torch.float32)), min(k, self.n_classes))

    def top_k_host(self, feats: torch.Tensor, k: int = 5):
        _, _, idx, tl, tp = self.forward(feats, k)
        return idx.cpu(), tl.cpu(), tp.cpu()

    def close(self):
        self.head.close()


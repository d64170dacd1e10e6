"""Classifier head handle for ``--show_pred``: the checkpoint's own last layer (ResNet / R(2+1)D ``fc``, I3D
``conv3d_0c_1x1``) on the device features an engine call already produced, with softmax and top-k in the same call
(include/vfeat.h vf_head_forward).  One class for all three extractors."""
from __future__ import annotations

import ctypes as C
from collections import deque
from typing import Callable, Dict, List, Sequence, Tuple

import numpy as np
import torch

from . import ops  # noqa: F401  (registers torch.ops.vfeat.*)
from ._lib import check, lib

FC_KEYS = ("fc.weight", "fc.bias")                                            # torchvision ResNet, r2plus1d_18
I3D_KEYS = ("conv3d_0c_1x1.conv3d.weight", "conv3d_0c_1x1.conv3d.bias")       # the reference's I3D
MAX_K = 8


class ClassHead:
    """``weight``: (C, K, ...) with trailing singleton dims (a 1x1x1 conv) or (C, K); ``bias``: (C,)."""

    def __init__(self, weight: torch.Tensor, bias: torch.Tensor, device: int = 0):
        if not torch.cuda.is_available():
            raise RuntimeError("ClassHead needs a CUDA device (sm_90a); there is no CPU fallback")
        w = np.ascontiguousarray(weight.detach().to("cpu", torch.float32).reshape(weight.shape[0], -1).numpy())
        b = np.ascontiguousarray(bias.detach().to("cpu", torch.float32).reshape(-1).numpy())
        if b.shape[0] != w.shape[0]:
            raise ValueError(f"classifier head: weight {tuple(weight.shape)} and bias {tuple(bias.shape)} disagree")
        self.n_classes, self.n_features = int(w.shape[0]), int(w.shape[1])
        self.device = torch.device("cuda", device)
        h = C.c_void_p()
        check(lib().vf_head_create(C.byref(h), w.ctypes.data, b.ctypes.data, self.n_classes, self.n_features, device))
        self._h = h

    @classmethod
    def from_state_dict(cls, state_dict: Dict[str, torch.Tensor], keys: Tuple[str, str], device: int = 0,
                        what: str = "checkpoint") -> "ClassHead":
        """The head stored under ``keys`` (weight, bias), with or without the ``module.`` prefix."""
        found = []
        for k in keys:
            v = state_dict.get(k, state_dict.get("module." + k))
            if v is None:
                raise KeyError(f"--show_pred needs the classifier head, but the {what} has no '{k}' "
                               "(the features themselves do not use it)")
            found.append(v)
        return cls(found[0], found[1], device)

    def forward(self, feats: torch.Tensor, k: int = 5):
        """feats (n, K) on this device -> (logits (n, C), probs (n, C), top_idx (n, k) int32, top_logit (n, k),
        top_prob (n, k)), all on the device, asynchronous on the current stream.  Top-k order: probability descending,
        equal probabilities by the lower class index."""
        if not feats.is_cuda:
            raise RuntimeError("ClassHead expects CUDA features (no CPU fallback)")
        feats = feats.to(torch.float32).contiguous()
        assert feats.dim() == 2 and feats.shape[1] == self.n_features, (tuple(feats.shape), self.n_features)
        return tuple(torch.ops.vfeat.class_head(int(self._h.value), feats, self.n_classes, int(k)))

    def __call__(self, feats: torch.Tensor):
        """-> (softmax, logits), as the reference's ``I3D(x, features=False)`` returns them."""
        logits, probs = self.forward(feats, 1)[:2]
        return probs, logits

    def top_k_host(self, feats: torch.Tensor, k: int = 5):
        """Only the top-k crosses to the host: (top_idx, top_logit, top_prob) as (n, k) CPU tensors (synchronous)."""
        _, _, idx, tl, tp = self.forward(feats, k)
        return idx.cpu(), tl.cpu(), tp.cpu()

    def close(self):
        if getattr(self, "_h", None):
            lib().vf_head_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class TopKQueue:
    """Top-k of engine calls copied into pinned host memory without blocking the host: ``submit`` enqueues the heads on
    the current stream and returns; an entry is printed (``emit``) once the next one is submitted, or at ``flush``.
    So the decode of the next chunk overlaps the network of this one with --show_pred as without it, and entries are
    emitted in submission order."""

    def __init__(self, k: int = 5):
        self.k = k
        self._pending = deque()

    def submit(self, heads_feats: Sequence[Tuple[ClassHead, torch.Tensor]],
               emit: Callable[[List[Tuple[torch.Tensor, torch.Tensor, torch.Tensor]]], None]) -> None:
        """heads_feats: [(head, (n, K) device features)]; emit receives one (top_idx, top_logit, top_prob) tuple of
        (n, k) host tensors per pair."""
        tops = []
        with torch.cuda.device(heads_feats[0][1].device):
            for head, feats in heads_feats:
                dev = head.forward(feats, self.k)[2:]
                host = tuple(torch.empty(t.shape, dtype=t.dtype, pin_memory=True) for t in dev)
                for h, d in zip(host, dev):
                    h.copy_(d, non_blocking=True)
                tops.append(host)
            done = torch.cuda.Event()
            done.record()
        self._pending.append((done, tops, emit))
        while len(self._pending) > 1:
            self._emit_oldest()

    def flush(self) -> None:
        while self._pending:
            self._emit_oldest()

    def _emit_oldest(self):
        done, tops, emit = self._pending.popleft()
        done.synchronize()
        emit(tops)

"""The reference's classification paths next to the trunk restatements (test oracle only): I3D ``forward(features=False)``
(models/i3d/i3d_src/i3d_net.py:266-274, in its order: avg pool -> conv3d_0c_1x1 per temporal position with bias ->
mean over time -> softmax) on oracle/i3d_net.py's trunk, and torchvision's ``fc`` for oracle/resnet_net.py and
oracle/r21d_net.py."""
from __future__ import annotations

from typing import Dict

import torch
import torch.nn.functional as F

from . import i3d_net, r21d_net, resnet_net


def _strip(sd):
    return {k[7:] if k.startswith("module.") else k: v for k, v in sd.items()}


@torch.no_grad()
def i3d_logits_from_5c(sd: Dict[str, torch.Tensor], mixed_5c: torch.Tensor):
    """mixed_5c output (B, 1024, T', 7, 7) -> (softmax, logits), each (B, 400), in the reference's order."""
    x = F.avg_pool3d(mixed_5c, (2, 7, 7), (1, 1, 1))                # (B, 1024, T'-1, 1, 1)
    x = F.conv3d(x, sd["conv3d_0c_1x1.conv3d.weight"], sd["conv3d_0c_1x1.conv3d.bias"])   # dropout: identity in eval
    logits = x.squeeze(3).squeeze(3).mean(2)
    return F.softmax(logits, dim=1), logits


@torch.no_grad()
def i3d_forward_logits(sd: Dict[str, torch.Tensor], inp: torch.Tensor, **kw):
    """== I3D.forward(inp, features=False) -> (softmax, logits); ``kw`` as i3d_net.forward_features."""
    _, st = i3d_net.forward_features(sd, inp, return_stages=True, **kw)
    return i3d_logits_from_5c(sd, st["5c"])


def fc_logits(sd: Dict[str, torch.Tensor], feats: torch.Tensor) -> torch.Tensor:
    """torchvision's ``model.fc(feats)`` (ResNet, r2plus1d_18), ``module.`` prefix accepted."""
    sd = _strip(sd)
    return F.linear(feats, sd["fc.weight"].to(feats.dtype), sd["fc.bias"].to(feats.dtype))


@torch.no_grad()
def resnet_logits(sd, x: torch.Tensor, depth: int) -> torch.Tensor:
    """x (n, 3, 224, 224) normalised -> (n, 1000) ImageNet logits."""
    return fc_logits(sd, resnet_net.forward(sd, x, depth))


@torch.no_grad()
def r21d_logits(sd, x: torch.Tensor) -> torch.Tensor:
    """x (n, 3, T, 112, 112) normalised -> (n, 400) Kinetics logits."""
    return fc_logits(sd, r21d_net.forward(sd, x))

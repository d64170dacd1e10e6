"""Functional restatement of the reference's PWC-Net (models/pwc/pwc_src/pwc_net.py:23-263 and the cost volume of
correlation.py:44-112) over a state dict, in fp32 or float64, with the intermediate tensors the engine's diagnostics
expose.  Test infrastructure, never imported by the product.

Semantics pinned here (DESIGN.md §2):
- the model swaps channels 0 and 2 and divides by 255 itself (pwc_net.py:230-231), then resizes to multiples of 64
  with F.interpolate(bilinear, align_corners=False) (pwc_net.py:241-245);
- the backward warp is grid_sample(bilinear, zeros) as torch 1.2 -- the version the reference pins
  (conda_env_pwc.yml:60) -- computes it, i.e. with align_corners=True: pixel (x + u, y + v).  Later torch releases
  silently switch the same call to align_corners=False; `align_corners=False` reproduces that for comparison only;
- the warp mask is the grid_sample of a ones channel thresholded at 0.999 (pwc_net.py:39).
"""
from __future__ import annotations

import math
import os
from typing import Dict, Optional

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STATS = os.path.join(ROOT, "tests", "golden", "pwc_checkpoint_stats.json")
CHECKPOINT = "pwc_net_sintel.pt"
LEVEL_NAMES = {1: "One", 2: "Two", 3: "Thr", 4: "Fou", 5: "Fiv", 6: "Six"}
DBL_BACKWARD = {5: 0.625, 4: 1.25, 3: 2.5, 2: 5.0}          # pwc_net.py:121
REFINER_DILATION = (1, 2, 4, 8, 16, 1, 1)                    # pwc_net.py:193-207


def _leaky(x):
    return F.leaky_relu(x, 0.1)


def _conv(sd, name, x, stride=1, dilation=1):
    w, b = sd[name + ".weight"], sd[name + ".bias"]
    return F.conv2d(x, w.to(x.dtype), b.to(x.dtype), stride=stride, padding=dilation, dilation=dilation)


def _deconv(sd, name, x):
    w, b = sd[name + ".weight"], sd[name + ".bias"]
    return F.conv_transpose2d(x, w.to(x.dtype), b.to(x.dtype), stride=2, padding=1)


def preprocess(frames: torch.Tensor) -> torch.Tensor:
    """(n, 3, H, W) in [0,255] as the caller passes them -> x[:, [2,1,0]] / 255 at the /64 size (pwc_net.py:230-245)."""
    x = frames[:, [2, 1, 0]] / 255
    h, w = x.shape[2:]
    hp, wp = int(math.floor(math.ceil(h / 64.0) * 64.0)), int(math.floor(math.ceil(w / 64.0) * 64.0))
    return F.interpolate(x, size=(hp, wp), mode="bilinear", align_corners=False)


def extractor(sd, x) -> list:
    """pwc_net.py:44-110: the six feature levels (1/2 .. 1/64)."""
    feats = []
    for l in range(1, 7):
        p = f"moduleExtractor.module{LEVEL_NAMES[l]}."
        x = _leaky(_conv(sd, p + "0", x, stride=2))
        x = _leaky(_conv(sd, p + "2", x))
        x = _leaky(_conv(sd, p + "4", x))
        feats.append(x)
    return feats


def correlation(first: torch.Tensor, second: torch.Tensor) -> torch.Tensor:
    """correlation.py:44-112: channel c = displacement (dx, dy) = (c % 9 - 4, c // 9 - 4),
    value = sum_c first(y, x) second(y + dy, x + dx) / C with zeros outside the map."""
    n, c, h, w = first.shape
    padded = F.pad(second, (4, 4, 4, 4))
    out = first.new_zeros((n, 81, h, w))
    for k in range(81):
        dy, dx = k // 9 - 4, k % 9 - 4
        out[:, k] = (first * padded[:, :, 4 + dy:4 + dy + h, 4 + dx:4 + dx + w]).sum(1) / c
    return out


def backward_warp(x: torch.Tensor, flow: torch.Tensor, align_corners: bool = True):
    """pwc_net.py:23-41 -> (warped, mask, raw mask): the raw mask is the in-bounds bilinear weight sum before the 0.999
    threshold.  align_corners=True is the reference's pinned torch 1.2 behaviour."""
    n, _, h, w = flow.shape
    hor = torch.linspace(-1.0, 1.0, w, dtype=flow.dtype).view(1, 1, 1, w).expand(n, -1, h, -1)
    ver = torch.linspace(-1.0, 1.0, h, dtype=flow.dtype).view(1, 1, h, 1).expand(n, -1, -1, w)
    grid = torch.cat([hor, ver], 1).to(flow.device)
    fl = torch.cat([flow[:, [0]] / ((x.shape[3] - 1.0) / 2.0), flow[:, [1]] / ((x.shape[2] - 1.0) / 2.0)], 1)
    inp = torch.cat([x, flow.new_ones((n, 1, h, w))], 1)
    out = F.grid_sample(inp, (grid + fl).permute(0, 2, 3, 1), mode="bilinear", padding_mode="zeros",
                        align_corners=align_corners)
    raw = out[:, -1:]
    mask = torch.where(raw > 0.999, torch.ones_like(raw), torch.zeros_like(raw))
    return out[:, :-1] * mask, mask, raw


def forward(sd: Dict[str, torch.Tensor], first: torch.Tensor, second: torch.Tensor, dtype=torch.float32,
            align_corners: bool = True, stages: Optional[dict] = None) -> torch.Tensor:
    """PWCNet()(first, second) (pwc_net.py:226-263): (n, 3, H, W) in [0,255] -> (n, 2, H, W) flow in ``dtype``.
    ``stages`` (a dict) receives feats1 / feats2 (lists per level 1..6) and per decoder level l: vol{l}, mask{l},
    upflow{l}, upfeat{l}, mask{l}, maskraw{l} (levels 5..2), flow{l}, feat{l}; then refine and flow."""
    st = stages if stages is not None else {}
    h, w = first.shape[2:]
    a, b = preprocess(first.to(dtype)), preprocess(second.to(dtype))
    hp, wp = a.shape[2:]
    f1s, f2s = extractor(sd, a), extractor(sd, b)
    st["feats1"], st["feats2"] = f1s, f2s
    prev = None
    for l in range(6, 1, -1):
        p = f"module{LEVEL_NAMES[l]}."
        f1, f2 = f1s[l - 1], f2s[l - 1]
        if prev is None:
            vol = _leaky(correlation(f1, f2))
            feat = vol
        else:
            upflow = _deconv(sd, p + "moduleUpflow", prev[0])
            upfeat = _deconv(sd, p + "moduleUpfeat", prev[1])
            warped, mask, raw = backward_warp(f2, upflow * DBL_BACKWARD[l], align_corners)
            vol = _leaky(correlation(f1, warped))
            feat = torch.cat([vol, f1, upflow, upfeat], 1)
            st[f"upflow{l}"], st[f"upfeat{l}"], st[f"mask{l}"], st[f"maskraw{l}"] = upflow, upfeat, mask, raw
        st[f"vol{l}"] = vol
        for k in ("One", "Two", "Thr", "Fou", "Fiv"):
            feat = torch.cat([_leaky(_conv(sd, p + f"module{k}.0", feat)), feat], 1)
        flow = _conv(sd, p + "moduleSix.0", feat)
        st[f"flow{l}"], st[f"feat{l}"] = flow, feat
        prev = (flow, feat)
    x = prev[1]
    for k, d in enumerate(REFINER_DILATION):
        x = _conv(sd, f"moduleRefiner.moduleMain.{2 * k}", x, dilation=d)
        if k < 6:
            x = _leaky(x)
    st["refine"] = x
    out = 20.0 * F.interpolate(prev[0] + x, size=(h, w), mode="bilinear", align_corners=False)
    out[:, 0] *= float(w) / float(wp)
    out[:, 1] *= float(h) / float(hp)
    st["flow"] = out
    return out


def flow_of_frames(sd, frames: torch.Tensor, dtype=torch.float32, align_corners: bool = True) -> torch.Tensor:
    """model(frames[:-1], frames[1:]) for (N, 3, H, W) frames."""
    return forward(sd, frames[:-1], frames[1:], dtype, align_corners)


def checkpoint_stats(sd) -> list:
    """[key, shape, dtype, mean, std] per tensor: the fixture stand_in_state_dict draws from."""
    return [[k, list(v.shape), str(v.dtype).replace("torch.", ""), float(v.double().mean()),
             float(v.double().std()) if v.numel() > 1 else 0.0] for k, v in sd.items()]


def stand_in_state_dict() -> Dict[str, torch.Tensor]:
    """Seeded stand-in for pwc_net_sintel.pt: the same keys and shapes, every tensor drawn with the mean and standard
    deviation of the trained tensor it replaces (tests/golden/pwc_checkpoint_stats.json), one generator per tensor
    seeded from its name.  The trained level-6 extractor weights (|w| <= 1e-36 .. 3e-14) keep their scale, so the
    stand-in exercises the engine's per-channel weight scaling as the checkpoint does."""
    import json
    import zlib
    from collections import OrderedDict
    rows = json.load(open(STATS))
    sd = OrderedDict()
    for key, shape, dtype, mean, std in rows:
        g = torch.Generator().manual_seed(zlib.crc32(f"{CHECKPOINT}/{key}".encode()))
        z = torch.randn(shape, generator=g, dtype=torch.float64)
        sd[key] = (mean + std * z).to(getattr(torch, dtype))
    return sd


def fetch_checkpoint() -> None:
    """Best effort, as oracle/fetch_ref.py: copy the reference's pwc_net_sintel.pt (data) into oracle/_ref/checkpoints/
    where scripts/pwc_time.py and the precision scripts read it; the tests use the stand-in."""
    import shutil
    import sys
    src = os.path.join(os.environ.get("VF_REFERENCE_DIR", "/root/reference"), "models", "pwc", "checkpoints", CHECKPOINT)
    dst = os.path.join(ROOT, "oracle", "_ref", "checkpoints", CHECKPOINT)
    if os.path.exists(dst):
        return
    if os.path.exists(src):
        os.makedirs(os.path.dirname(dst), exist_ok=True)
        shutil.copyfile(src, dst)
        print("copied", CHECKPOINT)
    else:
        print(f"pwc_net: {src} not found; {dst} stays missing", file=sys.stderr)


if __name__ == "__main__":
    fetch_checkpoint()

"""fp32 restatement of the reference's Inception-3D (I3D) forward, features=True -- test oracle only.

Follows models/i3d/i3d_src/i3d_net.py: ``Unit3Dpy`` (:37-105, TF-SAME padding via get_padding_shape :8-25, BN eval +
ReLU), ``MaxPool3dTFPadding`` (:108-120, ZERO padding then ceil-mode max pool), ``Mixed`` (:123-157),
``I3D.forward(inp, features=True)`` (:238-264).  Functional, driven by a state dict in the reference's own key layout
(the vendored checkpoints i3d_rgb.pt / i3d_flow.pt load unchanged).  Pinned against the reference module run with the
vendored checkpoints in the build container (scripts/make_golden.py -> tests/golden/i3d_*.npz).
"""
from __future__ import annotations

from collections import OrderedDict
from typing import Dict

import torch
import torch.nn.functional as F

BN_EPS = 1e-5
MIXED = OrderedDict([                      # i3d_net.py:206-224: in_channels, [b0, b1a, b1b, b2a, b2b, b3]
    ("mixed_3b", (192, [64, 96, 128, 16, 32, 32])),
    ("mixed_3c", (256, [128, 128, 192, 32, 96, 64])),
    ("mixed_4b", (480, [192, 96, 208, 16, 48, 64])),
    ("mixed_4c", (512, [160, 112, 224, 24, 64, 64])),
    ("mixed_4d", (512, [128, 128, 256, 24, 64, 64])),
    ("mixed_4e", (512, [112, 144, 288, 32, 64, 64])),
    ("mixed_4f", (528, [256, 160, 320, 32, 128, 128])),
    ("mixed_5b", (832, [256, 160, 320, 32, 128, 128])),
    ("mixed_5c", (832, [384, 192, 384, 48, 128, 128])),
])


def unit_names():
    """Conv units in the fixed order the engine's weight table uses."""
    names = ["conv3d_1a_7x7", "conv3d_2b_1x1", "conv3d_2c_3x3"]
    for m in MIXED:
        names += [f"{m}.branch_0", f"{m}.branch_1.0", f"{m}.branch_1.1", f"{m}.branch_2.0", f"{m}.branch_2.1",
                  f"{m}.branch_3.1"]
    return names


def unit_shapes(in_channels: int):
    """name -> (cout, cin, k)"""
    shapes = OrderedDict()
    shapes["conv3d_1a_7x7"] = (64, in_channels, 7)
    shapes["conv3d_2b_1x1"] = (64, 64, 1)
    shapes["conv3d_2c_3x3"] = (192, 64, 3)
    for m, (cin, oc) in MIXED.items():
        shapes[f"{m}.branch_0"] = (oc[0], cin, 1)
        shapes[f"{m}.branch_1.0"] = (oc[1], cin, 1)
        shapes[f"{m}.branch_1.1"] = (oc[2], oc[1], 3)
        shapes[f"{m}.branch_2.0"] = (oc[3], cin, 1)
        shapes[f"{m}.branch_2.1"] = (oc[4], oc[3], 3)
        shapes[f"{m}.branch_3.1"] = (oc[5], cin, 1)
    return shapes


def synthetic_state_dict(modality: str = "rgb", seed: int = 0) -> "OrderedDict[str, torch.Tensor]":
    """Seeded weights with He-scaled convs and mild BN statistics so activations stay O(1) through 58 layers."""
    g = torch.Generator().manual_seed(seed)
    cin0 = 3 if modality == "rgb" else 2
    sd = OrderedDict()
    for name, (co, ci, k) in unit_shapes(cin0).items():
        fan = ci * k ** 3
        sd[f"{name}.conv3d.weight"] = torch.randn(co, ci, k, k, k, generator=g) * (2.0 / fan) ** 0.5
        sd[f"{name}.batch3d.weight"] = 1.0 + 0.1 * torch.randn(co, generator=g)
        sd[f"{name}.batch3d.bias"] = 0.05 * torch.randn(co, generator=g)
        sd[f"{name}.batch3d.running_mean"] = 0.05 * torch.randn(co, generator=g)
        sd[f"{name}.batch3d.running_var"] = 1.0 + 0.1 * torch.rand(co, generator=g)
    return sd


def _same_pad(k, s):
    # i3d_net.py:8-25 get_padding_shape for one dim
    pad_along = max(k - s, 0)
    top = pad_along // 2
    return top, pad_along - top


def _fp16(t: torch.Tensor) -> torch.Tensor:
    return t.half().to(t.dtype)


# The operands the engine keeps as single fp16 (every other GEMM operand is a split-fp16 pair, every other weight hi +
# lo; i3d.cu): the stem input, the inputs of conv3d_2c and of every Mixed branch_1.1 / branch_2.1 (the 1x1x1 reducers'
# outputs), and the weights of the units in DECLARED_FP16_UNITS (indices into unit_names(): the stem and the 3x3x3
# convs of mixed_3b / 3c; prepare_unit's `chosen`, none of them with VF_I3D_SINGLE=none).
DECLARED_FP16_UNITS = (0, 5, 7, 11, 13)
_FP16_INPUT = ("conv3d_1a_7x7", "conv3d_2c_3x3") + tuple(f"{m}.branch_{b}.1" for m in MIXED for b in (1, 2))


def _unit(sd, name, x, k, stride=1, fp16=None):
    """fp16: None, or (unit names whose input is rounded to fp16, unit names whose weights are)."""
    w = sd[f"{name}.conv3d.weight"]
    if fp16 is not None:
        if name in fp16[0]:
            x = _fp16(x)
        if name in fp16[1]:
            w = _fp16(w)
    pt, pb = _same_pad(k, stride)
    if k > 1:
        x = F.pad(x, (pt, pb, pt, pb, pt, pb))            # zeros; symmetric for k=3,s=1, (2,3) for the 7/2 stem
    x = F.conv3d(x, w, None, stride=stride)
    x = F.batch_norm(x, sd[f"{name}.batch3d.running_mean"], sd[f"{name}.batch3d.running_var"],
                     sd[f"{name}.batch3d.weight"], sd[f"{name}.batch3d.bias"], False, 0.0, BN_EPS)
    return F.relu(x)


def _maxpool(x, k, s):
    # i3d_net.py:108-120: ConstantPad3d(zeros) then MaxPool3d(ceil_mode=True)
    pads = []
    for kd, sd_ in zip(reversed(k), reversed(s)):          # F.pad takes W, H, T order
        t, b = _same_pad(kd, sd_)
        pads += [t, b]
    x = F.pad(x, pads)
    return F.max_pool3d(x, k, s, ceil_mode=True)


def _fp16_sets(declared_rounding, fp16_units, fp16_inputs=(), fp16_weights=()):
    """The ``fp16`` argument of _unit: (unit names whose input is rounded, unit names whose weights are), or None."""
    if not (declared_rounding or fp16_inputs or fp16_weights):
        return None
    names = unit_names()
    return (set(fp16_inputs) | (set(_FP16_INPUT) if declared_rounding else set()),
            set(fp16_weights) | ({names[i] for i in fp16_units} if declared_rounding else set()))


def _mixed(sd, m, x, fp16=None):
    b0 = _unit(sd, f"{m}.branch_0", x, 1, fp16=fp16)
    b1 = _unit(sd, f"{m}.branch_1.1", _unit(sd, f"{m}.branch_1.0", x, 1, fp16=fp16), 3, fp16=fp16)
    b2 = _unit(sd, f"{m}.branch_2.1", _unit(sd, f"{m}.branch_2.0", x, 1, fp16=fp16), 3, fp16=fp16)
    b3 = _unit(sd, f"{m}.branch_3.1", _maxpool(x, (3, 3, 3), (1, 1, 1)), 1, fp16=fp16)
    return torch.cat((b0, b1, b2, b3), 1)


@torch.no_grad()
def forward_features(sd: Dict[str, torch.Tensor], inp: torch.Tensor, return_stages: bool = False,
                     declared_rounding: bool = False, fp16_units=DECLARED_FP16_UNITS, fp16_inputs=(),
                     fp16_weights=()):
    """inp (B, C, T, 224, 224) float in [-1, 1] -> (B, 1024).  == I3D.forward(inp, features=True), in the dtype of
    inp and sd.  ``declared_rounding`` rounds to fp16 exactly the operands the engine keeps as single fp16: the inputs
    listed at DECLARED_FP16_UNITS and the weights of the units `fp16_units` (() for an engine built with
    VF_I3D_SINGLE=none).  fp16_inputs / fp16_weights (unit names) round further conv inputs / weights (precision
    emulations: a pair tensor or a split weight left single fp16).  Stages: 1a, 2c, 3c, 4f, 5c."""
    fp16 = _fp16_sets(declared_rounding, fp16_units, fp16_inputs, fp16_weights)
    st = {}
    x = _unit(sd, "conv3d_1a_7x7", inp, 7, 2, fp16=fp16); st["1a"] = x
    x = _maxpool(x, (1, 3, 3), (1, 2, 2))
    x = _unit(sd, "conv3d_2b_1x1", x, 1, fp16=fp16)
    x = _unit(sd, "conv3d_2c_3x3", x, 3, fp16=fp16); st["2c"] = x
    x = _maxpool(x, (1, 3, 3), (1, 2, 2))
    x = _mixed(sd, "mixed_3b", x, fp16)
    x = _mixed(sd, "mixed_3c", x, fp16); st["3c"] = x
    x = _maxpool(x, (3, 3, 3), (2, 2, 2))
    for m in ("mixed_4b", "mixed_4c", "mixed_4d", "mixed_4e", "mixed_4f"):
        x = _mixed(sd, m, x, fp16)
    st["4f"] = x
    x = _maxpool(x, (2, 2, 2), (2, 2, 2))
    x = _mixed(sd, "mixed_5b", x, fp16)
    x = _mixed(sd, "mixed_5c", x, fp16); st["5c"] = x
    x = F.avg_pool3d(x, (2, 7, 7), (1, 1, 1))
    out = x.squeeze(3).squeeze(3).mean(2)
    return (out, st) if return_stages else out


@torch.no_grad()
def mixed_block(sd: Dict[str, torch.Tensor], m: str, x: torch.Tensor, declared_rounding: bool = False,
                fp16_units=DECLARED_FP16_UNITS, fp16_inputs=(), fp16_weights=()):
    """Mixed block ``m`` (a key of MIXED) on x, as forward_features runs it (the same rounding arguments): the concat
    (b0, b1, b2, b3) along channels."""
    return _mixed(sd, m, x, _fp16_sets(declared_rounding, fp16_units, fp16_inputs, fp16_weights))


@torch.no_grad()
def mixed_inputs(sd: Dict[str, torch.Tensor], inp: torch.Tensor, declared_rounding: bool = False,
                 fp16_units=DECLARED_FP16_UNITS):
    """The input of every Mixed block (MIXED order) in forward_features(inp) with the same rounding arguments."""
    fp16 = _fp16_sets(declared_rounding, fp16_units)
    x = _unit(sd, "conv3d_1a_7x7", inp, 7, 2, fp16=fp16)
    x = _maxpool(x, (1, 3, 3), (1, 2, 2))
    x = _unit(sd, "conv3d_2b_1x1", x, 1, fp16=fp16)
    x = _maxpool(_unit(sd, "conv3d_2c_3x3", x, 3, fp16=fp16), (1, 3, 3), (1, 2, 2))
    ins = []
    for m in MIXED:
        ins.append(x)
        x = _mixed(sd, m, x, fp16)
        if m == "mixed_3c":
            x = _maxpool(x, (3, 3, 3), (2, 2, 2))
        elif m == "mixed_4f":
            x = _maxpool(x, (2, 2, 2), (2, 2, 2))
    return ins


def maxpool(x: torch.Tensor, k, s) -> torch.Tensor:
    """MaxPool3dTFPadding(k, s, 'SAME'): zero padding, then a ceil-mode max pool (the trunk's pools)."""
    return _maxpool(x, k, s)


def rgb_transform(stack: torch.Tensor) -> torch.Tensor:
    """extract_i3d.py:62-66 on a (T,3,H,W) float [0,255] stack: TensorCenterCrop(224) (floor offsets,
    transforms.py:7-18) -> ScaleTo1_1 (2x/255 - 1) -> PermuteAndUnsqueeze -> (1,3,T,224,224)."""
    H, W = stack.shape[-2:]
    fh, fw = (H - 224) // 2, (W - 224) // 2
    x = stack[..., fh:fh + 224, fw:fw + 224]
    x = (2 * x / 255) - 1
    return x.permute(1, 0, 2, 3).unsqueeze(0)


def flow_transform(flow: torch.Tensor) -> torch.Tensor:
    """extract_i3d.py:67-73 on a (T,2,H,W) flow: crop 224 -> clamp(+-20) -> 128 + 255/40*f -> round (half to even;
    +20 maps to 256, not clipped) -> ScaleTo1_1 -> permute."""
    H, W = flow.shape[-2:]
    fh, fw = (H - 224) // 2, (W - 224) // 2
    x = flow[..., fh:fh + 224, fw:fw + 224]
    x = torch.clamp(x, min=-20, max=20)
    x = (128 + 255 / 40 * x).round()
    x = (2 * x / 255) - 1
    return x.permute(1, 0, 2, 3).unsqueeze(0)

"""The float64 bars of the ResNet and R(2+1)D engines (tests/split_engine_bars.py) can tell the designed precision
scheme from a broken one.  scripts/precision/emulate_{resnet,r21d}.py run the stand-in networks in float64 with the
conv operands of each tensor class rounded to fp32 ('split': a split-fp16 pair carries ~22 bits) or to one fp16 value.
At every stage the class reaches, leaving any one class in single fp16 must exceed the GPU bar by the factor
split_engine_bars.SEPARATION names (tenfold at the stem and through layer3), and the all-split scheme must stay tenfold
under it.  A lost lo half or W_lo pass in the engine is one of those classes (or a
part of one), so the GPU test would see it."""
import importlib.util
import os

import pytest
import torch

import split_engine_bars as bars
from oracle import r21d_net, resnet_net

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _emulation(name):
    path = os.path.join(ROOT, "scripts", "precision", f"emulate_{name}.py")
    spec = importlib.util.spec_from_file_location(f"emulate_{name}", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _schemes(classes):
    out = {"all split": {c: "split" for c in classes}}
    for c in classes:
        out[f"fp16 {c}"] = dict({k: "split" for k in classes}, **{c: "fp16"})
    return out


def _check(name, run, ref, stages, bar, first_stage, classes, factor):
    """run(scheme) -> (features, taps); ref = (features, taps) of the float64 forward."""
    failures = []
    for sname, scheme in _schemes(classes).items():
        y, taps = run(scheme)
        for s in stages:
            got, want = (y, ref[0]) if s == "features" else (taps[s], ref[1][s])
            err = bars.row_errors(got, want)
            print(f"{name} {sname:<12s} {s:<8s} rel-L2 {err[0]:.1e}  max-abs/max {err[1]:.1e}  bar {bar[s][0]:.0e}")
            if sname == "all split":
                if not bars.within(err, bar[s], 0.1):
                    failures.append((sname, s, err, "not 10x under the bar"))
            elif stages.index(s) >= stages.index(first_stage[sname[5:]]):
                if not (err[0] > factor[s] * bar[s][0] and err[1] > factor[s] * bar[s][1]):
                    failures.append((sname, s, err, f"not {factor[s]}x over the bar"))
    assert not failures, failures


def test_resnet18_bars_separate_split_from_single_fp16():
    emu = _emulation("resnet")
    torch.set_grad_enabled(False)
    sd = {k: v.double() if v.is_floating_point() else v for k, v in resnet_net.stand_in_state_dict(18).items()}
    x = resnet_net.calibration_images(seed=7, n=2).double()
    ref = resnet_net.forward(sd, x, 18, taps=True)
    # the first stage each class reaches in a basic-block ResNet (it has no 1x1 conv but the downsample)
    first = {"stem": "stem", "w": "stem", "c3x3": "layer1", "resid": "layer1", "down": "layer2"}
    classes = tuple(c for c in emu.CLASSES if c != "c1x1")
    _check("resnet18", lambda sc: emu.forward(sd, x, 18, dict(sc, c1x1="split"), taps=True), ref,
           bars.RESNET_STAGES, bars.RESNET_BARS[18], first, classes, bars.SEPARATION["resnet18"])


def test_r21d_bars_separate_split_from_single_fp16():
    emu = _emulation("r21d")
    torch.set_grad_enabled(False)
    sd = {k: v.double() if v.is_floating_point() else v for k, v in r21d_net.stand_in_state_dict().items()}
    x = r21d_net.calibration_clips(seed=7, n=1, T=8).double()
    ref = r21d_net.forward(sd, x, taps=True)
    # the stem has a temporal conv; layer1.0 keeps 64 channels (identity path), layer2.0 downsamples
    first = {"stem": "stem", "w": "stem", "temp": "stem", "spat": "layer1", "resid": "layer1", "down": "layer2"}
    _check("r21d", lambda sc: emu.forward(sd, x, sc, taps=True), ref, bars.R21D_STAGES, bars.R21D_BARS, first,
           emu.CLASSES, bars.SEPARATION["r21d"])

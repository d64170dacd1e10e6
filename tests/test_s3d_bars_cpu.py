"""The float64 bars of the S3D engine (tests/s3d_bars.py) tell its split scheme from a broken one.
scripts/precision/emulate_s3d.py runs the stand-in in float64 with the conv operands of each tensor class rounded to fp32
('split': a split-fp16 pair carries ~22 bits) or to one fp16 value.  The all-split scheme must stay tenfold under every
bar; leaving any one class in single fp16 must exceed the bar, in both rel-L2 and max-abs, by the factor
s3d_bars.SEPARATION names at every stage from the first one the class reaches.  A lost lo half, W_lo pass or pair
store in the engine is one of those classes (or a part of one), so the GPU test would see it."""
import importlib.util
import os

import torch

import s3d_bars as bars
from oracle import s3d_net

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _emulation():
    path = os.path.join(ROOT, "scripts", "precision", "emulate_s3d.py")
    spec = importlib.util.spec_from_file_location("emulate_s3d", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _errors(got, want):
    got, want = got.double().flatten(1), want.double().flatten(1)
    d = got - want
    return (d.norm(dim=1) / want.norm(dim=1)).max().item(), (d.abs().amax(dim=1) / want.abs().amax(dim=1)).max().item()


def test_s3d_bars_separate_split_from_single_fp16():
    emu = _emulation()
    assert set(emu.CLASSES) == set(bars.FIRST_STAGE)
    torch.set_grad_enabled(False)
    sd = {k: v.double() if v.is_floating_point() else v for k, v in s3d_net.stand_in_state_dict().items()}
    x = s3d_net.calibration_clips(seed=7, n=1, T=16).double()
    ref = s3d_net.forward(sd, x, taps=True)
    schemes = {"all split": {c: "split" for c in emu.CLASSES}}
    for c in emu.CLASSES:
        schemes[f"fp16 {c}"] = dict({k: "split" for k in emu.CLASSES}, **{c: "fp16"})
    failures = []
    for name, scheme in schemes.items():
        y, taps = emu.forward(sd, x, scheme, taps=True)
        for s in bars.STAGES:
            got, want = (y, ref[0]) if s == "features" else (taps[s], ref[1][s])
            err, bar = _errors(got, want), bars.BARS[s]
            print(f"s3d {name:<12s} {s:<9s} rel-L2 {err[0]:.1e} ({err[0] / bar[0]:6.1f}x bar)  "
                  f"max-abs/max {err[1]:.1e} ({err[1] / bar[1]:6.1f}x bar)")
            if name == "all split":
                if not (err[0] <= 0.1 * bar[0] and err[1] <= 0.1 * bar[1]):
                    failures.append((name, s, err, "not 10x under the bar"))
            elif bars.STAGES.index(s) >= bars.STAGES.index(bars.FIRST_STAGE[name[5:]]):
                f = bars.SEPARATION[s]
                if not (err[0] > f * bar[0] and err[1] > f * bar[1]):
                    failures.append((name, s, err, f"not {f}x over the bar"))
    assert not failures, failures

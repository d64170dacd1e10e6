"""The float64 bars of the ResNet and R(2+1)D engines (tests/split_engine_bars.py) can tell the designed precision
scheme from a broken one.  scripts/precision/emulate_{resnet,r21d}.py run the stand-in networks in float64 with the
conv operands of each tensor class rounded to fp32 ('split': a split-fp16 pair carries ~22 bits) or to one fp16 value.
At every stage the class reaches, leaving any one class in single fp16 must exceed the GPU bar by the factor
split_engine_bars.SEPARATION names (tenfold at the stem and through layer3), and the all-split scheme must stay tenfold
under it.  A lost lo half or W_lo pass in the engine is one of those classes (or a
part of one), so the GPU test would see it.

I3D and RAFT are held to a float64 reference with their declared fp16 rounding; here each class that the engine keeps as
a split pair or split weight is left single fp16 on top of it, and SEPARATION_I3D / SEPARATION_RAFT state where (and by
how much) the GPU bars tell it apart.  Where they do not, the conv read-back (test_i3d_raft_uploads_gpu.py) does."""
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


def _check_separation(name, variants, run, ref, bar, separation):
    """variants: class -> run() kwargs; every stated (stage, factor) of each class must fail the bar by that factor."""
    failures = []
    for c, kw in variants.items():
        got = run(**kw)
        for s, factor in separation[c].items():
            err = bars.row_errors(got[s], ref[s])
            print(f"{name} fp16 {c:<30s} {s:<8s} rel-L2 {err[0] / bar[s][0]:5.1f}x  max-abs {err[1] / bar[s][1]:5.1f}x"
                  f"  (asserted {factor}x)")
            if not bars.beyond(err, bar[s], factor):
                failures.append((c, s, err, factor))
    assert set(variants) == set(separation)
    assert not failures, failures


def test_i3d_bars_separate_declared_from_single_fp16():
    """I3D: each pair-tensor class and each group of split weights left single fp16, against the declared-rounding
    float64 reference (what the GPU test holds the engine to)."""
    from oracle import i3d_net as N
    from helpers import stand_in_state_dict
    torch.set_grad_enabled(False)
    sd = {k: v.double() for k, v in stand_in_state_dict("i3d_rgb.pt").items()}
    x = (torch.rand(1, 3, 10, 224, 224, generator=torch.Generator().manual_seed(3)) * 2 - 1).double()
    names = N.unit_names()
    M = list(N.MIXED)
    after_pool = ("mixed_3b", "mixed_4b", "mixed_5b")
    reducers = [f"{m}.branch_{b}" for m in M for b in ("0", "1.0", "2.0", "3.1")]
    variants = {
        "stem output": dict(fp16_inputs=["conv3d_2b_1x1"]),
        "pool outputs": dict(fp16_inputs=[f"{m}.branch_3.1" for m in M]
                             + [f"{m}.branch_{b}" for m in after_pool for b in ("0", "1.0", "2.0")]),
        "concat buffers": dict(fp16_inputs=[f"{m}.branch_{b}" for m in M if m not in after_pool
                                            for b in ("0", "1.0", "2.0")]),
        "1x1x1 inputs": dict(fp16_inputs=["conv3d_2b_1x1"] + reducers),
        "2b / 2c weights": dict(fp16_weights=["conv3d_2b_1x1", "conv3d_2c_3x3"]),
        "1x1x1 weights": dict(fp16_weights=reducers),
        "4x / 5x 3x3x3 weights": dict(fp16_weights=[f"{m}.branch_{b}.1" for m in M[2:] for b in (1, 2)]),
    }
    assert all(n in names for kw in variants.values() for v in kw.values() for n in v)

    def run(**kw):
        y, st = N.forward_features(sd, x, True, declared_rounding=True, **kw)
        return dict(st, features=y)
    _check_separation("i3d", variants, run, run(), bars.I3D_BARS["rgb"], bars.SEPARATION_I3D)


def test_raft_bars_separate_declared_from_single_fp16(monkeypatch):
    """RAFT: the operand groups of scripts/precision/emulate_raft.py left single fp16, after 3 iterations, against the
    declared-rounding float64 reference."""
    import torch.nn.functional as F
    from oracle import raft_net as R
    from helpers import stand_in_state_dict
    torch.set_grad_enabled(False)
    sd = {k: v.double() for k, v in stand_in_state_dict("raft-sintel.pth").items()}
    fr = R.synthetic_frames(2, 128, 160, seed=11, shift=(0.8, 0.5)).double()

    def run(round_input=lambda n: False, w16=lambda n: False, gru_motion=False):
        def conv(sd_, name, xx, stride=1, padding=0):
            w = sd_[name + ".weight"]
            w = w.half().double() if w16(name) else w
            xx = xx.half().double() if round_input(name) else xx
            if gru_motion and ".gru." in name:          # the motion-encoder slice of the GRU input
                xx = xx.clone()
                xx[:, 256:382] = xx[:, 256:382].half().double()
            return F.conv2d(xx, w, sd_[name + ".bias"], stride=stride, padding=padding)
        monkeypatch.setattr(R, "_conv", conv)
        up, st = R.forward(sd, fr[:-1], fr[1:], 3, taps=True, declared_rounding=True)
        pyr = torch.cat([p.reshape(fr.shape[0] - 1, -1) for p in st["pyramid"]], 1)
        return {"fnet": st["fnet"], "cnet": st["cnet"], "pyramid": pyr, "lookup": st["lookup"][-1],
                "net": st["net"][-1], "lowres": st["lowres"][-1], "flow_up": up}

    variants = {
        "fnet weights": dict(w16=lambda n: n.startswith("fnet")),
        "cnet weights": dict(w16=lambda n: n.startswith("cnet")),
        "motion encoder weights": dict(w16=lambda n: "update_block.encoder" in n),
        "GRU weights": dict(w16=lambda n: ".gru." in n),
        "flow head weights": dict(w16=lambda n: "flow_head" in n),
        "fnet inner inputs": dict(round_input=lambda n: n.startswith("fnet") and n != "fnet.conv1"),
        "cnet inner inputs": dict(round_input=lambda n: n.startswith("cnet") and n != "cnet.conv1"),
        "motion encoder intermediates": dict(round_input=lambda n: n.endswith(("convc2", "convf2", "encoder.conv"))),
        "flow head conv2 input": dict(round_input=lambda n: n.endswith("flow_head.conv2")),
        "GRU motion slice": dict(gru_motion=True),
    }
    _check_separation("raft", variants, run, run(), bars.RAFT_BARS, bars.SEPARATION_RAFT)

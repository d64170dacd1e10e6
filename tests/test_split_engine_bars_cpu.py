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


def test_clip_vit_bars_and_defect_share_separate_the_controls():
    """CLIP ViT: block 5 of the plain synthetic tower at 3 frames.  The engine is emulated by the declared-rounding block
    in fp32 (fp32 accumulation, rounding flips against the float64 reference: what the GPU bars consist of).  Against
    the committed block bar: the emulation passes; bf16 weights, an fp16 residual stream and a zeroed in_proj bias group
    fail it.  Unrounded P, fp16 scores, eps 1e-6 and a QuickGELU constant of 1.7 stay within about 1x of the bar -- each is
    smaller than the flips it causes -- and are told apart by defect_share instead: an emulated engine WITH the defect
    carries more than 0.65 of its direction (0.78 .. 1.0 here), the one without less than 0.5 (0.0 .. 0.24).  eps 1e-6 fails the head bar on a row of
    variance 1e-6; the zeroed bias group fails the attention bar."""
    import torch.nn.functional as F
    from oracle import clip_tower as C
    torch.set_grad_enabled(False)
    sd = C.synthetic_state_dict(0)
    sd64 = {k: v.double() for k, v in sd.items()}
    k = 5
    p = f"visual.transformer.resblocks.{k}."
    x = C.embed(sd64, torch.randn(3, 3, 224, 224, generator=torch.Generator().manual_seed(1)), declared_rounding=True)
    for i in range(k):
        x = C.block(sd64, i, x, declared_rounding=True)
    x = x.float().double()                                   # the engine's stream is fp32
    rows = lambda t: t.reshape(-1, t.shape[-1])
    ref = C.block(sd64, k, x, declared_rounding=True)
    bar = bars.CLIP_VIT["block"]["plain"]
    emu = C.block(sd, k, x.float(), declared_rounding=True)
    err = bars.row_errors(rows(emu), rows(ref))
    print(f"clip block fp32 emulation: {err[0]:.1e} / {err[1]:.1e} (bar {bar[0]:.0e} / {bar[1]:.0e})")
    assert bars.within(err, bar), err

    sdz = dict(sd64)
    sdz[p + "attn.in_proj_bias"] = sd64[p + "attn.in_proj_bias"].clone()
    sdz[p + "attn.in_proj_bias"][-8:] = 0
    sdb = {n: (v.bfloat16().double() if v.dim() >= 2 and "positional" not in n else v) for n, v in sd64.items()}
    f32 = lambda d: {n: v.float() for n, v in d.items()}
    # name -> (kwargs of the defect, state dict, least factor over the block bar or None where it is not separated)
    variants = {
        "bf16 weights": (dict(declared_rounding=True), sdb, bars.CLIP_VIT_CONTROLS["bf16 weights"][1]),
        "fp16 residual stream": (dict(rounding=C.DECLARED | {"resid"}), sd64, 2.5),
        "in_proj bias group zeroed": (dict(declared_rounding=True), sdz, 2.5),
        "P unrounded": (dict(rounding=C.DECLARED - {"p"}), sd64, None),
        "fp16 scores": (dict(rounding=C.DECLARED | {"scores"}), sd64, None),
        "eps 1e-6": (dict(declared_rounding=True, eps=1e-6), sd64, None),
        "QuickGELU 1.7": (dict(declared_rounding=True, gelu=1.7), sd64, None),
    }
    lo, hi = bars.CLIP_VIT_SHARE
    failures = []
    for name, (kw, sdv, factor) in variants.items():
        refd = C.block(sdv, k, x, **kw)
        e = bars.row_errors(rows(refd), rows(ref))
        with_defect = bars.defect_share(C.block(f32(sdv), k, x.float(), **kw), ref, refd)
        without = bars.defect_share(emu, ref, refd)
        print(f"clip {name:<26s} {e[0] / bar[0]:5.1f}x / {e[1] / bar[1]:5.1f}x the block bar; share with the defect "
              f"{with_defect:+.2f}, without {without:+.2f}")
        if factor is not None and not bars.beyond(e, bar, factor):
            failures.append((name, e, factor))
        if factor is None and bars.beyond(e, bar, 2):
            failures.append((name, e, "stated as not separated, yet 2x over the bar"))
        if not (with_defect > hi and abs(without) < lo):
            failures.append((name, with_defect, without))
    assert not failures, failures

    # the head: a row of variance 1e-6, where eps = 1e-5 decides the result
    row = (1e-3 * torch.randn(1, 768, generator=torch.Generator().manual_seed(3))).double()
    h_ref = C.head(sd64, row, declared_rounding=True)
    h_emu = C.head(sd, row.float(), declared_rounding=True)
    assert bars.within(bars.row_errors(h_emu, h_ref), bars.CLIP_VIT["head"])
    what, factor = bars.CLIP_VIT_CONTROLS["eps 1e-6"]
    assert bars.beyond(bars.row_errors(C.head(sd64, row, declared_rounding=True, eps=1e-6), h_ref), bars.CLIP_VIT[what], factor)

    # the attention half on the block's own ln_1 output: the zeroed bias group
    h = C._r16(C._ln_d(x, sd64[p + "ln_1.weight"], sd64[p + "ln_1.bias"], C.LN_EPS))
    w = C._r16(sd64[p + "attn.in_proj_weight"])
    att = frozenset({"qkv", "p", "att"})
    a_ref = C.attention_core(F.linear(h, w, sd64[p + "attn.in_proj_bias"]), rounding=att)
    a_emu = C.attention_core(F.linear(h.float(), w.float(), sd[p + "attn.in_proj_bias"]), rounding=att)
    a_ctl = C.attention_core(F.linear(h, w, sdz[p + "attn.in_proj_bias"]), rounding=att)
    what, factor = bars.CLIP_VIT_CONTROLS["in_proj bias group zeroed"]
    abar = bars.CLIP_VIT[what]
    assert bars.within(bars.row_errors(rows(a_emu), rows(a_ref)), abar)
    ctl = bars.row_errors(rows(a_ctl), rows(a_ref))
    print(f"clip attention, bias group zeroed: {ctl[0] / abar[0]:.1f}x / {ctl[1] / abar[1]:.1f}x the attention bar")
    assert bars.beyond(ctl, abar, factor), ctl

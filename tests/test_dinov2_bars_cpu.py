"""The DINOv2 bars (tests/dinov2_bars.py) against scripts/precision/emulate_dinov2.py, which runs the stand-ins in float64
with each tensor class either exact (a split-fp16 pair, or fp32) or rounded to one fp16 value, against the exact
forward, for all eight shapes at full depth.  The engine's scheme (weights split, the SwiGLU inputs fp32, every other
class fp16) must cost at most SCHEME_FRACTION of the feature bar, and so must every class the engine keeps in single
fp16 on its own: half the bar for S, B and L, and 0.8 for g/14, the explicit exception dinov2_bars.py gives the reason
for.  The feature is one token, so the activations' fp16 roundings are not averaged away and fp16 weights would cost
about as much as all of them together (DESIGN.md §4.17); a lost lo half is caught at the embedding, where weights
rounded to fp16 exceed the bar by SEPARATION."""
import functools
import importlib.util
import os

import pytest

import dinov2_bars as bars
from oracle import dinov2_net as D

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@functools.lru_cache(maxsize=1)
def _emulation():
    path = os.path.join(ROOT, "scripts", "precision", "emulate_dinov2.py")
    spec = importlib.util.spec_from_file_location("emulate_dinov2", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@functools.lru_cache(maxsize=None)
def _table(name):
    """The engine's scheme, each of its single-fp16 classes alone and, for g, the scheme with the w12 output in fp16 too,
    on 2 calibration frames at full depth."""
    emu = _emulation()
    schemes = {"engine": emu.ENGINE}
    schemes.update({c: (c,) for c in emu.ENGINE})
    if D.shape_of(name)[2] == "swiglu":
        schemes["engine + swiglu fp16"] = emu.ENGINE + ("swiglu",)
    return emu.table(name, 2, "cpu", schemes)


def _limit(name):
    d = D.shape_of(name)[0]
    f = bars.SCHEME_FRACTION[d]
    return bars.FEATURES[d][0] * f, bars.FEATURES[d][1] * f


@pytest.mark.parametrize("name", list(D.MODELS))
def test_engine_scheme_is_within_its_share_of_the_bar(name):
    rel, mx = _table(name)["engine"]
    lim = _limit(name)
    assert rel <= lim[0] and mx <= lim[1], (rel, mx, lim)


@pytest.mark.parametrize("name", list(D.MODELS))
def test_single_fp16_classes_stay_small(name):
    lim = _limit(name)
    for c in _emulation().ENGINE:
        rel, mx = _table(name)[c]
        assert rel <= lim[0] and mx <= lim[1], (c, rel, mx, lim)


@pytest.mark.parametrize("name", ["dinov2_vitg14", "dinov2_vitg14_reg"])
def test_swiglu_inputs_stay_fp32(name):
    """g/14's w12 output stays fp32 for the SwiGLU kernel: rounding it to fp16 as well would add 1.1-1.7e-4 rel-L2 to a
    scheme already at 54-61 % of the bar; keeping it removes at least 15 % of the feature's rel-L2."""
    tab = _table(name)
    assert tab["engine"][0] <= 0.85 * tab["engine + swiglu fp16"][0], tab


@pytest.mark.parametrize("name", ["dinov2_vits14", "dinov2_vitg14_reg"])
def test_a_lost_lo_half_exceeds_the_embedding_bar(name):
    sd = D.prepare(D.stand_in_state_dict(name, depth=1))
    x = D.calibration_frames(1, 2).double()
    ref = D.embed(sd, x, D.ENGINE_FP16)
    lost = D.embed(sd, x, D.ENGINE_FP16 + ("w",))
    d, r = (lost - ref).flatten(1), ref.flatten(1)
    rel = (d.norm(dim=1) / r.norm(dim=1)).max().item()
    mx = (d.abs().amax(dim=1) / r.abs().amax(dim=1)).max().item()
    bar = bars.BARS["embed"]
    assert rel >= bars.SEPARATION * bar[0] and mx >= bars.SEPARATION * bar[1], (rel, mx)

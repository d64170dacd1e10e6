"""The VideoMAE bars (tests/videomae_bars.py) against scripts/precision/emulate_videomae.py, which runs the stand-ins in
float64 with each tensor class either exact (a split-fp16 pair) or rounded to one fp16 value, against the exact
forward, on S, B and L at CONTROL_DEPTH blocks (the full-depth table is in DESIGN.md §4.18).

- The engine's scheme (weights split, every activation class fp16) costs at most SCHEME_FRACTION of the feature bar.
- Weights rounded to fp16 (a lost lo half) move the feature by at least SEPARATION times its bar, and the embedding by
  at least SEPARATION times the embedding bar: the GPU tests, which hold the engine to those bars, catch a lost lo half.
- fp16 weights cost more than all the fp16 activations together (WEIGHT_DOMINANCE times): the mean over 1568 tokens
  averages the activations' roundings away, not the weights', which every token shares.  That is why the weights stay
  split."""
import functools
import importlib.util
import os

import pytest
import torch

import videomae_bars as bars
from oracle import videomae_net as V

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CONTROL_DEPTH = 2


@functools.lru_cache(maxsize=1)
def _emulation():
    path = os.path.join(ROOT, "scripts", "precision", "emulate_videomae.py")
    spec = importlib.util.spec_from_file_location("emulate_videomae", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@functools.lru_cache(maxsize=None)
def _table(name):
    emu = _emulation()
    return emu.table(name, 1, "cpu", {"engine": emu.ENGINE, "fp16 weights": emu.PLAIN_FP16_WEIGHTS}, CONTROL_DEPTH)


NAMES = list(V.SHAPES)


@pytest.mark.parametrize("name", NAMES)
def test_engine_scheme_is_within_its_share_of_the_bar(name):
    bar = bars.FEATURES[V.SHAPES[name][0]]
    rel, mx = _table(name)["engine"]
    assert rel <= bars.SCHEME_FRACTION * bar[0] and mx <= bars.SCHEME_FRACTION * bar[1], (rel, mx, bar)


@pytest.mark.parametrize("name", NAMES)
def test_a_lost_lo_half_exceeds_the_feature_bar(name):
    bar = bars.FEATURES[V.SHAPES[name][0]]
    rel, mx = _table(name)["fp16 weights"]
    assert rel >= bars.SEPARATION * bar[0] and mx >= bars.SEPARATION * bar[1], (rel, mx, bar)


@pytest.mark.parametrize("name", NAMES)
def test_weights_dominate_the_rounding(name):
    tab = _table(name)
    assert tab["fp16 weights"][0] >= bars.WEIGHT_DOMINANCE * tab["engine"][0], tab


@pytest.mark.parametrize("name", ["videomae_vits16", "videomae_vitl16"])
def test_a_lost_lo_half_exceeds_the_embedding_bar(name):
    p = V.prepare(V.stand_in_state_dict(name, depth=1))
    rows = V.tubelets(V.calibration_clips(1, 1).double()).half().double()
    ref = V.embed(p, rows)
    lost = V.embed(p, rows, ("w",))
    d, r = (lost - ref).flatten(1), ref.flatten(1)
    rel = (d.norm(dim=1) / r.norm(dim=1)).max().item()
    mx = (d.abs().amax(dim=1) / r.abs().amax(dim=1)).max().item()
    bar = bars.BARS["embed"]
    assert rel >= bars.SEPARATION * bar[0] and mx >= bars.SEPARATION * bar[1], (rel, mx)


def test_exact_classes_reproduce_the_exact_forward():
    p = V.prepare(V.stand_in_state_dict("videomae_vits16", depth=1))
    x = V.calibration_clips(2, 1).double()
    with torch.no_grad():
        assert torch.equal(V.forward(p, x, fp16=()), V.forward(p, x))
        # the blocked online softmax with P unrounded is the plain softmax
        q, k, v = (torch.randn(1, 2, 200, 64, dtype=torch.float64) * 3 for _ in range(3))
        blocked = V._attention(q, k, v, ("p",))
        assert not torch.equal(blocked, V._attention(q, k, v, ()))
        assert torch.allclose(blocked, V._attention(q, k, v, ()), rtol=1e-3, atol=1e-3)

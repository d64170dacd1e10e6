"""The MViT bars (tests/mvit_bars.py) against scripts/precision/emulate_mvit.py, which runs the stand-in in float64 with
each tensor class either exact (a split-fp16 pair) or rounded to one fp16 value, on the clip of the GPU test's 1-clip
call.  The engine's scheme (weights split, every other class single fp16) must sit under half the feature bar, so the
classes left in single fp16 stay well under it together; rounding the weights as well -- what a lost W_lo half or
pass gives, and what the GPU control runs -- must raise the feature error by SEPARATION; and on mvit_v1_b the weights
alone in single fp16 must cross the 1e-3 feature gate, which is why they are split."""
import importlib.util
import os

import pytest

import mvit_bars as bars

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GATE = 1e-3


@pytest.fixture(scope="module")
def emu():
    path = os.path.join(ROOT, "scripts", "precision", "emulate_mvit.py")
    spec = importlib.util.spec_from_file_location("emulate_mvit", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.mark.parametrize("name", ["mvit_v1_b", "mvit_v2_s"])
def test_split_weights_are_needed_and_enough(emu, name):
    schemes = {"engine": emu.engine_scheme(), "all fp16": emu.CLASSES}
    if name == "mvit_v1_b":
        schemes["w fp16"] = ("w",)
    tab = emu.table(name, 1, "cpu", schemes)
    bar = bars.BARS["features"]
    rel, mx = tab["engine"]["features"]
    assert rel <= bar[0] / 2 and mx <= bar[1] / 2, (rel, mx)
    rel16, _ = tab["all fp16"]["features"]
    assert rel16 >= bars.SEPARATION * rel, (rel16, rel)
    if "w fp16" in tab:
        assert tab["w fp16"]["features"][1] > GATE, tab["w fp16"]["features"]

"""The Swin3D feature bar (tests/swin3d_bars.py) tells the engine's scheme from a lost lo half.
scripts/precision/emulate_swin3d.py runs the stand-in in float64 with each tensor class either exact (a split-fp16
pair) or rounded to one fp16 value.  The engine's scheme (weights split, every other class fp16) must sit under half
the feature bar; the weights alone in single fp16 -- what a lost W_lo half or pass would give -- must exceed it by
SEPARATION; and no class the engine keeps in single fp16 may cost more than half the bar on its own."""
import importlib.util
import os

import pytest

import swin3d_bars as bars

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _emulation():
    path = os.path.join(ROOT, "scripts", "precision", "emulate_swin3d.py")
    spec = importlib.util.spec_from_file_location("emulate_swin3d", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.fixture(scope="module")
def emu():
    return _emulation()


@pytest.mark.parametrize("name", ["swin3d_t", "swin3d_b"])
def test_split_weights_are_needed_and_enough(emu, name):
    fp16_w = ("w",)
    engine = tuple(c for c in emu.CLASSES if c not in emu.SPLIT)
    tab = emu.table(name, 10, "cpu", {"engine": engine, "w fp16": fp16_w})
    bar = bars.BARS["features"]
    rel, mx = tab["engine"]["features"]
    assert rel <= bar[0] / 2 and mx <= bar[1] / 2, (rel, mx)
    rel, mx = tab["w fp16"]["features"]
    assert rel >= bars.SEPARATION * bar[0] and mx >= bars.SEPARATION * bar[1], (rel, mx)


def test_single_fp16_classes_stay_small(emu):
    tab = emu.table("swin3d_t", 10, "cpu", {c: (c,) for c in emu.CLASSES if c not in emu.SPLIT})
    bar = bars.BARS["features"]
    for c, row in tab.items():
        rel, mx = row["features"]
        assert rel <= bar[0] / 2 and mx <= bar[1] / 2, (c, rel, mx)

"""oracle/mvit_net.py against torchvision's own MViT modules and preset, so that the float64 checker of the MViT engine
is pinned: the forward at every tap and at the features on the v1_b / v2_s stand-ins for 1 and 2 clips, the restated
transform bit for bit, and stand-ins whose position terms matter."""
import numpy as np
import pytest
import torch

from oracle import mvit_net as M


def _torchvision_taps(net, x):
    y = net.pos_encoding(net.conv_proj(x).flatten(2).transpose(1, 2))
    taps = {"embed": y}
    thw = (8, 56, 56)
    for i, b in enumerate(net.blocks):
        y, thw = b(y, thw)
        if i in M.STAGE_END:
            taps[f"stage{M.STAGE_END.index(i) + 1}"] = y
    y = net.norm(y)
    taps["norm"] = y
    return y[:, 0], taps


@pytest.mark.parametrize("n", [1, 2])
@pytest.mark.parametrize("name", M.MODELS)
def test_forward_equals_torchvision(name, n):
    sd = M.stand_in_state_dict(name)
    net = M.torchvision_model(name).double().eval()
    net.load_state_dict(sd)
    x = M.calibration_clips(n, n).double()
    with torch.no_grad():
        f, taps = M.forward(sd, x, taps=True)
        ref, ref_taps = _torchvision_taps(net, x)
        logits = net(x)
    for k in M.STAGES:
        assert taps[k].shape == ref_taps[k].shape, k
        rel = float((taps[k] - ref_taps[k]).norm() / ref_taps[k].norm())
        assert rel <= 1e-12, (k, rel)
    assert float((f - ref).norm() / ref.norm()) <= 1e-12
    assert float((M.logits(sd, f) - logits).norm() / logits.norm()) <= 1e-12


@pytest.mark.parametrize("hw", [(240, 320), (320, 240), (360, 640), (256, 256), (100, 100)])
def test_transform_equals_preset_bit_for_bit(hw):
    g = np.random.default_rng(hw[0] * 7 + hw[1])
    rgb = g.integers(0, 256, (3,) + hw + (3,), dtype=np.uint8)
    if hw == (100, 100):                              # an upscaled frame: smooth content so interpolation matters
        rgb = np.repeat(np.repeat(rgb[:, ::4, ::4], 4, 1), 4, 2)[:, :100, :100].copy()
    a = M.transform(rgb)
    for name in M.MODELS:
        b = M.transform_torchvision(rgb, name)
        assert a.shape == b.shape == (3, 3, 224, 224)
        assert torch.equal(a, b), (hw, name)


# (variant, what is zeroed): the stand-in terms torchvision's own init zeroes or shrinks
ABLATIONS = [("mvit_v1_b", "pos_encoding.spatial_pos"), ("mvit_v1_b", "pos_encoding.temporal_pos"),
             ("mvit_v1_b", "pos_encoding.class_pos"), ("mvit_v2_s", ".rel_pos_"), ("mvit_v2_s", "residual pool")]


@pytest.mark.parametrize("name,term", ABLATIONS)
def test_stand_ins_exercise_every_term(name, term, monkeypatch):
    """Zeroing the rel-pos tables, a position embedding or the pooled-q residual moves the features by far more than
    the feature bar (tests/mvit_bars.py)."""
    from mvit_bars import BARS
    sd = {k: v.double() for k, v in M.stand_in_state_dict(name).items()}
    x = M.calibration_clips(0, 1).double()
    with torch.no_grad():
        f = M.forward(sd, x)
        if term == "residual pool":
            attention = M.attention
            monkeypatch.setattr(M, "attention", lambda *a, resid=False: attention(*a, resid=False))
            g = M.forward(sd, x)
        else:
            g = M.forward({k: torch.zeros_like(v) if term in k else v for k, v in sd.items()}, x)
    rel = float((g - f).norm() / f.norm())
    assert rel >= 20 * BARS["features"][0], (name, term, rel)


def test_flop_counts():
    # shape-derived GFLOP of one 16-frame clip: twice torchvision's GMAC metadata (70.6 / 64.2) within the pooling
    # convs, norms and rel-pos dots it also counts
    for name, meta in {"mvit_v1_b": 70.599, "mvit_v2_s": 64.224}.items():
        att, tot = M.flops(name)
        assert 0.95 <= tot / (2 * meta) <= 1.0, (name, tot)
        assert 0.15 <= att / tot <= 0.25, (name, att, tot)

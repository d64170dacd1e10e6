"""oracle/swin3d_net.py against torchvision's own Swin3D modules and preset, so that the float64 checker of the Swin3D
engine is pinned: the forward per stage and at the features on the stand-ins of t / s / b, the restated transform bit
for bit, the arithmetic relative-position index, and the FLOP counts."""
import numpy as np
import pytest
import torch

from oracle import swin3d_net as S


def _torchvision_taps(net, x):
    taps = {}
    y = net.patch_embed(x)
    taps["embed"] = y
    for i, layer in enumerate(net.features):
        y = layer(y)
        if i % 2 == 0:
            taps[f"stage{i // 2 + 1}"] = y
    y = net.norm(y)
    taps["norm"] = y
    return y.permute(0, 4, 1, 2, 3).mean((2, 3, 4)), taps


# T = 32: no temporal padding; 17: T' = 9 padded to 16 with a temporal shift; 10: T' = 5, a clamped window, no shift
@pytest.mark.parametrize("T", [32, 17, 10])
@pytest.mark.parametrize("name", ["swin3d_t", "swin3d_s", "swin3d_b"])
def test_forward_equals_torchvision(name, T):
    sd = S.stand_in_state_dict(name)
    net = S.torchvision_model(name).double().eval()
    net.load_state_dict(sd)
    x = S.calibration_clips(0, 1, T).double()
    with torch.no_grad():
        f, taps = S.forward(sd, x, taps=True)
        ref, ref_taps = _torchvision_taps(net, x)
        logits = net(x)
    for k in S.STAGES:
        rel = float((taps[k] - ref_taps[k]).norm() / ref_taps[k].norm())
        assert rel <= 1e-12, (k, rel)
    assert float((f - ref).norm() / ref.norm()) <= 1e-12
    assert float((S.logits(sd, f) - logits).norm() / logits.norm()) <= 1e-12


def test_config_from_weights():
    for name, (dim, depths) in S.MODELS.items():
        sd = S.stand_in_state_dict(name)
        assert S.config(sd) == (dim, depths)
        assert S.config({"module." + k: v for k, v in sd.items()}) == (dim, depths)
        assert sd["norm.weight"].numel() == 8 * dim


def test_bias_index_equals_the_stored_buffer():
    for name in S.MODELS:
        sd = S.stand_in_state_dict(name)
        for key in [k for k in sd if k.endswith("relative_position_index")]:
            idx = sd[key]
            assert torch.equal(S.bias_index((8, 7, 7)), idx)
            for tq in (7, 5, 2, 1):                   # a window clamped to T' <= 8: relative_position_index[:vol, :vol]
                vol = tq * 49
                assert torch.equal(S.bias_index((tq, 7, 7)), idx[:vol, :vol])


@pytest.mark.parametrize("hw", [(240, 320), (320, 240), (360, 640), (720, 1280), (256, 256), (100, 100)])
def test_transform_equals_preset_bit_for_bit(hw):
    g = np.random.default_rng(hw[0] * 7 + hw[1])
    rgb = g.integers(0, 256, (3,) + hw + (3,), dtype=np.uint8)
    if hw == (100, 100):                              # an upscaled frame: smooth content so interpolation matters
        rgb = np.repeat(np.repeat(rgb[:, ::4, ::4], 4, 1), 4, 2)[:, :100, :100].copy()
    a, b = S.transform(rgb), S.transform_torchvision(rgb)
    assert a.shape == b.shape == (3, 3, 224, 224)
    assert torch.equal(a, b), hw


def test_flop_counts():
    # shape-derived counts for one 32-frame clip at 224 x 224: (window attention, total) GFLOP
    for name, (att, tot) in {"swin3d_t": (36, 176), "swin3d_s": (59, 331), "swin3d_b": (78, 563)}.items():
        a, t = S.flops(name, 32)
        assert round(a) == att and round(t) == tot, (name, a, t)

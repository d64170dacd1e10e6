"""oracle/s3d_net.py against torchvision: the functional forward against ``torchvision.models.video.s3d()`` with the
stand-in, the temporal sizes, the restated transform against ``S3D_Weights.KINETICS400_V1.transforms()`` bit for bit,
and the stand-in's calibration."""
import numpy as np
import pytest
import torch
import torchvision

from oracle import s3d_net


@pytest.fixture(scope="module")
def net():
    m = torchvision.models.video.s3d()
    m.load_state_dict(s3d_net.stand_in_state_dict())
    return m.eval()


@pytest.mark.parametrize("T,n", [(13, 1), (16, 2), (17, 1)])
def test_oracle_equals_torchvision(net, T, n):
    sd = s3d_net.stand_in_state_dict()
    x = s3d_net.calibration_clips(seed=T, n=n, T=T)
    with torch.no_grad():
        y = s3d_net.forward(sd, x)
        ref = net.avgpool(net.features(x)).mean(dim=(2, 3, 4))
        assert y.shape == (n, 1024)
        torch.testing.assert_close(y, ref, rtol=1e-5, atol=1e-6)
        # the head on the feature equals model(x): linear head, identity dropout
        torch.testing.assert_close(s3d_net.logits(sd, y), net(x), rtol=1e-4, atol=1e-5)


@pytest.mark.parametrize("T", list(range(13, 21)) + [64])
def test_temporal_sizes_match_torchvision(net, T):
    sd = {k: v.to("meta") for k, v in s3d_net.stand_in_state_dict().items()}
    _, taps = s3d_net.forward(sd, torch.zeros(1, 3, T, 224, 224, device="meta"), taps=True)
    T1, T2, T3 = s3d_net.temporal_sizes(T)
    assert taps["stem"].shape[2:] == (T1, 112, 112) and taps["mixed_3c"].shape[2:] == (T1, 28, 28)
    assert taps["mixed_4f"].shape[2:] == (T2, 14, 14) and taps["mixed_5c"].shape[2:] == (T3, 7, 7)
    with torch.no_grad():
        y = net.features(torch.zeros(1, 3, T, 64, 64))     # torchvision's own temporal size (spatial size aside)
    assert y.shape[2] == T3


def test_twelve_frames_are_too_few(net):
    with pytest.raises(RuntimeError):
        with torch.no_grad():
            net(torch.zeros(1, 3, 12, 224, 224))
    assert s3d_net.temporal_sizes(12)[2] == 1 and s3d_net.temporal_sizes(13)[2] == 2


@pytest.mark.parametrize("hw", [(240, 320), (360, 480), (100, 60), (256, 256), (480, 640), (720, 1280)])
def test_transform_is_the_preset_bit_for_bit(hw):
    g = np.random.default_rng(hw[0] * 7 + hw[1])
    rgb = g.integers(0, 256, (3, *hw, 3), dtype=np.uint8)
    a = s3d_net.transform(rgb)
    b = s3d_net.transform_torchvision(rgb)
    assert a.shape == b.shape == (3, 3, 224, 224)
    assert torch.equal(a, b)
    assert s3d_net.crop_offset(256) == 16


def test_stand_in_is_deterministic_and_alive():
    a, b = s3d_net.stand_in_state_dict(0), s3d_net.stand_in_state_dict(0)
    assert a.keys() == b.keys() and all(torch.equal(a[k], b[k]) for k in a)
    assert "classifier.1.weight" in a and tuple(a["classifier.1.weight"].shape) == (400, 1024, 1, 1, 1)
    x = s3d_net.calibration_clips(seed=5, n=1, T=16)
    with torch.no_grad():
        y, taps = s3d_net.forward(a, x, taps=True)
    for name, t in taps.items():
        live = (t > 0).double().mean().item()
        assert 0.3 < live < 0.7, (name, live)
        assert 0.3 < t.std().item() < 3, (name, t.std().item())
    assert y.abs().max().item() > 0.1

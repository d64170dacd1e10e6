"""The ResNet oracle (oracle/resnet_net.py) against live torchvision, the calibrated stand-in, and the fixture made by
the reference's own ExtractResNet (tests/golden/resnet_outputs.npz)."""
import os

import numpy as np
import pytest
import torch

from oracle import resnet_net

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")


@pytest.mark.parametrize("depth", [18, 34, 50, 101, 152])
def test_oracle_matches_torchvision(depth):
    import torchvision
    sd = resnet_net.stand_in_state_dict(depth)
    net = getattr(torchvision.models, f"resnet{depth}")(weights=None)
    net.load_state_dict(sd)
    net.fc = torch.nn.Identity()
    net.eval()
    x = resnet_net.calibration_images(seed=7, n=2)
    with torch.no_grad():
        ref = net(x)
        y, taps = resnet_net.forward(sd, x, depth, taps=True)
    assert y.shape == (2, resnet_net.out_dim(depth))
    rel = float((y - ref).norm() / ref.norm())
    assert rel < 1e-5, rel
    # the stand-in is calibrated: every stage's activations are O(1), not vanishing or exploding with depth
    for name in resnet_net.STAGES:
        rms = float(taps[name].pow(2).mean().sqrt())
        assert 0.05 < rms < 20, (name, rms)


def test_stand_in_is_deterministic():
    a = resnet_net.stand_in_state_dict(18)
    resnet_net._stand_in.cache_clear()
    b = resnet_net.stand_in_state_dict(18)
    assert a.keys() == b.keys()
    assert all(torch.equal(a[k], b[k]) for k in a)
    assert not torch.equal(a["bn1.weight"], resnet_net.stand_in_state_dict(18, seed=1)["bn1.weight"])
    # branch damping: the last BatchNorm of a residual branch has gains in [0.125, 0.375]
    g = a["layer2.1.bn2.weight"]
    assert float(g.min()) >= 0.125 and float(g.max()) <= 0.375


def _decoded_frames():
    import cv2
    cap = cv2.VideoCapture(os.path.join(GOLDEN, "v_GGSY1Qvo990.mp4"))
    frames = []
    first = True
    while cap.isOpened():
        ok, f = cap.read()
        if first:
            first = False
            if ok is False:
                continue
        if not ok:
            break
        frames.append(f)
    cap.release()
    return frames


def test_transform_and_features_vs_reference_fixture():
    g = np.load(os.path.join(GOLDEN, "resnet_outputs.npz"))
    frames = _decoded_frames()
    assert len(frames) == len(g["transform_sha1"]) == 355
    xs = [resnet_net.transform(f) for f in frames]
    # the restated transform is bit-exact with the reference's torchvision Compose on every frame
    assert [resnet_net.tensor_hash(x) for x in xs] == list(g["transform_sha1"])
    rows = g["rows"]
    x = torch.stack([xs[i] for i in rows])
    for depth in (18, 50):
        with torch.no_grad():
            y = resnet_net.forward(resnet_net.stand_in_state_dict(depth), x, depth).double()
        ref = torch.from_numpy(g[f"resnet{depth}"])
        assert ref.shape == (len(rows), resnet_net.out_dim(depth))
        rel = ((y - ref).norm(dim=1) / ref.norm(dim=1)).max().item()
        assert rel < 1e-5, (depth, rel)

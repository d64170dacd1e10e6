"""The R(2+1)D oracle (oracle/r21d_net.py) against live torchvision, the calibrated stand-in, the transform restated for
the CUDA kernel, and the fixture made from the reference's own transform and slicing (tests/golden/r21d_outputs.npz)."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import r21d_net

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
REFERENCE = os.environ.get("VF_REFERENCE_DIR", "/root/reference")     # a checkout of the upstream project, as oracle/fetch_ref.py


def test_oracle_matches_torchvision():
    import torchvision
    sd = r21d_net.stand_in_state_dict()
    net = torchvision.models.video.r2plus1d_18(weights=None)
    net.load_state_dict(sd)
    net.fc = torch.nn.Identity()
    net.eval()
    x = r21d_net.calibration_clips(seed=7, n=2, T=7)       # odd T: temporal sizes 7, 4, 2, 1
    with torch.no_grad():
        ref = net(x)
        y, taps = r21d_net.forward(sd, x, taps=True)
    assert y.shape == (2, 512)
    rel = float((y - ref).norm() / ref.norm())
    assert rel < 1e-5, rel
    assert [tuple(taps[s].shape[1:3]) for s in r21d_net.STAGES] == [(64, 7), (64, 7), (128, 4), (256, 2), (512, 1)]
    # the stand-in is calibrated: every stage's activations are O(1), not vanishing or exploding with depth
    for name in r21d_net.STAGES:
        rms = float(taps[name].pow(2).mean().sqrt())
        assert 0.05 < rms < 20, (name, rms)


def test_stand_in_is_deterministic():
    a = r21d_net.stand_in_state_dict()
    r21d_net._stand_in.cache_clear()
    b = r21d_net.stand_in_state_dict()
    assert a.keys() == b.keys()
    assert all(torch.equal(a[k], b[k]) for k in a)
    assert not torch.equal(a["stem.1.weight"], r21d_net.stand_in_state_dict(seed=1)["stem.1.weight"])
    # branch damping: the last BatchNorm of a residual branch has gains in [0.125, 0.375]
    g = a["layer2.1.conv2.1.weight"]
    assert float(g.min()) >= 0.125 and float(g.max()) <= 0.375


def decoded_rgb():
    """The sample video through OpenCV, BGR -> RGB: (T, H, W, 3) uint8 (read_video's layout)."""
    import cv2
    cap = cv2.VideoCapture(os.path.join(GOLDEN, "v_GGSY1Qvo990.mp4"))
    frames = []
    while True:
        ok, f = cap.read()
        if not ok:
            break
        frames.append(f[:, :, ::-1])
    cap.release()
    return np.stack(frames)


def test_transform_and_features_vs_reference_fixture():
    g = np.load(os.path.join(GOLDEN, "r21d_outputs.npz"))
    rgb = decoded_rgb()
    assert len(rgb) == int(g["n_frames"]) == 355
    slices = r21d_net.form_slices(len(rgb), 16, 16)
    assert len(slices) == len(g["transform_sha1"]) == 22
    x = r21d_net.transform(rgb)
    # the restated transform is bit-exact with the reference's Compose on every stack
    assert [r21d_net.tensor_hash(x[:, s:e]) for s, e in slices] == list(g["transform_sha1"])
    clips = torch.stack([x[:, s:e] for s, e in slices])
    with torch.no_grad():
        y = r21d_net.forward(r21d_net.stand_in_state_dict(), clips).double()
    ref = torch.from_numpy(g["r21d_rgb"])
    assert ref.shape == (22, 512) and ref.dtype == torch.float64
    rel = ((y - ref).norm(dim=1) / ref.norm(dim=1)).max().item()
    assert rel < 1e-5, rel


GEOMETRIES = [(240, 320), (360, 480), (100, 60), (128, 171), (113, 200), (720, 1280)]


def _frames(h, w, n=3, seed=0):
    g = np.random.default_rng(seed + h * 7 + w)
    return g.integers(0, 256, (n, h, w, 3), dtype=np.uint8)


@pytest.mark.parametrize("hw", GEOMETRIES)
def test_kernel_resize_arithmetic_is_torch_exact(hw):
    """The source-index / weight / blend arithmetic the CUDA transform uses (oracle.r21d_net.resize_restated) gives
    torch's CPU upsample_bilinear2d bit for bit, down- and upsampling."""
    x = torch.from_numpy(_frames(*hw)).permute(3, 0, 1, 2).to(torch.float32) / 255
    ref = F.interpolate(x, size=(128, 171), mode="bilinear", align_corners=False).numpy()
    got = r21d_net.resize_restated(x.numpy(), 128, 171)
    assert np.array_equal(got, ref), (np.mean(got != ref), np.abs(got - ref).max())


@pytest.mark.parametrize("hw", GEOMETRIES)
def test_transform_vs_reference_compose(hw):
    """oracle.r21d_net.transform against the reference's own rgb_transforms, imported from a reference checkout."""
    if not os.path.isdir(os.path.join(REFERENCE, "models", "r21d")):
        pytest.skip("no reference checkout")
    import importlib.util
    spec = importlib.util.spec_from_file_location(
        "ref_rgb_transforms", os.path.join(REFERENCE, "models", "r21d", "transforms", "rgb_transforms.py"))
    T = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(T)
    rgb = _frames(*hw, n=4, seed=1)
    vid = torch.from_numpy(rgb)
    for tf in (T.ToFloatTensorInZeroOne(), T.Resize((128, 171)),
               T.Normalize(mean=r21d_net.KINETICS_MEAN, std=r21d_net.KINETICS_STD), T.CenterCrop((112, 112))):
        vid = tf(vid)
    assert torch.equal(r21d_net.transform(rgb), vid)

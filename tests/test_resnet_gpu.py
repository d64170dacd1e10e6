"""ResNetEngine (vf_resnet_*) against the plain-torch fp32 oracle (oracle/resnet_net.py) on calibrated stand-in weights."""
import numpy as np
import pytest
import torch

from oracle import resnet_net

pytestmark = pytest.mark.gpu

# per-stage rel-L2 bars of read_stage against the oracle's taps: the trunk carries every operand as a split-fp16 pair
# (emulated fp32), so a stage far above the fp32-class error points at that stage
STAGE_BAR = {"stem": 1e-5, "maxpool": 1e-5, "layer1": 2e-5, "layer2": 1e-4, "layer3": 5e-4, "layer4": 1e-3}


def frames_bgr(n, h=256, w=341, seed=0):
    """n smooth random uint8 BGR frames, already at the resized geometry."""
    g = torch.Generator().manual_seed(seed)
    low = torch.rand(n, 3, 12, 16, generator=g)
    img = torch.nn.functional.interpolate(low, size=(h, w), mode="bilinear", align_corners=False)
    img = img * 0.85 + 0.15 * torch.rand(n, 3, h, w, generator=g)
    return img.mul(255).round().clamp(0, 255).to(torch.uint8).permute(0, 2, 3, 1).contiguous()


def normalised(u8_bgr):
    return torch.stack([resnet_net.normalize(f[:, :, ::-1].copy()) for f in u8_bgr.numpy()])


def row_errors(y, ref):
    y, ref = y.double().cpu(), ref.double().cpu()
    rel = ((y - ref).norm(dim=1) / ref.norm(dim=1)).max().item()
    mx = ((y - ref).abs().amax(dim=1) / ref.abs().amax(dim=1)).max().item()
    return rel, mx


@pytest.mark.parametrize("depth", [18, 34, 50, 101, 152])
def test_engine_vs_oracle(cuda_device, depth):
    from video_features_b200.resnet_engine import ResNetEngine
    sd = resnet_net.stand_in_state_dict(depth)
    sdg = {k: v.to(cuda_device) for k, v in sd.items()}
    eng = ResNetEngine(sd, depth, 0, max_frames=20)
    for n in (5, 37):                              # 37 frames: two internal chunks of the 20-frame workspace
        x = normalised(frames_bgr(n, seed=n)).to(cuda_device)
        y = eng.forward_f32(x)
        with torch.no_grad():
            ref, taps = resnet_net.forward(sdg, x, depth, taps=True)
        assert y.shape == (n, resnet_net.out_dim(depth))
        rel, mx = row_errors(y, ref)
        print(f"resnet{depth} n={n}: worst row rel-L2 {rel:.2e}, max-abs/max {mx:.2e}")
        assert rel <= 1e-3 and mx <= 1e-3, (rel, mx)
        m = n if n <= 20 else n - 20                # read_stage holds the last chunk
        for sid, name in enumerate(resnet_net.STAGES):
            got = eng.read_stage(sid)
            want = taps[name][n - m:]
            assert got.shape == want.shape, (name, got.shape, want.shape)
            srel = float((got.double() - want.double()).norm() / want.double().norm())
            print(f"  {name}: rel-L2 {srel:.2e}")
            assert srel <= STAGE_BAR[name], (name, srel)
    assert eng.launch_count > 0
    eng.close()


def test_u8_entry_and_call_splits_are_bit_identical(cuda_device):
    from video_features_b200.resnet_engine import ResNetEngine
    sd = resnet_net.stand_in_state_dict(50)
    eng = ResNetEngine(sd, 50, 0, max_frames=16)
    u8 = frames_bgr(37, seed=3)
    x = normalised(u8).to(cuda_device)
    a = eng.forward_f32(x)
    b = eng.forward_u8(u8.to(cuda_device))          # fused transform: bit-exact with the f32 entry's input
    assert torch.equal(a, b)
    parts = torch.cat([eng.forward_u8(u8[i:j].to(cuda_device)) for i, j in ((0, 5), (5, 21), (21, 37))])
    assert torch.equal(a, parts)
    # a wider resized frame (short side 256, long side 455) crops at its own centre
    u8w = frames_bgr(3, 256, 455, seed=4)
    ref = eng.forward_f32(normalised(u8w).to(cuda_device))
    assert torch.equal(eng.forward_u8(u8w.to(cuda_device)), ref)
    eng.close()


def test_errors(cuda_device):
    from video_features_b200._lib import VfError
    from video_features_b200.resnet_engine import ResNetEngine
    sd = resnet_net.stand_in_state_dict(18)
    with pytest.raises(VfError, match="depth 20"):
        ResNetEngine(sd, 20, 0)
    bad = dict(sd)
    del bad["layer3.1.bn2.running_var"]
    with pytest.raises(VfError, match="missing tensor 'layer3.1.bn2.running_var'"):
        ResNetEngine(bad, 18, 0)
    bad = dict(sd)
    bad["layer2.0.downsample.0.weight"] = torch.zeros(128, 64, 3, 3)
    with pytest.raises(VfError, match="layer2.0.downsample.0.weight"):
        ResNetEngine(bad, 18, 0)
    # basic-block weights for a bottleneck depth: layer1.0.conv1 is 3x3 there, 1x1 in a bottleneck
    with pytest.raises(VfError, match="'layer1.0.conv1.weight' has 36864 elements, expected 4096"):
        ResNetEngine(sd, 50, 0)
    # DataParallel's "module." prefix is accepted
    eng = ResNetEngine({"module." + k: v for k, v in sd.items()}, 18, 0, max_frames=4)
    with pytest.raises(VfError, match="smaller than the 224 crop"):
        eng.forward_u8(torch.zeros(2, 223, 300, 3, dtype=torch.uint8, device=cuda_device))
    y = eng.forward_u8(frames_bgr(2, 224, 298).to(cuda_device))
    assert y.shape == (2, 512) and torch.isfinite(y).all()
    eng.close()

"""R21DEngine (vf_r21d_*) against the plain-torch fp32 oracle (oracle/r21d_net.py) on calibrated stand-in weights."""
import numpy as np
import pytest
import torch

from oracle import r21d_net

pytestmark = pytest.mark.gpu

# per-stage rel-L2 bars of read_stage against the oracle's taps: the trunk carries every operand as a split-fp16 pair
# (emulated fp32), so a stage far above the fp32-class error points at that stage
STAGE_BAR = {"stem": 1e-5, "layer1": 3e-5, "layer2": 1e-4, "layer3": 3e-4, "layer4": 1e-3}


def frames_bgr(n, h=240, w=320, seed=0):
    """n smooth random uint8 BGR frames, slowly changing in time."""
    g = torch.Generator().manual_seed(seed)
    low = torch.rand(1, 3, max(n // 4, 2), 8, 10, generator=g)
    vid = torch.nn.functional.interpolate(low, size=(n, h, w), mode="trilinear", align_corners=False)[0]
    vid = vid * 0.85 + 0.15 * torch.rand(3, n, h, w, generator=g)
    return vid.mul(255).round().clamp(0, 255).to(torch.uint8).permute(1, 2, 3, 0).contiguous()


def clips_f32(u8_bgr, starts, T):
    """The oracle transform (the reference's Compose) of each clip of RGB frames: (n, 3, T, 112, 112)."""
    rgb = u8_bgr.numpy()[..., ::-1].copy()
    return torch.stack([r21d_net.transform(rgb[s:s + T]) for s in starts])


def row_errors(y, ref):
    y, ref = y.double().cpu(), ref.double().cpu()
    rel = ((y - ref).norm(dim=1) / ref.norm(dim=1)).max().item()
    mx = ((y - ref).abs().amax(dim=1) / ref.abs().amax(dim=1)).max().item()
    return rel, mx


@pytest.mark.parametrize("T", [16, 7])
def test_engine_vs_oracle(cuda_device, T):
    from video_features_b200.r21d_engine import R21DEngine
    sd = r21d_net.stand_in_state_dict()
    sdg = {k: v.to(cuda_device) for k, v in sd.items()}
    eng = R21DEngine(sd, 0, max_clips=2, max_T=16)     # 36 frame slots: 2 clips of 16, or 4 of 7, per chunk
    per_chunk = 36 // (T + 2)
    for n in (1, per_chunk + 1):                        # one chunk, then two
        u8 = frames_bgr(n * T, seed=n + T)
        x = clips_f32(u8, [i * T for i in range(n)], T).to(cuda_device)
        y = eng.forward_f32(x)
        with torch.no_grad():
            ref, taps = r21d_net.forward(sdg, x, taps=True)
        assert y.shape == (n, 512)
        rel, mx = row_errors(y, ref)
        print(f"r21d T={T} n={n}: worst row rel-L2 {rel:.2e}, max-abs/max {mx:.2e}")
        assert rel <= 1e-3 and mx <= 1e-3, (rel, mx)
        m = n if n <= per_chunk else n - per_chunk      # read_stage holds the last chunk
        for sid, name in enumerate(r21d_net.STAGES):
            got = eng.read_stage(sid)
            want = taps[name][n - m:]
            assert got.shape == want.shape, (name, got.shape, want.shape)
            srel = float((got.double() - want.double()).norm() / want.double().norm())
            print(f"  {name}: rel-L2 {srel:.2e}")
            assert srel <= STAGE_BAR[name], (name, srel)
    assert eng.launch_count > 0
    eng.close()


@pytest.mark.parametrize("hw", [(240, 320), (100, 60), (360, 480)])
def test_u8_entry_and_call_splits_are_bit_identical(cuda_device, hw):
    from video_features_b200.r21d_engine import R21DEngine
    sd = r21d_net.stand_in_state_dict()
    eng = R21DEngine(sd, 0, max_clips=2, max_T=16)
    T, step = 16, 8                                     # overlapping stacks share frames
    u8 = frames_bgr(56, *hw, seed=sum(hw))
    starts = [s for s, _ in r21d_net.form_slices(56, T, step)]
    a = eng.forward_f32(clips_f32(u8, starts, T).to(cuda_device))
    ud = u8.to(cuda_device)
    b = eng.forward_u8(ud, starts, T)                   # fused transform: bit-exact with the oracle transform
    assert torch.equal(a, b)
    parts = torch.cat([eng.forward_u8(ud, starts[i:j], T) for i, j in ((0, 1), (1, 4), (4, len(starts)))])
    assert torch.equal(a, parts)
    # the same clips from a buffer that holds only their frames (the extractor's compacted window)
    c = eng.forward_u8(ud[8:40], [0, 8, 16], T)
    assert torch.equal(c, a[1:4])
    eng.close()


def test_odd_stack_and_gaps(cuda_device):
    """stack 5 / step 9: frames between stacks are never read; any stack size works, including T = 1."""
    from video_features_b200.r21d_engine import R21DEngine
    sd = r21d_net.stand_in_state_dict()
    eng = R21DEngine(sd, 0, max_clips=2, max_T=16)
    u8 = frames_bgr(40, seed=9)
    for T, step in ((5, 9), (1, 3)):
        starts = [s for s, _ in r21d_net.form_slices(40, T, step)]
        a = eng.forward_u8(u8.to(cuda_device), starts, T)
        ref = r21d_net.forward({k: v.to(cuda_device) for k, v in sd.items()},
                               clips_f32(u8, starts, T).to(cuda_device))
        rel, mx = row_errors(a, ref)
        print(f"T={T} step={step} ({len(starts)} clips): worst row rel-L2 {rel:.2e}, max-abs/max {mx:.2e}")
        assert rel <= 1e-3 and mx <= 1e-3, (rel, mx)
    eng.close()


def test_errors(cuda_device):
    from video_features_b200._lib import VfError
    from video_features_b200.r21d_engine import R21DEngine
    sd = r21d_net.stand_in_state_dict()
    bad = dict(sd)
    del bad["layer3.1.conv2.1.running_var"]
    with pytest.raises(VfError, match="missing tensor 'layer3.1.conv2.1.running_var'"):
        R21DEngine(bad, 0)
    bad = dict(sd)
    bad["layer2.0.downsample.0.weight"] = torch.zeros(128, 64, 1, 3, 3)
    with pytest.raises(VfError, match="layer2.0.downsample.0.weight"):
        R21DEngine(bad, 0)
    # DataParallel's "module." prefix is accepted
    eng = R21DEngine({"module." + k: v for k, v in sd.items()}, 0, max_clips=1, max_T=8)
    u8 = frames_bgr(12, seed=1).to(cuda_device)
    with pytest.raises(VfError, match="outside the 12 frames"):
        eng.forward_u8(u8, [0, 5], 8)
    with pytest.raises(VfError, match="exceeds the workspace"):
        eng.forward_u8(u8, [0], 9)
    y = eng.forward_u8(u8, [0, 4], 8)
    assert y.shape == (2, 512) and torch.isfinite(y).all()
    assert eng.forward_u8(u8, [], 8).shape == (0, 512)
    eng.close()

"""The front end the single-frame towers share (CLIP ViT-B / ViT-L / ResNet, DINOv2): the resize scratch a handle grows
for a larger frame size serves a smaller one again with unchanged bits; each handle's graph admission policy (the ViT
towers capture a chunk size on its second sighting and keep at most 32 / 16 graphs, DINOv2 captures on first use) is
visible through VF_GRAPH_TRACE=1 and gives the eager bits and launch count on every call."""
import pytest
import torch

from oracle import clip_resnet, dinov2_net
from video_features_b200 import synthetic_weights

pytestmark = pytest.mark.gpu


def _frames(n, h, w, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, 256, (n, h, w, 3), dtype=torch.uint8, generator=g)


def _vit_b(sd):
    from video_features_b200.clip_engine import ClipEngine
    eng = ClipEngine(sd, 0, chunk_frames=2)
    return eng, eng.encode_frames_u8


def _vit_l(sd):
    from video_features_b200.clip_vitl_engine import ClipViTLEngine
    eng = ClipViTLEngine(sd, 0, max_frames=2)
    return eng, eng.encode_frames_u8


def _rn(sd):
    from video_features_b200.clip_resnet_engine import ClipResNetEngine
    eng = ClipResNetEngine(sd, 0, max_frames=2)
    return eng, eng.encode_frames_u8


def _dinov2(sd):
    from video_features_b200.dinov2_engine import DINOv2Engine
    eng = DINOv2Engine(sd, 0, max_frames=2)
    return eng, eng.encode_u8


TOWERS = {
    "ViT-B/32": (_vit_b, lambda: synthetic_weights.clip_vit_b32_state_dict(0)),
    "ViT-L/14": (_vit_l, lambda: synthetic_weights.clip_vit_l14_state_dict(0)),
    "RN50": (_rn, lambda: clip_resnet.stand_in_state_dict("RN50")),
    "DINOv2 ViT-S/14": (_dinov2, lambda: dinov2_net.stand_in_state_dict("dinov2_vits14")),
}


@pytest.mark.parametrize("tower", list(TOWERS))
def test_resize_scratch_regrows_and_serves_smaller_frames(cuda_device, tower):
    """Small frames, then larger ones (the scratch is re-allocated), then the small ones again on one handle: each call
    equals a fresh handle's output for the same frames.  Three frames per call: two chunks of the handle."""
    make, weights = TOWERS[tower]
    sd = weights()
    small, large = _frames(3, 181, 241, 1).to(cuda_device), _frames(3, 301, 409, 2).to(cuda_device)
    eng, encode = make(sd)
    got = [encode(small), encode(large), encode(small)]
    torch.cuda.synchronize()
    eng.close()
    for frames, y in ((small, got[0]), (large, got[1]), (small, got[2])):
        fresh, fresh_encode = make(sd)
        want = fresh_encode(frames)
        torch.cuda.synchronize()
        fresh.close()
        assert torch.equal(y, want), tower


def _captures(capfd):
    """The graph captures VF_GRAPH_TRACE=1 reported on stderr since the last call."""
    return [line for line in capfd.readouterr().err.splitlines() if "graph captured" in line]


@pytest.mark.parametrize("tower", ["ViT-B/32", "ViT-L/14", "DINOv2 ViT-S/14"])
def test_chunk_size_is_captured_on_the_towers_sighting(cuda_device, tower, monkeypatch, capfd):
    """The ViT towers run a chunk size eagerly the first time, capture it the second and replay it the third; DINOv2
    captures on first use.  Every call gives the same bits and launch count as a handle that never captures
    (VF_NO_GRAPH=1)."""
    make, weights = TOWERS[tower]
    sd = weights()
    frames = _frames(2, 200, 260, 3).to(cuda_device)
    monkeypatch.setenv("VF_GRAPH_TRACE", "1")
    eng, encode = make(sd)
    capture_on = 1 if tower.startswith("DINOv2") else 2
    ys, counts = [], []
    _captures(capfd)
    for call in (1, 2, 3):
        before = eng.launch_count
        ys.append(encode(frames))
        torch.cuda.synchronize()
        counts.append(eng.launch_count - before)
        assert len(_captures(capfd)) == (call == capture_on), (tower, call)
    eng.close()
    monkeypatch.setenv("VF_NO_GRAPH", "1")
    eager, encode = make(sd)
    before = eager.launch_count
    y_eager = encode(frames)
    torch.cuda.synchronize()
    eager_count = eager.launch_count - before
    eager.close()
    assert counts[0] > 0 and counts == [eager_count] * 3, counts
    for y in ys:
        assert torch.equal(y, y_eager)


def test_vit_b_keeps_32_graphs_and_runs_further_sizes_eagerly(cuda_device, monkeypatch, capfd):
    """ViT-B's cache holds 32 chunk sizes; a 33rd size seen twice is not captured (and nothing is evicted), and its
    output equals the eager one."""
    from video_features_b200.clip_engine import ClipEngine
    sd = TOWERS["ViT-B/32"][1]()
    monkeypatch.setenv("VF_GRAPH_TRACE", "1")
    eng = ClipEngine(sd, 0, chunk_frames=40)
    frames = _frames(33, 224, 224, 4).to(cuda_device)
    _captures(capfd)
    for n in range(1, 34):
        eng.encode_frames_u8(frames[:n])
        y = eng.encode_frames_u8(frames[:n])
    torch.cuda.synchronize()
    captures = _captures(capfd)
    assert len(captures) == 32 and captures[-1].endswith("32 cached"), captures[-3:]
    eng.close()
    monkeypatch.setenv("VF_NO_GRAPH", "1")
    eager = ClipEngine(sd, 0, chunk_frames=40)
    y_eager = eager.encode_frames_u8(frames)
    torch.cuda.synchronize()
    eager.close()
    assert torch.equal(y, y_eager)

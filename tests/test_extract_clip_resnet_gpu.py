"""ExtractCLIP with the ResNet towers end to end: the stand-in written to a checkpoint file (read back through
$VF_CLIP_CKPT and read_clip_checkpoint), decode -> sampler -> fused resize / crop / normalise + tower, against the fp32
oracle on the very same decoded frames; the batched list path against per-video calls; --output_direct files."""
import argparse
import os

import numpy as np
import pytest
import torch

from oracle import clip_resnet

pytestmark = pytest.mark.gpu

SAMPLE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "v_GGSY1Qvo990.mp4")


def _args(paths, out, feature_type, method, **kw):
    d = dict(feature_type=feature_type, video_paths=paths, flow_paths=None, file_with_video_paths=None,
             video_dir=None, flow_dir=None, extraction_fps=None, extract_method=method, on_extraction='save_numpy',
             output_path=out, output_direct=True, tmp_path=os.path.join(out, 'tmp'))
    d.update(kw)
    return argparse.Namespace(**d)


def _stand_in_file(tmp_path, name, monkeypatch):
    sd = clip_resnet.stand_in_state_dict(name)
    path = str(tmp_path / f"{name}.pt")
    torch.save(sd, path)
    monkeypatch.setenv("VF_CLIP_CKPT", path)
    monkeypatch.delenv("VF_CLIP_SYNTHETIC", raising=False)
    return sd


def _oracle(sd, frames, dev):
    x = clip_resnet.preprocess_batch(frames, clip_resnet.config(sd)["n_px"]).to(dev)
    with torch.no_grad():
        return clip_resnet.forward({k: v.to(dev) for k, v in sd.items()}, x).cpu().numpy()


def _rel(a, b):
    return float((np.linalg.norm(a - b, axis=1) / np.linalg.norm(b, axis=1)).max())


@pytest.mark.parametrize("feature_type,method,dim", [("CLIP-RN50", "uni_12", 1024), ("CLIP-RN50x4", "uni_3", 640)])
def test_external_call_matches_oracle(cuda_device, tmp_path, monkeypatch, feature_type, method, dim):
    from video_features_b200 import utils
    from video_features_b200.extract.extract_clip import ExtractCLIP
    sd = _stand_in_file(tmp_path, feature_type[5:], monkeypatch)
    ex = ExtractCLIP(_args([SAMPLE], str(tmp_path / "o"), feature_type, method), external_call=True)
    d = ex(torch.zeros([1], dtype=torch.long, device=cuda_device))[0]
    assert set(d) == {feature_type, 'fps', 'timestamps_ms'}
    f = d[feature_type]
    assert f.shape == (int(method.split("_")[1]), dim) and f.dtype == np.float32
    frames = utils.extract_frames(SAMPLE, method)[0]
    rel = _rel(f, _oracle(sd, frames, cuda_device))
    print(f"{feature_type} {method}: worst row rel-L2 vs fp32 oracle {rel:.2e}")
    assert rel < 1e-3, rel


def test_batched_list_equals_per_video_and_writes_files(cuda_device, tmp_path, monkeypatch):
    import cv2
    from video_features_b200.extract.extract_clip import ExtractCLIP
    _stand_in_file(tmp_path, "RN50", monkeypatch)
    small = str(tmp_path / "small.mp4")                  # a second geometry: 120 x 160
    vw = cv2.VideoWriter(small, cv2.VideoWriter_fourcc(*"mp4v"), 10.0, (160, 120))
    rng = np.random.default_rng(0)
    base = rng.integers(0, 256, (120, 160, 3), dtype=np.uint8)
    for i in range(20):
        vw.write(np.roll(base, 3 * i, axis=1))
    vw.release()
    vids = [SAMPLE, small]
    out = str(tmp_path / "out")
    ex = ExtractCLIP(_args(vids, out, "CLIP-RN50", "uni_5"))
    ex(torch.arange(2, device=cuda_device))                  # the batched list path, save_numpy --output_direct
    one = ExtractCLIP(_args(vids, out, "CLIP-RN50", "uni_5"), external_call=True)
    for i, v in enumerate(vids):
        saved = np.load(os.path.join(out, os.path.splitext(os.path.basename(v))[0] + ".npy"))
        alone = one(torch.tensor([i], device=cuda_device))[0]["CLIP-RN50"]
        assert saved.shape == (5, 1024)
        assert np.array_equal(saved, alone), v

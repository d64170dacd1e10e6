"""ExtractResNet and `main.py --feature_type resnetXX` on the sample video, with the calibrated stand-in weights, against
the fixture the reference's own ExtractResNet produced (tests/golden/resnet_outputs.npz) and the fp32 oracle."""
import argparse
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import resnet_net

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
VIDEO = os.path.join(ROOT, "tests", "golden", "v_GGSY1Qvo990.mp4")


@pytest.fixture(scope="module")
def ckpt_dir(tmp_path_factory):
    """Stand-in weights under torchvision's checkpoint file names."""
    d = tmp_path_factory.mktemp("ckpt")
    for depth in (18, 50):
        torch.save(resnet_net.stand_in_state_dict(depth), str(d / f"resnet{depth}-standin.pth"))
    return str(d)


@pytest.fixture
def weights(ckpt_dir, monkeypatch):
    from video_features_b200.extract import extract_resnet
    monkeypatch.setenv("VF_CKPT_DIR", ckpt_dir)
    monkeypatch.setattr(extract_resnet, "_STATE_DICTS", {})
    return ckpt_dir


def _ns(**kw):
    d = dict(feature_type='resnet50', video_paths=None, flow_paths=None, file_with_video_paths=None, video_dir=None,
             flow_dir=None, extraction_fps=None, on_extraction='save_numpy', output_path='./output', tmp_path='./tmp',
             show_pred=False, keep_tmp_files=False, batch_size=1)
    d.update(kw)
    return argparse.Namespace(**d)


def _row_errors(y, ref):
    y, ref = torch.as_tensor(y).double(), torch.as_tensor(ref).double()
    rel = ((y - ref).norm(dim=1) / ref.norm(dim=1)).max().item()
    mx = ((y - ref).abs().amax(dim=1) / ref.abs().amax(dim=1)).max().item()
    return rel, mx


@pytest.mark.parametrize("depth", [18, 50])
def test_extract_resnet_vs_reference_and_oracle(cuda_device, weights, tmp_path, depth):
    from video_features_b200.extract.extract_resnet import ExtractResNet
    g = np.load(os.path.join(ROOT, "tests", "golden", "resnet_outputs.npz"))
    name = f"resnet{depth}"
    ex = ExtractResNet(_ns(feature_type=name, video_paths=[VIDEO], output_path=str(tmp_path / "out"),
                           tmp_path=str(tmp_path / "tmp")))
    ex.keep_features = True
    res = ex(torch.zeros([1], dtype=torch.long, device=cuda_device))[0]
    assert set(res) == {name, 'fps', 'timestamps_ms'}
    feats = res[name]
    assert feats.shape == (355, resnet_net.out_dim(depth)) and feats.dtype == np.float64
    assert float(res['fps']) == float(g['fps'])
    np.testing.assert_array_equal(res['timestamps_ms'], g['timestamps_ms'])
    saved = np.load(str(tmp_path / "out" / name / f"v_GGSY1Qvo990_{name}.npy"))
    np.testing.assert_array_equal(saved, feats)
    # against the rows the reference's ExtractResNet produced with the same weights
    rel, mx = _row_errors(feats[g['rows']], g[name])
    print(f"ExtractResNet {name} vs reference rows: rel-L2 {rel:.2e}, max-abs/max {mx:.2e}")
    assert rel <= 1e-3 and mx <= 1e-3
    # against the fp32 oracle on the same decoded frames (oracle transform: bit-exact with the reference's)
    from test_resnet_oracle_cpu import _decoded_frames
    x = torch.stack([resnet_net.transform(f) for f in _decoded_frames()])
    sd = {k: v.to(cuda_device) for k, v in resnet_net.stand_in_state_dict(depth).items()}
    with torch.no_grad():
        ref = torch.cat([resnet_net.forward(sd, x[i:i + 64].to(cuda_device), depth) for i in range(0, len(x), 64)])
    rel, mx = _row_errors(feats, ref.cpu())
    print(f"ExtractResNet {name} vs fp32 oracle, all 355 frames: rel-L2 {rel:.2e}, max-abs/max {mx:.2e}")
    assert rel <= 1e-3 and mx <= 1e-3


def test_main_cli_save_numpy_broken_file_and_resume(cuda_device, weights, tmp_path):
    broken = tmp_path / "broken.mp4"
    broken.write_bytes(b"not a video")
    out = tmp_path / "out"
    env = dict(os.environ, VF_CKPT_DIR=weights)
    cmd = [sys.executable, os.path.join(ROOT, "main.py"), "--feature_type", "resnet18", "--on_extraction", "save_numpy",
           "--output_path", str(out), "--tmp_path", str(tmp_path / "tmp"), "--video_paths", str(broken), VIDEO]
    r = subprocess.run(cmd, cwd=str(tmp_path), env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    target = out / "resnet18" / "v_GGSY1Qvo990_resnet18.npy"
    y = np.load(str(target))
    assert y.shape == (355, 512) and y.dtype == np.float64
    # OpenCV cannot open the broken file: like the reference, it yields no frames and an empty, reported result,
    # and the list goes on
    assert "Warning: the value is empty for resnet18" in r.stdout, r.stdout[-3000:]
    mtime = os.path.getmtime(target)
    env["VF_RESUME"] = "1"
    r = subprocess.run(cmd, cwd=str(tmp_path), env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    assert os.path.getmtime(target) == mtime                     # finished video skipped

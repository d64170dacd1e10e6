"""ExtractR21D and `main.py --feature_type r21d_rgb` on the sample video, with the calibrated stand-in weights, against
the fixture made from the reference's transform and slicing (tests/golden/r21d_outputs.npz) and the fp32 oracle."""
import argparse
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import r21d_net

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
VIDEO = os.path.join(ROOT, "tests", "golden", "v_GGSY1Qvo990.mp4")


@pytest.fixture(scope="module")
def ckpt_dir(tmp_path_factory):
    """Stand-in weights under torchvision's checkpoint file name."""
    d = tmp_path_factory.mktemp("ckpt")
    torch.save(r21d_net.stand_in_state_dict(), str(d / "r2plus1d_18-standin.pth"))
    return str(d)


@pytest.fixture
def weights(ckpt_dir, monkeypatch):
    from video_features_b200.extract import extract_r21d
    monkeypatch.setenv("VF_CKPT_DIR", ckpt_dir)
    monkeypatch.setattr(extract_r21d, "_STATE_DICT", {})
    return ckpt_dir


def _ns(**kw):
    d = dict(feature_type='r21d_rgb', video_paths=None, flow_paths=None, file_with_video_paths=None, video_dir=None,
             flow_dir=None, extraction_fps=None, on_extraction='save_numpy', output_path='./output', tmp_path='./tmp',
             show_pred=False, keep_tmp_files=False, stack_size=None, step_size=None)
    d.update(kw)
    return argparse.Namespace(**d)


def _row_errors(y, ref):
    y, ref = torch.as_tensor(y).double(), torch.as_tensor(ref).double()
    rel = ((y - ref).norm(dim=1) / ref.norm(dim=1)).max().item()
    mx = ((y - ref).abs().amax(dim=1) / ref.abs().amax(dim=1)).max().item()
    return rel, mx


def _extract(tmp_path, **kw):
    from video_features_b200.extract.extract_r21d import ExtractR21D
    ex = ExtractR21D(_ns(video_paths=[VIDEO], output_path=str(tmp_path / "out"), tmp_path=str(tmp_path / "tmp"), **kw))
    ex.keep_features = True
    return ex(torch.zeros([1], dtype=torch.long, device="cuda:0"))[0]


def test_extract_r21d_vs_reference_fixture(cuda_device, weights, tmp_path):
    g = np.load(os.path.join(ROOT, "tests", "golden", "r21d_outputs.npz"))
    res = _extract(tmp_path)
    assert set(res) == {"r21d_rgb"}
    feats = res["r21d_rgb"]
    assert feats.shape == (22, 512) and feats.dtype == np.float64
    saved = np.load(str(tmp_path / "out" / "r21d_rgb" / "v_GGSY1Qvo990_r21d_rgb.npy"))
    np.testing.assert_array_equal(saved, feats)
    rel, mx = _row_errors(feats, g["r21d_rgb"])
    print(f"ExtractR21D vs reference-transform fixture, 22 stacks: rel-L2 {rel:.2e}, max-abs/max {mx:.2e}")
    assert rel <= 1e-3 and mx <= 1e-3


@pytest.mark.parametrize("stack,step", [(16, 8), (8, 20)])
def test_extract_r21d_stack_step_vs_oracle(cuda_device, weights, tmp_path, stack, step):
    from test_r21d_oracle_cpu import decoded_rgb
    feats = _extract(tmp_path, stack_size=stack, step_size=step)["r21d_rgb"]
    rgb = decoded_rgb()
    slices = r21d_net.form_slices(len(rgb), stack, step)
    assert feats.shape == (len(slices), 512)
    x = r21d_net.transform(rgb)
    sd = {k: v.to(cuda_device) for k, v in r21d_net.stand_in_state_dict().items()}
    with torch.no_grad():
        ref = torch.cat([r21d_net.forward(sd, torch.stack([x[:, s:e] for s, e in slices[i:i + 8]]).to(cuda_device))
                         for i in range(0, len(slices), 8)])
    rel, mx = _row_errors(feats, ref.cpu())
    print(f"ExtractR21D stack {stack} step {step} ({len(slices)} stacks) vs fp32 oracle: rel-L2 {rel:.2e}, "
          f"max-abs/max {mx:.2e}")
    assert rel <= 1e-3 and mx <= 1e-3


def test_video_shorter_than_a_stack(cuda_device, weights, tmp_path):
    feats = _extract(tmp_path, stack_size=400)["r21d_rgb"]         # 355 frames: no full stack
    assert feats.shape == (0,) and feats.dtype == np.float64      # np.array([]), as the reference returns


def test_main_cli_save_numpy_and_broken_file(cuda_device, weights, tmp_path):
    broken = tmp_path / "broken.mp4"
    broken.write_bytes(b"not a video")
    out = tmp_path / "out"
    env = dict(os.environ, VF_CKPT_DIR=weights)
    cmd = [sys.executable, os.path.join(ROOT, "main.py"), "--feature_type", "r21d_rgb", "--on_extraction", "save_numpy",
           "--output_path", str(out), "--tmp_path", str(tmp_path / "tmp"), "--video_paths", str(broken), VIDEO]
    r = subprocess.run(cmd, cwd=str(tmp_path), env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    y = np.load(str(out / "r21d_rgb" / "v_GGSY1Qvo990_r21d_rgb.npy"))
    assert y.shape == (22, 512) and y.dtype == np.float64
    g = np.load(os.path.join(ROOT, "tests", "golden", "r21d_outputs.npz"))
    rel, mx = _row_errors(y, g["r21d_rgb"])
    assert rel <= 1e-3 and mx <= 1e-3
    # the broken file is reported and skipped; the list goes on
    assert f"Extraction failed at: {broken}" in r.stdout, r.stdout[-3000:]

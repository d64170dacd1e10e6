"""ExtractDINOv2 and `main.py --feature_type dinov2_vits14` on the sample video (355 frames), with seeded stand-in
weights under the hub's file name, against OpenCV decode -> the hub's PIL preset -> the float64 oracle per frame."""
import argparse
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from dinov2_bars import FEATURES
from oracle import dinov2_net as D

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
VIDEO = os.path.join(ROOT, "tests", "golden", "v_GGSY1Qvo990.mp4")
NAME = "dinov2_vits14"


@pytest.fixture(scope="module")
def ckpt_dir(tmp_path_factory):
    d = tmp_path_factory.mktemp("ckpt")
    torch.save(D.stand_in_state_dict(NAME), str(d / "dinov2_vits14_pretrain.pth"))
    return str(d)


@pytest.fixture
def weights(ckpt_dir, monkeypatch):
    from video_features_b200.extract import extract_dinov2
    monkeypatch.setenv("VF_CKPT_DIR", ckpt_dir)
    monkeypatch.setattr(extract_dinov2, "_STATE_DICTS", {})
    return ckpt_dir


@pytest.fixture(scope="module")
def oracle_feats():
    """(exact, declared-rounding) float64 features of every decoded frame."""
    import cv2
    cap = cv2.VideoCapture(VIDEO)
    xs = []
    while True:
        ok, f = cap.read()
        if not ok:
            break
        xs.append(D.transform(f[:, :, ::-1]))
    cap.release()
    assert len(xs) == 355
    sd = D.prepare(D.stand_in_state_dict(NAME), torch.float64, "cuda")
    exact, declared = [], []
    with torch.no_grad():
        for i in range(0, len(xs), 64):
            x = torch.stack(xs[i:i + 64]).cuda().double()
            exact.append(D.forward(sd, x).cpu())
            declared.append(D.forward_engine(sd, x).cpu())
    return torch.cat(exact), torch.cat(declared)


def _ns(**kw):
    d = dict(feature_type=NAME, video_paths=None, flow_paths=None, file_with_video_paths=None, video_dir=None,
             flow_dir=None, extraction_fps=None, on_extraction='save_numpy', output_path='./output', tmp_path='./tmp',
             show_pred=False, keep_tmp_files=False, stack_size=None, step_size=None)
    d.update(kw)
    return argparse.Namespace(**d)


def _row_errors(y, ref):
    y, ref = torch.as_tensor(y).double(), torch.as_tensor(ref).double()
    rel = ((y - ref).norm(dim=1) / ref.norm(dim=1)).max().item()
    mx = ((y - ref).abs().amax(dim=1) / ref.abs().amax(dim=1)).max().item()
    return rel, mx


def _extract_all(tmp_path, **kw):
    from video_features_b200.extract.extract_dinov2 import ExtractDINOv2
    ex = ExtractDINOv2(_ns(video_paths=[VIDEO], output_path=str(tmp_path / "out"), tmp_path=str(tmp_path / "tmp"), **kw))
    ex.keep_features = True
    return ex(torch.zeros([1], dtype=torch.long, device="cuda:0"))


def test_extract_dinov2_vs_float64(cuda_device, weights, tmp_path, oracle_feats):
    res = _extract_all(tmp_path)[0]
    assert set(res) == {NAME, "fps", "timestamps_ms"}
    feats = res[NAME]
    assert feats.shape == (355, 384) and feats.dtype == np.float32
    assert len(res["timestamps_ms"]) == 355
    saved = np.load(str(tmp_path / "out" / NAME / f"v_GGSY1Qvo990_{NAME}.npy"))
    np.testing.assert_array_equal(saved, feats)
    e_exact, e_decl = _row_errors(feats, oracle_feats[0]), _row_errors(feats, oracle_feats[1])
    print(f"ExtractDINOv2 vs float64, 355 frames: exact {e_exact[0]:.2e}/{e_exact[1]:.2e}, "
          f"declared {e_decl[0]:.2e}/{e_decl[1]:.2e}")
    assert e_exact[0] <= FEATURES[384][0] and e_exact[1] <= FEATURES[384][1], e_exact


def test_resume_skips_a_video_whose_output_exists(cuda_device, weights, tmp_path, monkeypatch):
    out = tmp_path / "out" / NAME
    out.mkdir(parents=True)
    marker = np.full((1, 1), 7.0, np.float32)
    np.save(str(out / f"v_GGSY1Qvo990_{NAME}.npy"), marker)
    monkeypatch.setenv("VF_RESUME", "1")
    assert _extract_all(tmp_path) == []
    np.testing.assert_array_equal(np.load(str(out / f"v_GGSY1Qvo990_{NAME}.npy")), marker)


def test_main_cli_end_to_end(cuda_device, weights, tmp_path, oracle_feats):
    out = tmp_path / "out"
    env = dict(os.environ, VF_CKPT_DIR=weights, VF_ASYNC_SINK="1")
    cmd = [sys.executable, os.path.join(ROOT, "main.py"), "--feature_type", NAME, "--device_ids", "0",
           "--on_extraction", "save_numpy", "--output_path", str(out), "--tmp_path", str(tmp_path / "tmp"),
           "--video_paths", VIDEO]
    r = subprocess.run(cmd, cwd=str(tmp_path), env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    y = np.load(str(out / NAME / f"v_GGSY1Qvo990_{NAME}.npy"))
    assert y.shape == (355, 384) and y.dtype == np.float32
    rel, mx = _row_errors(y, oracle_feats[0])
    assert rel <= FEATURES[384][0] and mx <= FEATURES[384][1]

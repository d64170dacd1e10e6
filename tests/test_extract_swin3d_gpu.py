"""ExtractSwin3D and `main.py --feature_type swin3d_t` on the sample video (355 frames: 11 stacks at 32 / 32), with the
seeded stand-in weights, against OpenCV decode -> torchvision's Swin3D preset -> float64 Swin3D-T per stack."""
import argparse
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import swin3d_net

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
VIDEO = os.path.join(ROOT, "tests", "golden", "v_GGSY1Qvo990.mp4")


@pytest.fixture(scope="module")
def ckpt_dir(tmp_path_factory):
    """Stand-in weights under torchvision's checkpoint file name."""
    d = tmp_path_factory.mktemp("ckpt")
    torch.save(swin3d_net.stand_in_state_dict("swin3d_t"), str(d / "swin3d_t-standin.pth"))
    return str(d)


@pytest.fixture
def weights(ckpt_dir, monkeypatch):
    from video_features_b200.extract import extract_swin3d
    monkeypatch.setenv("VF_CKPT_DIR", ckpt_dir)
    monkeypatch.setattr(extract_swin3d, "_STATE_DICTS", {})
    return ckpt_dir


@pytest.fixture(scope="module")
def oracle_logits_feats():
    """Per stack of form_slices(355, 32, 32): OpenCV decode, BGR -> RGB, the preset, float64 Swin3D-T -> (features,
    logits)."""
    import cv2
    cap = cv2.VideoCapture(VIDEO)
    frames = []
    while True:
        ok, f = cap.read()
        if not ok:
            break
        frames.append(f[:, :, ::-1])
    cap.release()
    rgb = np.stack(frames)
    slices = swin3d_net.form_slices(len(rgb), 32, 32)
    assert len(rgb) == 355 and len(slices) == 11
    dev = torch.device("cuda", 0)
    sd = {k: (v.double() if v.is_floating_point() else v).to(dev) for k, v in swin3d_net.stand_in_state_dict("swin3d_t").items()}
    feats = []
    with torch.no_grad():
        for s, e in slices:
            x = swin3d_net.transform_torchvision(rgb[s:e]).unsqueeze(0).to(dev).double()
            feats.append(swin3d_net.forward(sd, x))
        y = torch.cat(feats)
        return y.cpu(), swin3d_net.logits(sd, y).cpu()


def _ns(**kw):
    d = dict(feature_type='swin3d_t', video_paths=None, flow_paths=None, file_with_video_paths=None, video_dir=None,
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
    from video_features_b200.extract.extract_swin3d import ExtractSwin3D
    ex = ExtractSwin3D(_ns(video_paths=[VIDEO], output_path=str(tmp_path / "out"), tmp_path=str(tmp_path / "tmp"), **kw))
    ex.keep_features = True
    return ex(torch.zeros([1], dtype=torch.long, device="cuda:0"))


def _extract(tmp_path, **kw):
    return _extract_all(tmp_path, **kw)[0]


def test_extract_swin3d_vs_float64(cuda_device, weights, tmp_path, oracle_logits_feats):
    res = _extract(tmp_path)
    assert set(res) == {"swin3d_t"}
    feats = res["swin3d_t"]
    assert feats.shape == (11, 768) and feats.dtype == np.float32
    saved = np.load(str(tmp_path / "out" / "swin3d_t" / "v_GGSY1Qvo990_swin3d_t.npy"))
    np.testing.assert_array_equal(saved, feats)
    rel, mx = _row_errors(feats, oracle_logits_feats[0])
    print(f"ExtractSwin3D vs float64 Swin3D-T, 11 stacks: rel-L2 {rel:.2e}, max-abs/max {mx:.2e}")
    assert rel <= 1e-3 and mx <= 1e-3


def test_show_pred_prints_the_oracle_top5(cuda_device, weights, tmp_path, oracle_logits_feats, capsys):
    from video_features_b200.utils import _class_names
    res = _extract(tmp_path, show_pred=True, on_extraction='print')
    out = capsys.readouterr().out
    headers = re.findall(r"^(.*) @ frames \((\d+), (\d+)\)$", out, re.M)
    assert [(int(a), int(b)) for _, a, b in headers] == [(i * 32, i * 32 + 32) for i in range(11)]
    blocks = out.split(" @ frames (")[1:]
    names = _class_names("kinetics")
    logits = oracle_logits_feats[1]
    probs = torch.softmax(logits, dim=-1)
    order = torch.sort(probs, dim=-1, descending=True, stable=True)[1][:, :5]
    for i, blk in enumerate(blocks):
        lines = re.findall(r"^(-?\d+\.\d{3}) (\d\.\d{3}) (.+)$", blk, re.M)[:5]
        assert len(lines) == 5, blk
        scale = logits[i].abs().max().item()
        tol = 5e-4 * scale + 5e-4
        # the oracle's top-5 in order, except that two classes whose float64 logits lie within the tolerance may swap
        got = [names.index(c) for _, _, c in lines]
        for r, (c, j) in enumerate(zip(got, order[i].tolist())):
            assert c == j or abs(logits[i, c].item() - logits[i, j].item()) <= tol, (i, r, got, order[i].tolist())
        for (lg, pr, _), j in zip(lines, got):
            assert abs(float(lg) - logits[i, j].item()) <= tol
            assert abs(float(pr) - probs[i, j].item()) <= tol
    assert res["swin3d_t"].shape == (11, 768)


def test_resume_skips_a_video_whose_output_exists(cuda_device, weights, tmp_path, monkeypatch):
    out = tmp_path / "out" / "swin3d_t"
    out.mkdir(parents=True)
    marker = np.full((1, 1), 7.0, np.float32)
    np.save(str(out / "v_GGSY1Qvo990_swin3d_t.npy"), marker)
    monkeypatch.setenv("VF_RESUME", "1")
    assert _extract_all(tmp_path) == []
    np.testing.assert_array_equal(np.load(str(out / "v_GGSY1Qvo990_swin3d_t.npy")), marker)


def test_main_cli_end_to_end(cuda_device, weights, tmp_path, oracle_logits_feats):
    out = tmp_path / "out"
    env = dict(os.environ, VF_CKPT_DIR=weights)
    cmd = [sys.executable, os.path.join(ROOT, "main.py"), "--feature_type", "swin3d_t", "--device_ids", "0",
           "--on_extraction", "save_numpy", "--output_path", str(out), "--tmp_path", str(tmp_path / "tmp"),
           "--video_paths", VIDEO]
    r = subprocess.run(cmd, cwd=str(tmp_path), env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    y = np.load(str(out / "swin3d_t" / "v_GGSY1Qvo990_swin3d_t.npy"))
    assert y.shape == (11, 768) and y.dtype == np.float32
    rel, mx = _row_errors(y, oracle_logits_feats[0])
    assert rel <= 1e-3 and mx <= 1e-3


def test_stack_longer_than_the_video_is_empty(cuda_device, weights, tmp_path):
    res = _extract(tmp_path, stack_size=400, step_size=400)
    assert isinstance(res["swin3d_t"], np.ndarray) and res["swin3d_t"].size == 0

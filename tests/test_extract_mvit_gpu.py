"""ExtractMViT and `main.py --feature_type mvit_v2_s` on the sample video (355 frames: 22 stacks at 16 / 16), with the
seeded stand-in weights, against OpenCV decode -> torchvision's MViT preset -> float64 MViT-V2-S per stack."""
import argparse
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

from mvit_bars import BARS
from oracle import mvit_net
from oracle.r21d_net import form_slices

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
VIDEO = os.path.join(ROOT, "tests", "golden", "v_GGSY1Qvo990.mp4")


@pytest.fixture(scope="module")
def ckpt_dir(tmp_path_factory):
    """Stand-in weights under torchvision's checkpoint file name."""
    d = tmp_path_factory.mktemp("ckpt")
    torch.save(mvit_net.stand_in_state_dict("mvit_v2_s"), str(d / "mvit_v2_s-standin.pth"))
    return str(d)


@pytest.fixture
def weights(ckpt_dir, monkeypatch):
    from video_features_b200.extract import extract_mvit
    monkeypatch.setenv("VF_CKPT_DIR", ckpt_dir)
    monkeypatch.setattr(extract_mvit, "_STATE_DICTS", {})
    return ckpt_dir


@pytest.fixture(scope="module")
def oracle_logits_feats():
    """Per stack of form_slices(355, 16, 16): OpenCV decode, BGR -> RGB, the preset, float64 MViT-V2-S -> (features,
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
    slices = form_slices(len(rgb), 16, 16)
    assert len(rgb) == 355 and len(slices) == 22
    dev = torch.device("cuda", 0)
    sd = {k: (v.double() if v.is_floating_point() else v).to(dev) for k, v in mvit_net.stand_in_state_dict("mvit_v2_s").items()}
    feats = []
    with torch.no_grad():
        for s, e in slices:
            x = mvit_net.transform_torchvision(rgb[s:e], "mvit_v2_s").unsqueeze(0).to(dev).double()
            feats.append(mvit_net.forward(sd, x))
        y = torch.cat(feats)
        return y.cpu(), mvit_net.logits(sd, y).cpu()


def _ns(**kw):
    d = dict(feature_type='mvit_v2_s', video_paths=None, flow_paths=None, file_with_video_paths=None, video_dir=None,
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
    from video_features_b200.extract.extract_mvit import ExtractMViT
    ex = ExtractMViT(_ns(video_paths=[VIDEO], output_path=str(tmp_path / "out"), tmp_path=str(tmp_path / "tmp"), **kw))
    ex.keep_features = True
    return ex(torch.zeros([1], dtype=torch.long, device="cuda:0"))


def _extract(tmp_path, **kw):
    return _extract_all(tmp_path, **kw)[0]


def test_extract_mvit_vs_float64(cuda_device, weights, tmp_path, oracle_logits_feats):
    res = _extract(tmp_path)
    assert set(res) == {"mvit_v2_s"}
    feats = res["mvit_v2_s"]
    assert feats.shape == (22, 768) and feats.dtype == np.float32
    saved = np.load(str(tmp_path / "out" / "mvit_v2_s" / "v_GGSY1Qvo990_mvit_v2_s.npy"))
    np.testing.assert_array_equal(saved, feats)
    rel, mx = _row_errors(feats, oracle_logits_feats[0])
    print(f"ExtractMViT vs float64 MViT-V2-S, 22 stacks: rel-L2 {rel:.2e}, max-abs/max {mx:.2e}")
    assert rel <= BARS["features"][0] and mx <= BARS["features"][1]


def test_show_pred_prints_the_oracle_top5(cuda_device, weights, tmp_path, oracle_logits_feats, capsys):
    from video_features_b200.utils import _class_names
    res = _extract(tmp_path, show_pred=True, on_extraction='print')
    out = capsys.readouterr().out
    headers = re.findall(r"^(.*) @ frames \((\d+), (\d+)\)$", out, re.M)
    assert [(int(a), int(b)) for _, a, b in headers] == [(i * 16, i * 16 + 16) for i in range(22)]
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
    assert res["mvit_v2_s"].shape == (22, 768)


def test_resume_skips_a_video_whose_output_exists(cuda_device, weights, tmp_path, monkeypatch):
    out = tmp_path / "out" / "mvit_v2_s"
    out.mkdir(parents=True)
    marker = np.full((1, 1), 7.0, np.float32)
    np.save(str(out / "v_GGSY1Qvo990_mvit_v2_s.npy"), marker)
    monkeypatch.setenv("VF_RESUME", "1")
    assert _extract_all(tmp_path) == []
    np.testing.assert_array_equal(np.load(str(out / "v_GGSY1Qvo990_mvit_v2_s.npy")), marker)


def test_main_cli_end_to_end(cuda_device, weights, tmp_path, oracle_logits_feats):
    out = tmp_path / "out"
    env = dict(os.environ, VF_CKPT_DIR=weights)
    cmd = [sys.executable, os.path.join(ROOT, "main.py"), "--feature_type", "mvit_v2_s", "--device_ids", "0",
           "--on_extraction", "save_numpy", "--output_path", str(out), "--tmp_path", str(tmp_path / "tmp"),
           "--video_paths", VIDEO]
    r = subprocess.run(cmd, cwd=str(tmp_path), env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    y = np.load(str(out / "mvit_v2_s" / "v_GGSY1Qvo990_mvit_v2_s.npy"))
    assert y.shape == (22, 768) and y.dtype == np.float32
    rel, mx = _row_errors(y, oracle_logits_feats[0])
    assert rel <= BARS["features"][0] and mx <= BARS["features"][1]


def test_step_shorter_than_the_stack(cuda_device, weights, tmp_path, oracle_logits_feats):
    """Overlapping 16-frame stacks every 8 frames: the even stacks are the 16 / 16 stacks."""
    feats = _extract(tmp_path, step_size=8)["mvit_v2_s"]
    assert feats.shape == (43, 768)
    rel, mx = _row_errors(feats[0::2], oracle_logits_feats[0])
    assert rel <= BARS["features"][0] and mx <= BARS["features"][1]

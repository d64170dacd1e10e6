"""ExtractVideoMAE and `main.py --feature_type videomae_vitb16` on the sample video (355 frames: 22 stacks at 16 / 16),
with seeded stand-in weights in a Hugging Face checkpoint directory, against OpenCV decode -> the processor's PIL
preset -> float64 VideoMAE per stack."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import videomae_net as V
from oracle.r21d_net import form_slices
from videomae_bars import FEATURES

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
VIDEO = os.path.join(ROOT, "tests", "golden", "v_GGSY1Qvo990.mp4")
NAME = "videomae_vitb16"
N_CHECK = 3          # stacks checked against float64


@pytest.fixture(scope="module")
def ckpt_dir(tmp_path_factory):
    """$VF_CKPT_DIR/videomae-base-finetuned-kinetics/ with config.json (named classes) and model.safetensors."""
    from safetensors.torch import save_file
    root = tmp_path_factory.mktemp("ckpt")
    d = root / "videomae-base-finetuned-kinetics"
    d.mkdir()
    cfg = V.config_dict(NAME, id2label={str(i): f"class {i}" for i in range(V.N_CLASSES)})
    (d / "config.json").write_text(json.dumps(cfg))
    save_file({k: v.contiguous() for k, v in V.stand_in_state_dict(NAME).items()}, str(d / "model.safetensors"))
    return str(root)


@pytest.fixture
def weights(ckpt_dir, monkeypatch):
    from video_features_b200.extract import extract_videomae
    monkeypatch.setenv("VF_CKPT_DIR", ckpt_dir)
    monkeypatch.setattr(extract_videomae, "_CHECKPOINTS", {})
    return ckpt_dir


@pytest.fixture(scope="module")
def oracle_feats():
    import cv2
    cap = cv2.VideoCapture(VIDEO)
    frames = []
    while True:
        ok, f = cap.read()
        if not ok:
            break
        frames.append(f)
    cap.release()
    bgr = np.stack(frames)
    slices = form_slices(len(bgr), 16, 16)
    assert len(bgr) == 355 and len(slices) == 22
    p = V.prepare(V.stand_in_state_dict(NAME), torch.float64, "cuda")
    with torch.no_grad():
        x = torch.stack([V.preset_clip(bgr[s:e]) for s, e in slices[:N_CHECK]]).cuda().double()
        y = V.forward(p, x)
        return y.cpu(), V.logits(p, y).cpu()


def _ns(**kw):
    d = dict(feature_type=NAME, video_paths=None, flow_paths=None, file_with_video_paths=None, video_dir=None,
             flow_dir=None, extraction_fps=None, on_extraction='save_numpy', output_path='./output', tmp_path='./tmp',
             show_pred=False, keep_tmp_files=False, stack_size=None, step_size=None)
    d.update(kw)
    return argparse.Namespace(**d)


def test_extract_matches_float64(cuda_device, weights, oracle_feats, tmp_path, capsys):
    from video_features_b200.extract.extract_videomae import ExtractVideoMAE
    ex = ExtractVideoMAE(_ns(video_paths=[VIDEO], output_path=str(tmp_path / "out"), tmp_path=str(tmp_path / "tmp"),
                             show_pred=True))
    ex.keep_features = True
    out = ex(torch.zeros([1], dtype=torch.long, device="cuda:0"))[0]
    assert set(out) == {NAME}
    y = out[NAME]
    assert y.shape == (22, 768) and y.dtype == np.float32
    ref, logits = oracle_feats
    yt = torch.from_numpy(y[:N_CHECK]).double()
    rel = ((yt - ref).norm(dim=1) / ref.norm(dim=1)).max().item()
    mx = ((yt - ref).abs().amax(dim=1) / ref.abs().amax(dim=1)).max().item()
    saved = np.load(os.path.join(str(tmp_path / "out"), NAME, f"v_GGSY1Qvo990_{NAME}.npy"))
    assert np.array_equal(saved, y)
    text = capsys.readouterr().out
    top = logits[0].softmax(-1).topk(5).indices.tolist()
    lines = text.split("@ frames (0, 16)")[1].strip().splitlines()[:5]
    assert [ln.split(" ", 2)[2] for ln in lines] == [f"class {i}" for i in top], lines
    print(f"\nextract {NAME} first {N_CHECK} stacks vs float64: {rel:.2e} / {mx:.2e}")
    assert rel <= FEATURES[768][0] and mx <= FEATURES[768][1]


def test_stack_size_refused(weights):
    from video_features_b200.extract.extract_videomae import ExtractVideoMAE
    with pytest.raises(ValueError, match="16"):
        ExtractVideoMAE(_ns(video_paths=[VIDEO], stack_size=8))


def test_main_cli(cuda_device, weights, tmp_path):
    env = dict(os.environ, VF_CKPT_DIR=weights)
    r = subprocess.run([sys.executable, os.path.join(ROOT, "main.py"), "--feature_type", NAME, "--video_paths", VIDEO,
                        "--on_extraction", "save_numpy", "--output_path", str(tmp_path / "o")], cwd=ROOT, env=env,
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    y = np.load(os.path.join(str(tmp_path / "o"), NAME, f"v_GGSY1Qvo990_{NAME}.npy"))
    assert y.shape == (22, 768)

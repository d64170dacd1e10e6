"""ExtractCLIP --show_pred end to end on the sample video: synthetic weights (ViT) or the oracle stand-in (RN50) with a
synthetic text tower, and a vocabulary trained on the prompts.  The printed top-5 of every frame must be the float64
oracle's (the declared-rounding text tower against the engine's own image features), the printed logits within the
bar, and the features bit-identical to a run without --show_pred."""
import argparse
import os
import re

import numpy as np
import pytest
import torch

from clip_text_bars import LOGITS
from clip_text_vocab import standard_vocab
from oracle import clip_resnet
from oracle import clip_text as T
from video_features_b200 import clip_tokenizer as ct
from video_features_b200 import synthetic_weights

pytestmark = pytest.mark.gpu

SAMPLE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "v_GGSY1Qvo990.mp4")
CUSTOM = ["a person playing the guitar", "a dog's birthday party", "SNOW on 3 mountains!"]
LINE = re.compile(r"^(-?\d+\.\d{3}) (\d\.\d{3}) (.+)$")


def _args(paths, out, feature_type, show_pred, pred_texts=None):
    return argparse.Namespace(feature_type=feature_type, video_paths=paths, flow_paths=None, file_with_video_paths=None,
                              video_dir=None, flow_dir=None, extraction_fps=None, extract_method="uni_6",
                              on_extraction="save_numpy", output_path=out, output_direct=True,
                              tmp_path=os.path.join(out, "tmp"), show_pred=show_pred, pred_texts=pred_texts)


@pytest.fixture(scope="module")
def bpe(tmp_path_factory):
    return standard_vocab(str(tmp_path_factory.mktemp("bpe") / ct.BPE_NAME))


def _weights(feature_type, tmp_path, monkeypatch, bpe):
    """The state dict ExtractCLIP will load, text tower included."""
    from video_features_b200.extract.extract_clip import load_clip_state_dict
    monkeypatch.setenv("VF_CLIP_BPE", bpe)
    vocab = ct.SimpleTokenizer(bpe).vocab_size
    if feature_type == "CLIP-RN50":
        sd = clip_resnet.stand_in_state_dict("RN50")
        sd.update(synthetic_weights.clip_text_state_dict(4, 512, 1024, vocab))
        path = str(tmp_path / "RN50.pt")
        torch.save(sd, path)
        monkeypatch.setenv("VF_CLIP_CKPT", path)
        monkeypatch.delenv("VF_CLIP_SYNTHETIC", raising=False)
        return sd
    monkeypatch.setenv("VF_CLIP_SYNTHETIC", "0")
    return load_clip_state_dict(feature_type, vocab)


def _printed(text, k):
    """stdout -> one list of (logit, prob, prompt) per frame."""
    frames, cur = [], []
    for ln in text.splitlines():
        m = LINE.match(ln)
        if m:
            cur.append((float(m.group(1)), float(m.group(2)), m.group(3)))
        elif ln == "" and cur:
            frames.append(cur)
            cur = []
    assert all(len(f) == k for f in frames)
    return frames


def _check_against_oracle(frames, feats, sd, prompts, bpe):
    tokens = ct.SimpleTokenizer(bpe).tokenize(prompts)
    logits = T.zero_shot_logits(sd, torch.from_numpy(feats), T.encode_text_declared(sd, tokens))
    assert len(frames) == feats.shape[0]
    index = {p: i for i, p in enumerate(prompts)}
    k = min(5, len(prompts))
    for f, rows in enumerate(frames):
        order = torch.sort(logits[f], descending=True, stable=True).indices[:k].tolist()
        for r, (lg, _, p) in enumerate(rows):
            j = index[p]
            assert abs(lg - logits[f, j].item()) < LOGITS + 5e-4, (f, r, p)
            # the oracle's own rank-r class, unless the two are within the bar of each other
            assert j == order[r] or abs(logits[f, j] - logits[f, order[r]]).item() < LOGITS, (f, r, p)


@pytest.mark.parametrize("feature_type", ["CLIP-ViT-B/32", "CLIP-ViT-L/14", "CLIP-RN50"])
@pytest.mark.parametrize("custom", [False, True])
def test_show_pred_matches_oracle_and_keeps_features(cuda_device, tmp_path, monkeypatch, capsys, bpe, feature_type,
                                                     custom):
    from video_features_b200.extract.extract_clip import ExtractCLIP
    sd = _weights(feature_type, tmp_path, monkeypatch, bpe)
    prompts = CUSTOM if custom else ct.default_prompts()
    out = str(tmp_path / "o")
    plain = ExtractCLIP(_args([SAMPLE], out, feature_type, False), external_call=True)(torch.tensor([0], device=cuda_device))
    capsys.readouterr()
    ex = ExtractCLIP(_args([SAMPLE], out, feature_type, True, CUSTOM if custom else None), external_call=True)
    got = ex(torch.tensor([0], device=cuda_device))
    frames = _printed(capsys.readouterr().out, min(5, len(prompts)))
    feats = got[0][feature_type]
    assert np.array_equal(feats, plain[0][feature_type])
    _check_against_oracle(frames, feats, sd, prompts, bpe)


def test_show_pred_on_the_batched_list_path(cuda_device, tmp_path, monkeypatch, capsys, bpe):
    """Two videos through _forward_batched: per video, list order, the same lines as the one-video call."""
    from video_features_b200.extract.extract_clip import ExtractCLIP
    _weights("CLIP-ViT-B/32", tmp_path, monkeypatch, bpe)
    out = str(tmp_path / "o")
    one = ExtractCLIP(_args([SAMPLE], out, "CLIP-ViT-B/32", True, CUSTOM), external_call=True)
    one(torch.tensor([0], device=cuda_device))
    single = capsys.readouterr().out
    ex = ExtractCLIP(_args([SAMPLE, SAMPLE], out, "CLIP-ViT-B/32", True, CUSTOM))
    ex(torch.tensor([0, 1], device=cuda_device))
    both = _printed(capsys.readouterr().out, 3)
    first = _printed(single, 3)
    assert both == first + first
    assert os.path.exists(os.path.join(out, "v_GGSY1Qvo990.npy"))

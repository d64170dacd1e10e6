"""oracle/videomae_net.py against Hugging Face: the forward against ``VideoMAEForVideoClassification`` built from a
random config, the sinusoid table bit for bit against ``get_sinusoid_encoding_table``, the PIL preset against
``VideoMAEImageProcessorPil``; and the engine wrapper's own table and preset against the oracle's."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import videomae_net as V  # noqa: E402

transformers = pytest.importorskip("transformers")


def _hf_model(name, depth):
    from transformers import VideoMAEConfig, VideoMAEForVideoClassification
    cfg = VideoMAEConfig(**V.config_dict(name, depth))
    torch.manual_seed(0)
    m = VideoMAEForVideoClassification(cfg).eval()
    with torch.no_grad():      # HF initialises biases and LayerNorms trivially: give them random values too
        for k, v in m.state_dict().items():
            if k.endswith("bias") or "layernorm" in k or "fc_norm" in k:
                v.copy_(torch.randn_like(v) * 0.1 + (1.0 if k.endswith("weight") else 0.0))
    return m


@pytest.mark.parametrize("name,depth", [("videomae_vits16", None), ("videomae_vitb16", None), ("videomae_vitl16", 2)])
def test_oracle_matches_hf(name, depth):
    m = _hf_model(name, depth)
    sd = m.state_dict()
    x = V.calibration_clips(1, 1)
    with torch.no_grad():
        out = m(pixel_values=x, output_hidden_states=True)
        ref_feat = m.fc_norm(out.hidden_states[-1].mean(1))
    p = V.prepare(sd, torch.float32)
    feat = V.forward(p, x)
    rel = float((feat - ref_feat).norm() / ref_feat.norm())
    assert rel < 2e-6, rel
    lg = V.logits(p, feat)
    assert float((lg - out.logits).norm() / out.logits.norm()) < 2e-6


@pytest.mark.parametrize("d", [384, 768, 1024])
def test_sinusoid_table_bit_equal(d):
    from transformers.models.videomae.modeling_videomae import get_sinusoid_encoding_table
    from video_features_b200.videomae_engine import sinusoid_table
    ref = get_sinusoid_encoding_table(V.TOKENS, d)[0].numpy()
    assert ref.dtype == np.float32
    assert np.array_equal(V.sinusoid_table(V.TOKENS, d), ref)
    assert np.array_equal(sinusoid_table(V.TOKENS, d), ref)


@pytest.mark.parametrize("hw", [(240, 320), (240, 321), (360, 480), (224, 224), (480, 270)])
def test_preset_matches_pil_processor(hw):
    from transformers.models.videomae.image_processing_pil_videomae import VideoMAEImageProcessorPil
    proc = VideoMAEImageProcessorPil(image_mean=list(V.IMAGENET_MEAN), image_std=list(V.IMAGENET_STD))
    g = np.random.default_rng(hw[0] * 1000 + hw[1])
    frames = g.integers(0, 256, (2,) + hw + (3,), dtype=np.uint8)
    ref = np.asarray(proc([list(frames)], return_tensors="np")["pixel_values"][0])
    ours = np.stack([V.preset_frame(f) for f in frames])
    assert ours.shape == ref.shape == (2, 3, 224, 224)
    assert np.array_equal(ours, ref)


def test_odd_margin_crops_at_the_floor():
    """240 x 321 resizes to 224 x 299: a margin of 75 columns, cropped from column 37 (torchvision's round gives 38)."""
    from PIL import Image
    g = np.random.default_rng(3)
    f = g.integers(0, 256, (240, 321, 3), dtype=np.uint8)
    r = np.asarray(Image.fromarray(f).resize((299, 224), Image.BILINEAR)).transpose(2, 0, 1)
    x = V.preset_frame(f)
    want = ((r[:, :, 37:37 + 224].astype(np.float64) / 255).astype(np.float32).T
            - np.float32(V.IMAGENET_MEAN)) / np.float32(V.IMAGENET_STD)
    assert np.array_equal(x, want.T)
    shifted = ((r[:, :, 38:38 + 224].astype(np.float64) / 255).astype(np.float32).T
               - np.float32(V.IMAGENET_MEAN)) / np.float32(V.IMAGENET_STD)
    assert not np.array_equal(x, shifted.T)


def test_tubelet_layout_is_the_conv3d():
    x = V.calibration_clips(2, 1).double()
    w = torch.randn(8, 3, 2, 16, 16, dtype=torch.float64)
    conv = torch.nn.functional.conv3d(x.permute(0, 2, 1, 3, 4), w, stride=(2, 16, 16)).flatten(2).transpose(1, 2)
    lin = V.tubelets(x) @ w.reshape(8, -1).T
    assert torch.allclose(conv, lin, rtol=0, atol=1e-12)

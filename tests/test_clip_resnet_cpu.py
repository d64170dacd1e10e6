"""CPU checks of the CLIP ResNet towers' test infrastructure and host logic: the oracle's attention pool against
torch.nn.MultiheadAttention, the engine's restated layouts (tests/clip_rn_layout.py) against float64 convolutions,
configuration inference, the towers' preprocess against the ViT transform at 224 and against PIL + torchvision at
288 / 384, and ExtractCLIP's tower names."""
import argparse
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import clip_rn_layout as lay
from oracle import clip_preprocess, clip_resnet

SAMPLE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "v_GGSY1Qvo990.mp4")


@pytest.mark.parametrize("T", [50, 82, 145])
def test_attention_pool_equals_multihead_attention(T):
    E, heads, out_dim, n = 256, 4, 96, 3
    g = torch.Generator().manual_seed(T)
    a = "visual.attnpool."
    sd = {a + "positional_embedding": torch.randn(T, E, generator=g, dtype=torch.float64) / E ** 0.5}
    for p in ("q", "k", "v"):
        sd[f"{a}{p}_proj.weight"] = torch.randn(E, E, generator=g, dtype=torch.float64) / E ** 0.5
        sd[f"{a}{p}_proj.bias"] = torch.randn(E, generator=g, dtype=torch.float64) * 0.1
    sd[a + "c_proj.weight"] = torch.randn(out_dim, E, generator=g, dtype=torch.float64) / E ** 0.5
    sd[a + "c_proj.bias"] = torch.randn(out_dim, generator=g, dtype=torch.float64) * 0.1
    side = int(round((T - 1) ** 0.5))
    x = torch.randn(n, E, side, side, generator=g, dtype=torch.float64)
    tok = clip_resnet.pool_tokens(sd, x)
    assert tok.shape == (T, n, E)
    torch.testing.assert_close(tok[0], x.flatten(2).mean(2) + sd[a + "positional_embedding"][0], rtol=0, atol=1e-14)
    got = clip_resnet.attention_pool(sd, tok, heads)
    mha = torch.nn.MultiheadAttention(E, heads, dtype=torch.float64)
    mha.out_proj = torch.nn.Linear(E, out_dim, dtype=torch.float64)       # c_proj: E -> out_dim
    with torch.no_grad():
        mha.in_proj_weight.copy_(torch.cat([sd[f"{a}{p}_proj.weight"] for p in "qkv"]))
        mha.in_proj_bias.copy_(torch.cat([sd[f"{a}{p}_proj.bias"] for p in "qkv"]))
        mha.out_proj.weight.copy_(sd[a + "c_proj.weight"])
        mha.out_proj.bias.copy_(sd[a + "c_proj.bias"])
        full, _ = mha(tok, tok, tok, need_weights=False)      # every token as a query; row 0 is the pool's output
    torch.testing.assert_close(got, full[0], rtol=1e-12, atol=1e-12)
    pre = clip_resnet.attention_pool(sd, tok, heads, out_proj=False)
    torch.testing.assert_close(F.linear(pre, sd[a + "c_proj.weight"], sd[a + "c_proj.bias"]), got, rtol=1e-12, atol=1e-12)


def test_chained_blocks_reproduce_trunk_and_forward():
    """block_inputs + block, chained, give the float64 trunk's layer outputs and the features bit for bit: the block
    tests compare the engine's blocks against exactly the computation the tower tests compare its stages against."""
    sd = {k: v.double() for k, v in clip_resnet.stand_in_state_dict("RN50").items()}
    cfg = clip_resnet.config(sd)
    x = clip_resnet.calibration_images(cfg["n_px"], seed=7, n=1).double()
    with torch.no_grad():
        ref, taps = clip_resnet.forward(sd, x, taps=True)
        ins = clip_resnet.block_inputs(sd, x, cfg)
        assert len(ins) == sum(cfg["layers"]) and torch.equal(ins[0], taps["stem"])
        y = ins[0]
        for i, (p, stride, L) in enumerate(clip_resnet.blocks(cfg)):
            assert torch.equal(y, ins[i]), p
            out, branch, short = clip_resnet.block(sd, cfg, i, y)
            assert torch.equal(out, torch.relu(short + branch)), p
            if i + 1 == len(ins) or clip_resnet.blocks(cfg)[i + 1][2] != L:
                assert torch.equal(out, taps[f"layer{L + 1}"]), p
            y = out
        feats = clip_resnet.attention_pool(sd, clip_resnet.pool_tokens(sd, y), cfg["heads"])
    assert torch.equal(feats, ref)


def _eff(t):
    hi, lo = lay.split(t)
    return hi.double() + lo.double()


def _launch(V, f):
    """emulate() on a volume (n, Hp, Wp, pitch) -> (n, n_out, Hp - 2, Wp - 2) valid region."""
    n, hp, wp, pitch = V.shape
    y = lay.emulate(V.reshape(-1, pitch), f, wp).reshape(n, hp, wp, -1)
    return y[:, 1:hp - 1, 1:wp - 1].permute(0, 3, 1, 2)


@pytest.mark.parametrize("ci,co,S", [(8, 16, 5), (40, 24, 4), (48, 8, 3)])
def test_pooled_1x1_over_phase_repack_equals_avgpool_conv(ci, co, S):
    g = torch.Generator().manual_seed(ci)
    x = torch.randn(2, ci, 2 * S, 2 * S, generator=g)
    w = torch.randn(co, ci, 1, 1, generator=g)
    f = lay.pooled_filter(w)
    y = _launch(lay.phase_repack(lay.volume(x)), f) * 0.25            # the 1/4 is the epilogue scale's
    ref = F.conv2d(F.avg_pool2d(_eff(x), 2), _eff(w))
    torch.testing.assert_close(y, ref, rtol=1e-12, atol=1e-12)
    assert f["lo_mask"] == 0                                        # every 64-column block meets a hi half


@pytest.mark.parametrize("npx", [32, 48])
def test_stem_over_the_transform_phase_volume_equals_conv(npx):
    g = torch.Generator().manual_seed(npx)
    x = torch.randn(2, 3, npx, npx, generator=g)
    w = torch.randn(16, 3, 3, 3, generator=g)
    y = _launch(lay.stem_phase_volume(x), lay.stem_filter(w))
    torch.testing.assert_close(y, F.conv2d(_eff(x), _eff(w), stride=2, padding=1), rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("k", [1, 3])
def test_same_filter_equals_conv(k):
    g = torch.Generator().manual_seed(k)
    x = torch.randn(2, 40, 6, 7, generator=g)
    w = torch.randn(24, 40, k, k, generator=g)
    y = _launch(lay.volume(x), lay.same_filter(w))
    torch.testing.assert_close(y, F.conv2d(_eff(x), _eff(w), padding=k // 2), rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("name", list(clip_resnet.TOWERS))
def test_configuration_inference(name):
    layers, width, n_px, out_dim = clip_resnet.TOWERS[name]
    cfg = clip_resnet.config(clip_resnet.stand_in_state_dict(name))
    E = 32 * width
    assert cfg == dict(layers=layers, width=width, n_px=n_px, embed=E, heads=E // 64, out_dim=out_dim,
                       tokens=(n_px // 32) ** 2 + 1)


def test_configuration_names_a_missing_or_missized_key():
    sd = clip_resnet.stand_in_state_dict("RN50")
    bad = dict(sd)
    del bad["visual.layer2.1.bn3.running_mean"]
    with pytest.raises(KeyError, match="visual.layer2.1.bn3.running_mean"):
        clip_resnet.config(bad)
    bad = dict(sd)
    bad["visual.attnpool.v_proj.bias"] = torch.zeros(7)
    with pytest.raises(ValueError, match="visual.attnpool.v_proj.bias"):
        clip_resnet.config(bad)


def test_preprocess_at_224_equals_the_vit_transform():
    """At 224 the towers' transform is oracle.clip_preprocess's, bit for bit."""
    rng = np.random.default_rng(7)
    for h, w in ((240, 320), (224, 300), (500, 400)):
        frame = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        assert torch.equal(clip_resnet.preprocess_frame(frame, 224), clip_preprocess.preprocess_frame(frame))


@pytest.mark.parametrize("size", [288, 384])
def test_preprocess_at_size_equals_pil_and_torchvision(size):
    from PIL import Image
    from torchvision.transforms import functional as TF
    rng = np.random.default_rng(size)
    for h, w in ((240, 320), (400, 300), (size, 500)):
        frame = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        got = clip_resnet.preprocess_frame(frame, size)
        img = Image.fromarray(frame)
        short = min(h, w)
        if short != size:
            oh, ow = (size, int(size * w / h)) if h <= w else (int(size * h / w), size)
            img = img.resize((ow, oh), Image.BICUBIC)
        t = TF.normalize(TF.to_tensor(TF.center_crop(img, size)), clip_preprocess.MEAN, clip_preprocess.STD)
        assert got.shape == (3, size, size)
        assert torch.equal(got, t), (h, w)


def _args(feature_type):
    return argparse.Namespace(feature_type=feature_type, video_paths=[SAMPLE], flow_paths=None,
                              file_with_video_paths=None, video_dir=None, flow_dir=None, extraction_fps=None,
                              extract_method="uni_4", on_extraction="save_numpy", output_path="/nonexistent",
                              output_direct=True, tmp_path="/nonexistent/tmp")


@pytest.mark.parametrize("name,file", [("CLIP-RN50", "RN50.pt"), ("CLIP-RN101", "RN101.pt"),
                                       ("CLIP-RN50x4", "RN50x4.pt"), ("CLIP-RN50x16", "RN50x16.pt")])
def test_extract_clip_takes_the_resnet_towers(name, file, monkeypatch, tmp_path):
    from video_features_b200.extract import extract_clip
    ex = extract_clip.ExtractCLIP(_args(name))
    assert ex.feature_type == name
    monkeypatch.delenv("VF_CLIP_CKPT", raising=False)
    monkeypatch.setenv("VF_CLIP_SYNTHETIC", "0")              # seeded ViT weights do not stand in for a ResNet tower
    monkeypatch.setenv("HOME", str(tmp_path))
    with pytest.raises(FileNotFoundError, match=file) as e:
        extract_clip.load_clip_state_dict(name)
    assert os.path.join(str(tmp_path), ".cache", "clip", file) in str(e.value)


def test_resnet_stand_in_checkpoint_reads_back(tmp_path):
    from video_features_b200.extract.extract_clip import read_clip_checkpoint
    sd = clip_resnet.stand_in_state_dict("RN50")
    path = str(tmp_path / "RN50.pt")
    torch.save(sd, path)
    back = read_clip_checkpoint(path)
    assert set(back) == set(sd) and all(torch.equal(back[k], sd[k]) for k in sd)


def test_other_names_stay_refused():
    from video_features_b200.extract.extract_clip import ExtractCLIP
    ex = ExtractCLIP(_args("CLIP-RN50x64"))
    with pytest.raises(NotImplementedError, match="CLIP-RN50x64"):
        ex._engine(torch.device("cuda", 0))


def test_emulation_script_runs_at_a_tiny_size():
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, os.path.join(root, "scripts", "precision", "emulate_clip_rn.py"), "--tiny"],
                       capture_output=True, text=True, cwd=root, timeout=600)
    assert r.returncode == 0, r.stderr
    assert "weights" in r.stdout and "attn_out" in r.stdout

"""VideoMAE without a GPU: checkpoint lookup order and its refusals, the config and preset checks, the stack-size
refusals of the CLI and the extractor, and the ABI declarations."""
import argparse
import json
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import videomae_net as V  # noqa: E402
from video_features_b200 import videomae_engine as E  # noqa: E402
from video_features_b200.extract import extract_videomae as X  # noqa: E402

NAME = "videomae_vits16"


def _write(d, cfg=None, weights=True, pre=None):
    os.makedirs(d, exist_ok=True)
    with open(os.path.join(d, "config.json"), "w") as f:
        json.dump(cfg or V.config_dict(NAME, depth=1), f)
    if weights:
        torch.save(dict(V.stand_in_state_dict(NAME, depth=1)), os.path.join(d, "pytorch_model.bin"))
    if pre is not None:
        with open(os.path.join(d, "preprocessor_config.json"), "w") as f:
            json.dump(pre, f)


@pytest.fixture
def env(tmp_path, monkeypatch):
    for k in ("VF_CKPT_DIR", "HF_HUB_CACHE", "HF_HOME"):
        monkeypatch.delenv(k, raising=False)
    monkeypatch.setenv("HOME", str(tmp_path / "home"))
    monkeypatch.setattr(X, "_CHECKPOINTS", {})
    return tmp_path


def test_lookup_order(env, monkeypatch):
    repo = "videomae-small-finetuned-kinetics"
    snap = env / "hub" / f"models--MCG-NJU--{repo}" / "snapshots" / "abc"
    _write(str(snap))
    monkeypatch.setenv("HF_HUB_CACHE", str(env / "hub"))
    assert X.find_checkpoint(NAME) == str(snap)
    _write(str(env / "ckpt" / repo))
    monkeypatch.setenv("VF_CKPT_DIR", str(env / "ckpt"))
    assert X.find_checkpoint(NAME) == str(env / "ckpt" / repo)
    monkeypatch.delenv("HF_HUB_CACHE")
    monkeypatch.setenv("HF_HOME", str(env / "hf"))
    assert X.candidate_dirs(NAME) == [str(env / "ckpt" / repo)]
    monkeypatch.delenv("HF_HOME")
    home_snap = env / "home" / ".cache" / "huggingface" / "hub" / f"models--MCG-NJU--{repo}" / "snapshots" / "s1"
    _write(str(home_snap))
    assert X.candidate_dirs(NAME)[-1] == str(home_snap)


def test_lookup_needs_weights(env, monkeypatch):
    _write(str(env / "ckpt" / "videomae-small-finetuned-kinetics"), weights=False)
    monkeypatch.setenv("VF_CKPT_DIR", str(env / "ckpt"))
    with pytest.raises(FileNotFoundError, match="model.safetensors"):
        X.find_checkpoint(NAME)


def test_width_must_match_the_feature_type(env, monkeypatch):
    _write(str(env / "ckpt" / "videomae-base-finetuned-kinetics"))
    monkeypatch.setenv("VF_CKPT_DIR", str(env / "ckpt"))
    with pytest.raises(ValueError, match="hidden_size 384, not 768"):
        X.load_videomae("videomae_vitb16")


def test_config_refusals():
    E.VideoMAEConfig.from_dict(V.config_dict(NAME))
    with pytest.raises(ValueError, match="head dim 80"):
        E.VideoMAEConfig.from_dict(V.config_dict(NAME, hidden_size=1280, num_attention_heads=16))
    with pytest.raises(ValueError, match="use_mean_pooling"):
        E.VideoMAEConfig.from_dict(V.config_dict(NAME, use_mean_pooling=False))
    for key, val in (("num_frames", 32), ("tubelet_size", 1), ("image_size", 288)):
        with pytest.raises(ValueError, match=key):
            E.VideoMAEConfig.from_dict(V.config_dict(NAME, **{key: val}))


def test_state_dict_checks_name_the_key():
    cfg = E.VideoMAEConfig.from_dict(V.config_dict(NAME, depth=2))
    sd = dict(V.stand_in_state_dict(NAME, depth=2))
    E.check_state_dict(sd, cfg)
    key = "videomae.encoder.layer.1.attention.attention.v_bias"
    with pytest.raises(ValueError, match=key.replace(".", r"\.")):
        E.check_state_dict({k: v for k, v in sd.items() if k != key}, cfg)
    key = "videomae.encoder.layer.0.intermediate.dense.weight"
    with pytest.raises(ValueError, match="shape"):
        E.check_state_dict(dict(sd, **{key: sd[key][:-1]}), cfg)


def test_stray_qkv_bias_refused():
    cfg = E.VideoMAEConfig.from_dict(V.config_dict(NAME, depth=1, qkv_bias=False))
    sd = dict(V.stand_in_state_dict(NAME, depth=1))
    with pytest.raises(ValueError, match="qkv_bias = false"):
        E.check_state_dict(sd, cfg)
    E.check_state_dict({k: v for k, v in sd.items() if not k.endswith(("q_bias", "v_bias"))}, cfg)


def test_preset():
    assert E.Preset.from_dict(None) == E.Preset(mean=V.IMAGENET_MEAN, std=V.IMAGENET_STD)
    p = E.Preset.from_dict({"image_mean": [0.5, 0.5, 0.5], "image_std": [0.5, 0.5, 0.5], "resample": 2,
                            "size": {"shortest_edge": 224}, "crop_size": {"height": 224, "width": 224}})
    assert p.mean == (0.5, 0.5, 0.5)
    with pytest.raises(ValueError, match="resample"):
        E.Preset.from_dict({"resample": 3})
    with pytest.raises(ValueError, match="shortest_edge"):
        E.Preset.from_dict({"size": {"shortest_edge": 256}})


def test_class_names():
    cfg = E.VideoMAEConfig.from_dict(V.config_dict(NAME, id2label={"0": "a", "1": "b"}))
    assert cfg.class_names(2) == ["a", "b"] and cfg.class_names(3) is None
    bare = E.VideoMAEConfig.from_dict(V.config_dict(NAME, id2label={"0": "LABEL_0", "1": "LABEL_1"}))
    assert bare.class_names(2) is None


def _ns(**kw):
    d = dict(feature_type=NAME, video_paths=[os.path.join(ROOT, "tests", "golden", "v_GGSY1Qvo990.mp4")], flow_paths=None, file_with_video_paths=None, video_dir=None,
             flow_dir=None, extraction_fps=None, on_extraction='save_numpy', output_path='./output', tmp_path='./tmp',
             show_pred=False, keep_tmp_files=False, stack_size=None, step_size=None, device_ids=[0])
    d.update(kw)
    return argparse.Namespace(**d)


def test_stack_size_refused():
    from video_features_b200.utils import sanity_check
    with pytest.raises(AssertionError, match="16"):
        sanity_check(_ns(stack_size=8))
    sanity_check(_ns(stack_size=16))
    with pytest.raises(ValueError, match="16"):
        X.ExtractVideoMAE(_ns(stack_size=24))


def test_cli_lists_the_types():
    import main
    for n in E.FEATURE_TYPES:
        assert n in main.SUPPORTED and n in main._FEATURE_TYPES


def test_abi_declared():
    from video_features_b200 import _lib
    for n in ("create", "destroy", "info", "forward_u8", "forward_f32", "attention", "debug_drop_lo", "launch_count"):
        assert f"vf_videomae_{n}" in _lib.SIGNATURES
    text = open(os.path.join(ROOT, "include", "vfeat.h")).read()
    assert "int vf_videomae_create(" in text and "int vf_videomae_attention(" in text

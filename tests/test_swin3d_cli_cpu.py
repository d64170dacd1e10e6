"""`main.py --feature_type swin3d_t|swin3d_s|swin3d_b` reaches ExtractSwin3D; its attributes, refusals and weight lookup
need no GPU."""
import os

import pytest
import torch

import main

TYPES = ["swin3d_t", "swin3d_s", "swin3d_b"]


def _args(tmp_path, ft, *extra):
    a = str(tmp_path / "a.mp4")
    open(a, "wb").close()
    return main.make_parser().parse_args(["--feature_type", ft, "--video_paths", a,
                                          "--output_path", str(tmp_path / "out"), "--on_extraction", "save_numpy",
                                          *extra]), a


@pytest.mark.parametrize("ft", TYPES)
def test_cli_builds_swin3d_extractor(tmp_path, ft):
    from video_features_b200.extract.extract_swin3d import ExtractSwin3D
    assert ft in main.SUPPORTED
    args, a = _args(tmp_path, ft)
    ex = main.build_extractor(args)
    assert isinstance(ex, ExtractSwin3D) and ex.feature_type == ft
    assert ex.path_list == [a]
    assert ex.output_path == os.path.join(str(tmp_path / "out"), ft)
    assert ex.stack_size == 32 and ex.step_size == 32
    assert ex.extraction_fps is None and ex.show_pred is False and ex.on_extraction == "save_numpy"
    args, _ = _args(tmp_path, ft, "--stack_size", "17", "--step_size", "8")
    ex = main.build_extractor(args)
    assert ex.stack_size == 17 and ex.step_size == 8


@pytest.mark.parametrize("ft", TYPES)
def test_extraction_fps_is_refused(tmp_path, ft):
    args, _ = _args(tmp_path, ft, "--extraction_fps", "2")
    with pytest.raises(NotImplementedError, match="extraction_fps re-encodes with ffmpeg"):
        main.build_extractor(args)


@pytest.mark.parametrize("ft", TYPES)
def test_model_name_is_refused(tmp_path, ft):
    from video_features_b200.utils import sanity_check
    args, _ = _args(tmp_path, ft, "--model_name", "r2plus1d_18_16_kinetics")
    with pytest.raises(AssertionError, match="r21d_rgb"):
        sanity_check(args)


def test_show_pred_help_names_swin3d():
    helps = {a.dest: a.help for a in main.make_parser()._actions}
    assert "Swin3D" in helps["show_pred"] and "S3D" in helps["show_pred"]


@pytest.mark.parametrize("ft,pattern,name", [("swin3d_t", "swin3d_t-*.pth", "swin3d_t-7615ae03.pth"),
                                             ("swin3d_s", "swin3d_s-*.pth", "swin3d_s-da41c237.pth"),
                                             ("swin3d_b", "swin3d_b_1k-*.pth", "swin3d_b_1k-24f7c7c6.pth")])
def test_missing_weights_name_the_pattern(tmp_path, monkeypatch, ft, pattern, name):
    from video_features_b200.extract import extract_swin3d
    monkeypatch.setenv("VF_CKPT_DIR", str(tmp_path / "none"))
    monkeypatch.setenv("TORCH_HOME", str(tmp_path / "th"))
    monkeypatch.setattr(extract_swin3d, "_STATE_DICTS", {})
    with pytest.raises(FileNotFoundError) as e:
        extract_swin3d.load_swin3d_weights(ft)
    assert pattern in str(e.value) and str(tmp_path / "none") in str(e.value)
    d = tmp_path / "th" / "hub" / "checkpoints"
    d.mkdir(parents=True)
    if ft == "swin3d_b":          # the IN-22k checkpoint is not the Kinetics-400 one
        torch.save({"x": torch.zeros(1)}, str(d / "swin3d_b_22k-7c6ae6fa.pth"))
        with pytest.raises(FileNotFoundError):
            extract_swin3d.load_swin3d_weights(ft)
    torch.save({"x": torch.ones(1)}, str(d / name))
    assert float(extract_swin3d.load_swin3d_weights(ft)["x"]) == 1.0


@pytest.mark.parametrize("ft", TYPES)
def test_show_pred_without_head_is_a_key_error(tmp_path, monkeypatch, ft):
    from video_features_b200.extract import extract_swin3d
    monkeypatch.setattr(extract_swin3d, "_STATE_DICTS", {ft: {"patch_embed.proj.weight": torch.zeros(1)}})
    args, _ = _args(tmp_path, ft, "--show_pred")
    ex = main.build_extractor(args)
    with pytest.raises(KeyError, match="head.weight"):
        ex._head(torch.device("cuda", 0))

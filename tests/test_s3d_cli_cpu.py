"""`main.py --feature_type s3d` reaches ExtractS3D; its attributes, refusals and weight lookup need no GPU."""
import os

import pytest
import torch

import main


def _args(tmp_path, *extra):
    a = str(tmp_path / "a.mp4")
    open(a, "wb").close()
    return main.make_parser().parse_args(["--feature_type", "s3d", "--video_paths", a,
                                          "--output_path", str(tmp_path / "out"), "--on_extraction", "save_numpy",
                                          *extra]), a


def test_cli_builds_s3d_extractor(tmp_path):
    from video_features_b200.extract.extract_s3d import ExtractS3D
    assert "s3d" in main.SUPPORTED
    args, a = _args(tmp_path)
    ex = main.build_extractor(args)
    assert isinstance(ex, ExtractS3D)
    assert ex.path_list == [a]
    assert ex.output_path == os.path.join(str(tmp_path / "out"), "s3d")
    assert ex.stack_size == 64 and ex.step_size == 64
    assert ex.extraction_fps is None and ex.show_pred is False and ex.on_extraction == "save_numpy"
    args, _ = _args(tmp_path, "--stack_size", "13", "--step_size", "20")
    ex = main.build_extractor(args)
    assert ex.stack_size == 13 and ex.step_size == 20


def test_short_stacks_are_refused(tmp_path):
    args, _ = _args(tmp_path, "--stack_size", "12")
    with pytest.raises(ValueError, match="13"):
        main.build_extractor(args)


def test_extraction_fps_is_refused(tmp_path):
    args, _ = _args(tmp_path, "--extraction_fps", "2")
    with pytest.raises(NotImplementedError, match="extraction_fps re-encodes with ffmpeg"):
        main.build_extractor(args)


def test_show_pred_help_names_s3d():
    helps = {a.dest: a.help for a in main.make_parser()._actions}
    assert "S3D" in helps["show_pred"]


def test_missing_weights_name_the_pattern(tmp_path, monkeypatch):
    from video_features_b200.extract import extract_s3d
    monkeypatch.setenv("VF_CKPT_DIR", str(tmp_path / "none"))
    monkeypatch.setenv("TORCH_HOME", str(tmp_path / "th"))
    monkeypatch.setattr(extract_s3d, "_STATE_DICT", {})
    with pytest.raises(FileNotFoundError) as e:
        extract_s3d.load_s3d_weights()
    assert "s3d-*.pth" in str(e.value) and str(tmp_path / "none") in str(e.value)
    d = tmp_path / "th" / "hub" / "checkpoints"
    d.mkdir(parents=True)
    torch.save({"x": torch.ones(1)}, str(d / "s3d-d76dad2f.pth"))
    assert float(extract_s3d.load_s3d_weights()["x"]) == 1.0


def test_show_pred_without_classifier_is_a_key_error(tmp_path, monkeypatch):
    from video_features_b200.extract import extract_s3d
    monkeypatch.setattr(extract_s3d, "_STATE_DICT", {"features.0.0.0.weight": torch.zeros(1)})
    args, _ = _args(tmp_path, "--show_pred")
    ex = main.build_extractor(args)
    with pytest.raises(KeyError, match="classifier.1.weight"):
        ex._head(torch.device("cuda", 0))

"""`main.py --feature_type r21d_rgb` reaches ExtractR21D; its attributes, refusals and weight lookup need no GPU."""
import os

import pytest

import main


def _args(tmp_path, *extra):
    a = str(tmp_path / "a.mp4")
    open(a, "wb").close()
    return main.make_parser().parse_args(["--feature_type", "r21d_rgb", "--video_paths", a,
                                          "--output_path", str(tmp_path / "out"), "--on_extraction", "save_numpy",
                                          *extra]), a


def test_cli_builds_r21d_extractor(tmp_path):
    from video_features_b200.extract.extract_r21d import ExtractR21D
    args, a = _args(tmp_path)
    ex = main.build_extractor(args)
    assert isinstance(ex, ExtractR21D)
    assert ex.path_list == [a]
    assert ex.output_path == os.path.join(str(tmp_path / "out"), "r21d_rgb")
    assert ex.tmp_path == os.path.join("./tmp", "r21d_rgb")
    # the reference's defaults: 16-frame stacks every 16 frames, a 112 crop
    assert ex.stack_size == 16 and ex.step_size == 16 and ex.central_crop_min_side_size == 112
    assert ex.extraction_fps is None and ex.show_pred is False and ex.keep_tmp_files is False
    assert ex.on_extraction == "save_numpy"
    args, _ = _args(tmp_path, "--stack_size", "8", "--step_size", "20")
    ex = main.build_extractor(args)
    assert ex.stack_size == 8 and ex.step_size == 20


def test_extraction_fps_is_refused(tmp_path):
    args, _ = _args(tmp_path, "--extraction_fps", "2")
    with pytest.raises(NotImplementedError, match="extraction_fps re-encodes with ffmpeg"):
        main.build_extractor(args)


def test_missing_weights_name_the_places_searched(tmp_path, monkeypatch):
    from video_features_b200.extract import extract_r21d
    monkeypatch.setenv("VF_CKPT_DIR", str(tmp_path / "none"))
    monkeypatch.setenv("TORCH_HOME", str(tmp_path / "th"))
    monkeypatch.setattr(extract_r21d, "_STATE_DICT", {})
    with pytest.raises(FileNotFoundError) as e:
        extract_r21d.load_r21d_weights()
    assert "r2plus1d_18-*.pth" in str(e.value) and str(tmp_path / "none") in str(e.value)
    assert os.path.join(str(tmp_path / "th"), "hub", "checkpoints") in str(e.value)
    # the first matching file of the first directory that has one
    import torch
    d = tmp_path / "th" / "hub" / "checkpoints"
    d.mkdir(parents=True)
    torch.save({"x": torch.ones(1)}, str(d / "r2plus1d_18-91a641e6.pth"))
    assert float(extract_r21d.load_r21d_weights()["x"]) == 1.0

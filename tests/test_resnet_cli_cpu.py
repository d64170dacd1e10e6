"""`main.py --feature_type resnetXX` reaches ExtractResNet; its refusals and weight lookup need no GPU."""
import os

import pytest

import main


@pytest.mark.parametrize("depth", [18, 34, 50, 101, 152])
def test_cli_builds_resnet_extractor(depth, tmp_path):
    from video_features_b200.extract.extract_resnet import ExtractResNet
    a, b = str(tmp_path / "a.mp4"), str(tmp_path / "b.mp4")
    for p in (a, b):
        open(p, "wb").close()
    args = main.make_parser().parse_args(["--feature_type", f"resnet{depth}", "--video_paths", a, b,
                                          "--output_path", str(tmp_path / "out"), "--on_extraction", "save_numpy"])
    ex = main.build_extractor(args)
    assert isinstance(ex, ExtractResNet) and ex.depth == depth
    assert ex.path_list == [a, b]
    assert ex.output_path == os.path.join(str(tmp_path / "out"), f"resnet{depth}")
    assert ex.batch_size == 1 and ex.central_crop_size == 224 and ex.extraction_fps is None


def test_extraction_fps_is_refused(tmp_path):
    a = str(tmp_path / "a.mp4")
    open(a, "wb").close()
    args = main.make_parser().parse_args(["--feature_type", "resnet50", "--video_paths", a,
                                          "--extraction_fps", "2"])
    with pytest.raises(NotImplementedError, match="extraction_fps re-encodes with ffmpeg"):
        main.build_extractor(args)


def test_missing_weights_name_the_places_searched(tmp_path, monkeypatch):
    from video_features_b200.extract import extract_resnet
    monkeypatch.setenv("VF_CKPT_DIR", str(tmp_path / "none"))
    monkeypatch.setenv("TORCH_HOME", str(tmp_path / "th"))
    monkeypatch.setattr(extract_resnet, "_STATE_DICTS", {})
    with pytest.raises(FileNotFoundError) as e:
        extract_resnet.load_resnet_weights(34)
    assert "resnet34-*.pth" in str(e.value) and str(tmp_path / "none") in str(e.value)
    assert os.path.join(str(tmp_path / "th"), "hub", "checkpoints") in str(e.value)
    # the first matching file of the first directory that has one
    import torch
    d = tmp_path / "th" / "hub" / "checkpoints"
    d.mkdir(parents=True)
    torch.save({"x": torch.ones(1)}, str(d / "resnet34-b627a593.pth"))
    assert float(extract_resnet.load_resnet_weights(34)["x"]) == 1.0

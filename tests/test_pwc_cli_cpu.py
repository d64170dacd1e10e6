"""`main.py --feature_type pwc` reaches ExtractPWC, and ExtractI3D accepts its default flow type; neither needs a GPU to
be constructed."""
import os

import pytest

import main


def test_cli_builds_pwc_extractor(tmp_path):
    from video_features_b200.extract.extract_pwc import ExtractPWC
    a = str(tmp_path / "a.mp4")
    open(a, "wb").close()
    args = main.make_parser().parse_args(["--feature_type", "pwc", "--video_paths", a, "--output_path",
                                          str(tmp_path / "out"), "--batch_size", "4", "--side_size", "128"])
    ex = main.build_extractor(args)
    assert isinstance(ex, ExtractPWC)
    assert ex.path_list == [a] and ex.feature_type == "pwc"
    assert ex.output_path == os.path.join(str(tmp_path / "out"), "pwc")
    assert ex.batch_size == 4 and ex.side_size == 128 and ex.resize_to_smaller_edge is True
    assert ex.pairs_per_call >= 4


def test_i3d_default_flow_type_constructs(tmp_path):
    from video_features_b200.extract.extract_i3d import ExtractI3D
    a = str(tmp_path / "a.mp4")
    open(a, "wb").close()
    args = main.make_parser().parse_args(["--feature_type", "i3d", "--video_paths", a])
    assert args.flow_type == "pwc"
    ex = main.build_extractor(args)
    assert isinstance(ex, ExtractI3D) and ex.flow_type == "pwc" and ex.streams == ["rgb", "flow"]


def test_pwc_extraction_fps_is_refused(tmp_path):
    a = str(tmp_path / "a.mp4")
    open(a, "wb").close()
    args = main.make_parser().parse_args(["--feature_type", "pwc", "--video_paths", a, "--extraction_fps", "2"])
    with pytest.raises(NotImplementedError, match="extraction_fps re-encodes with ffmpeg"):
        main.build_extractor(args)


def test_only_vggish_stays_refused(tmp_path):
    a = str(tmp_path / "a.mp4")
    open(a, "wb").close()
    for ft in ("vggish", "vggish_torch"):
        args = main.make_parser().parse_args(["--feature_type", ft, "--video_paths", a])
        with pytest.raises(NotImplementedError):
            main.build_extractor(args)

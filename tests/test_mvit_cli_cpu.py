"""`main.py --feature_type mvit_v1_b|mvit_v2_s` reaches ExtractMViT; its attributes, refusals and weight lookup need no
GPU."""
import os

import pytest
import torch

import main

TYPES = ["mvit_v1_b", "mvit_v2_s"]


def _args(tmp_path, ft, *extra):
    a = str(tmp_path / "a.mp4")
    open(a, "wb").close()
    return main.make_parser().parse_args(["--feature_type", ft, "--video_paths", a,
                                          "--output_path", str(tmp_path / "out"), "--on_extraction", "save_numpy",
                                          *extra]), a


@pytest.mark.parametrize("ft", TYPES)
def test_cli_builds_mvit_extractor(tmp_path, ft):
    from video_features_b200.extract.extract_mvit import ExtractMViT
    assert ft in main.SUPPORTED
    args, a = _args(tmp_path, ft)
    ex = main.build_extractor(args)
    assert isinstance(ex, ExtractMViT) and ex.feature_type == ft
    assert ex.path_list == [a]
    assert ex.output_path == os.path.join(str(tmp_path / "out"), ft)
    assert ex.stack_size == 16 and ex.step_size == 16
    assert ex.extraction_fps is None and ex.show_pred is False and ex.on_extraction == "save_numpy"
    args, _ = _args(tmp_path, ft, "--stack_size", "16", "--step_size", "8")
    ex = main.build_extractor(args)
    assert ex.stack_size == 16 and ex.step_size == 8


@pytest.mark.parametrize("ft", TYPES)
@pytest.mark.parametrize("stack", ["8", "32"])
def test_other_stack_sizes_are_refused(tmp_path, ft, stack):
    args, _ = _args(tmp_path, ft, "--stack_size", stack)
    with pytest.raises(ValueError, match="position tables fix T = 16"):
        main.build_extractor(args)


@pytest.mark.parametrize("ft", TYPES)
def test_extraction_fps_is_refused(tmp_path, ft):
    args, _ = _args(tmp_path, ft, "--extraction_fps", "2")
    with pytest.raises(NotImplementedError, match="extraction_fps re-encodes with ffmpeg"):
        main.build_extractor(args)


def test_help_names_mvit():
    helps = {a.dest: a.help for a in main.make_parser()._actions}
    assert "MViT" in helps["show_pred"] and "MViT" in helps["stack_size"]


@pytest.mark.parametrize("ft,pattern,name", [("mvit_v1_b", "mvit_v1_b-*.pth", "mvit_v1_b-dbeb1030.pth"),
                                             ("mvit_v2_s", "mvit_v2_s-*.pth", "mvit_v2_s-ae3be167.pth")])
def test_missing_weights_name_the_pattern(tmp_path, monkeypatch, ft, pattern, name):
    from video_features_b200.extract import extract_mvit
    monkeypatch.setenv("VF_CKPT_DIR", str(tmp_path / "none"))
    monkeypatch.setenv("TORCH_HOME", str(tmp_path / "th"))
    monkeypatch.setattr(extract_mvit, "_STATE_DICTS", {})
    with pytest.raises(FileNotFoundError) as e:
        extract_mvit.load_mvit_weights(ft)
    assert pattern in str(e.value) and str(tmp_path / "none") in str(e.value)
    d = tmp_path / "th" / "hub" / "checkpoints"
    d.mkdir(parents=True)
    torch.save({"x": torch.ones(1)}, str(d / name))
    assert float(extract_mvit.load_mvit_weights(ft)["x"]) == 1.0


@pytest.mark.parametrize("ft", TYPES)
def test_show_pred_without_head_is_a_key_error(tmp_path, monkeypatch, ft):
    from video_features_b200.extract import extract_mvit
    monkeypatch.setattr(extract_mvit, "_STATE_DICTS", {ft: {"conv_proj.weight": torch.zeros(1)}})
    args, _ = _args(tmp_path, ft, "--show_pred")
    ex = main.build_extractor(args)
    with pytest.raises(KeyError, match="head.1.weight"):
        ex._head(torch.device("cuda", 0))


def test_variant_is_inferred_from_the_keys():
    """The oracle infers the variant from the same keys the engine's create does (v2: rel-pos tables, v1: absolute
    position embeddings), with or without the "module." prefix, and refuses a state dict of neither; the engine's own
    refusal of a wrong-shape key, named, is tests/test_mvit_gpu.py::test_refuses_other_shapes."""
    from oracle import mvit_net as M
    for ft in TYPES:
        sd = M.stand_in_state_dict(ft)
        assert M.config(sd) == ft and M.config({"module." + k: v for k, v in sd.items()}) == ft
    with pytest.raises(ValueError):
        M.config({"conv_proj.weight": torch.zeros(1)})

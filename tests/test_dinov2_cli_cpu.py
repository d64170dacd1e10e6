"""`main.py --feature_type dinov2_*` reaches ExtractDINOv2; its attributes, refusals, weight lookup and the engine's
shape refusals need no GPU."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

import main
from oracle import dinov2_net as D

TYPES = list(D.MODELS)


def _args(tmp_path, ft, *extra):
    a = str(tmp_path / "a.mp4")
    open(a, "wb").close()
    return main.make_parser().parse_args(["--feature_type", ft, "--video_paths", a,
                                          "--output_path", str(tmp_path / "out"), "--on_extraction", "save_numpy",
                                          *extra]), a


@pytest.mark.parametrize("ft", TYPES)
def test_cli_builds_dinov2_extractor(tmp_path, ft):
    from video_features_b200.extract.extract_dinov2 import ExtractDINOv2
    assert ft in main.SUPPORTED
    args, a = _args(tmp_path, ft)
    ex = main.build_extractor(args)
    assert isinstance(ex, ExtractDINOv2) and ex.feature_type == ft
    assert ex.path_list == [a]
    assert ex.output_path == os.path.join(str(tmp_path / "out"), ft)
    assert ex.extraction_fps is None and ex.show_pred is False and ex.on_extraction == "save_numpy"


@pytest.mark.parametrize("ft", TYPES)
def test_extraction_fps_is_refused(tmp_path, ft):
    args, _ = _args(tmp_path, ft, "--extraction_fps", "2")
    with pytest.raises(NotImplementedError, match="extraction_fps re-encodes with ffmpeg"):
        main.build_extractor(args)


@pytest.mark.parametrize("flags,match", [(("--show_pred",), "without a classifier"),
                                         (("--stack_size", "16"), "stacks do not apply"),
                                         (("--model_name", "r2plus1d_18_16_kinetics"), "r21d_rgb")])
def test_flags_that_do_not_apply_are_refused(tmp_path, flags, match):
    from video_features_b200.utils import sanity_check
    for ft in ("dinov2_vits14", "dinov2_vitg14_reg"):
        args, _ = _args(tmp_path, ft, *flags)
        with pytest.raises(AssertionError, match=match):
            sanity_check(args)


def test_show_pred_help_names_dinov2():
    helps = {a.dest: a.help for a in main.make_parser()._actions}
    assert "DINOv2" in helps["show_pred"]


@pytest.mark.parametrize("ft", TYPES)
def test_checkpoint_lookup_picks_the_hub_file(tmp_path, monkeypatch, ft):
    from video_features_b200.extract import extract_dinov2
    base = ft[:-4] if ft.endswith("_reg") else ft
    name = f"{base}_reg4_pretrain.pth" if ft.endswith("_reg") else f"{base}_pretrain.pth"
    assert extract_dinov2.checkpoint_name(ft) == name
    monkeypatch.setenv("VF_CKPT_DIR", str(tmp_path / "none"))
    monkeypatch.setenv("TORCH_HOME", str(tmp_path / "th"))
    monkeypatch.setattr(extract_dinov2, "_STATE_DICTS", {})
    with pytest.raises(FileNotFoundError) as e:
        extract_dinov2.load_dinov2_weights(ft)
    assert name in str(e.value) and str(tmp_path / "none") in str(e.value)
    d = tmp_path / "th" / "hub" / "checkpoints"
    d.mkdir(parents=True)
    other = f"{base}_pretrain.pth" if ft.endswith("_reg") else f"{base}_reg4_pretrain.pth"
    torch.save({"x": torch.zeros(1)}, str(d / other))     # the other family's file is not taken
    with pytest.raises(FileNotFoundError):
        extract_dinov2.load_dinov2_weights(ft)
    torch.save({"x": torch.ones(1)}, str(d / name))
    assert float(extract_dinov2.load_dinov2_weights(ft)["x"]) == 1.0
    (tmp_path / "none").mkdir()
    torch.save({"x": torch.full((1,), 2.0)}, str(tmp_path / "none" / name))    # $VF_CKPT_DIR first ...
    assert float(extract_dinov2.load_dinov2_weights(ft)["x"]) == 1.0            # ... but loaded once per process
    monkeypatch.setattr(extract_dinov2, "_STATE_DICTS", {})
    assert float(extract_dinov2.load_dinov2_weights(ft)["x"]) == 2.0


def _create_message(numels):
    """vf_dinov2_create's inference and refusals run on the sizes alone, before any tensor is read or a device is
    touched: every name points at one placeholder float.  Returns the error text."""
    from video_features_b200._lib import NamedTensor, VfError, check, lib
    dummy = np.zeros(1, np.float32)
    arr = (NamedTensor * len(numels))()
    names = [k.encode() for k in numels]
    for i, (nm, n) in enumerate(zip(names, numels.values())):
        arr[i].name = nm
        arr[i].data = dummy.ctypes.data_as(C.POINTER(C.c_float))
        arr[i].numel = n
    h = C.c_void_p()
    with pytest.raises(VfError) as e:
        check(lib().vf_dinov2_create(C.byref(h), arr, len(numels), 0, 1))
    return str(e.value)


def _numels(name):
    d, depth, ffn, reg = D.shape_of(name)
    sd = {k: v.numel() for k, v in D.stand_in_state_dict(name, depth=1).items() if not k.startswith("blocks.")}
    one = {k[len("blocks.0."):]: v.numel() for k, v in D.stand_in_state_dict(name, depth=1).items()
           if k.startswith("blocks.0.")}
    for i in range(depth):
        sd.update({f"blocks.{i}.{k}": n for k, n in one.items()})
    sd["pos_embed_224"] = 257 * d
    return sd


@pytest.mark.parametrize("change,key", [("width", "cls_token"), ("depth", "blocks.11.norm1.weight"),
                                        ("ffn", "blocks.0.mlp.w12.weight"), ("registers", "register_tokens"),
                                        ("table", "pos_embed_224")])
def test_wrong_shapes_are_refused_naming_the_key(change, key):
    sd = _numels("dinov2_vits14_reg" if change == "registers" else "dinov2_vits14")
    if change == "width":
        sd["cls_token"] = 512
    elif change == "depth":
        for k in [k for k in sd if k.startswith("blocks.11.")]:
            del sd[k]
    elif change == "ffn":
        sd["blocks.0.mlp.w12.weight"] = 2 * 4096 * 384
    elif change == "registers":
        sd["register_tokens"] = 2 * 384
    else:
        sd["pos_embed_224"] = 1370 * 384
    msg = _create_message(sd)
    assert key in msg, msg


@pytest.mark.parametrize("name,swap", [("dinov2_vitg14", True), ("dinov2_vitg14", False), ("dinov2_vits14", False)])
def test_a_missing_or_wrong_ffn_names_the_key(name, swap):
    """g without mlp.w12 (with the GELU MLP's fc1 instead, or with neither) and S without mlp.fc1 name the missing key."""
    sd = _numels(name)
    key = "blocks.0.mlp.w12.weight" if name == "dinov2_vitg14" else "blocks.0.mlp.fc1.weight"
    del sd[key]
    if swap:
        sd["blocks.0.mlp.fc1.weight"] = 4 * 1536 * 1536
    msg = _create_message(sd)
    assert f"'{key}' missing" in msg or f"missing tensor '{key}'" in msg, msg

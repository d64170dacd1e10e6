"""The IG65M R(2+1)D-34 models without a GPU: the depth-34 reference (tests/r21d_34_ref.py) against torchvision's
VideoResNet with the IG65M changes and, at depth 18, against oracle/r21d_net.py; `--model_name` on the CLI and the
weight lookup of the new models."""
import os

import pytest
import torch

import main
import r21d_34_ref as ref34
from oracle import r21d_net


def test_oracle_34_matches_torchvision():
    sd = ref34.stand_in_state_dict_34()
    net = ref34.r2plus1d_34()
    net.load_state_dict(sd)
    assert sum(v.numel() for v in net.parameters()) == 63_697_175          # 63.7 M with fc 512 -> 400
    assert all(m.eps == 1e-3 for m in net.modules() if isinstance(m, torch.nn.BatchNorm3d))
    # conv1 keeps torchvision's mid width, conv2 of layer2..4's first block is wider; elsewhere the two agree
    mids = {(L, b): (sd[f"layer{L}.{b}.conv1.0.0.weight"].shape[0], sd[f"layer{L}.{b}.conv2.0.0.weight"].shape[0])
            for L, n in zip(range(1, 5), ref34.LAYERS_34) for b in range(n)}
    assert mids[(2, 0)] == (230, 288) and mids[(3, 0)] == (460, 576) and mids[(4, 0)] == (921, 1152)
    assert all(a == b for (L, b_), (a, b) in mids.items() if not (b_ == 0 and L > 1))
    net.fc = torch.nn.Identity()
    net.eval()
    x = r21d_net.calibration_clips(seed=7, n=1, T=8)       # temporal sizes 8, 4, 2, 1
    with torch.no_grad():
        ref = net(x)
        y, taps = ref34.forward(sd, x, taps=True)
        y5 = ref34.forward(sd, x, eps=1e-5)
    assert y.shape == (1, 512)
    rel = float((y - ref).norm() / ref.norm())
    assert rel < 1e-5, rel
    assert float((y5 - ref).norm() / ref.norm()) > 1e-4           # the eps is seen
    assert [tuple(taps[s].shape[1:3]) for s in r21d_net.STAGES] == [(64, 8), (64, 8), (128, 4), (256, 2), (512, 1)]
    for name in r21d_net.STAGES:                              # calibrated: O(1) activations at every stage
        rms = float(taps[name].pow(2).mean().sqrt())
        assert 0.05 < rms < 20, (name, rms)


def test_reference_at_depth_18_is_the_oracle():
    """With r2plus1d_18's blocks and eps the depth-34 reference is oracle/r21d_net.forward bit for bit, stage by stage:
    it differs from the oracle only in what it reads from its arguments."""
    sd = r21d_net.stand_in_state_dict()
    x = r21d_net.calibration_clips(seed=3, n=1, T=4)
    with torch.no_grad():
        a, ta = r21d_net.forward(sd, x, taps=True)
        b, tb = ref34.forward(sd, x, taps=True, eps=1e-5, layers=ref34.LAYERS_18)
    assert torch.equal(a, b) and all(torch.equal(ta[s], tb[s]) for s in r21d_net.STAGES)
    assert "layer1.2.conv1.0.0.weight" not in sd and "layer1.2.conv1.0.0.weight" in ref34.stand_in_state_dict_34()


def _args(tmp_path, *extra, feature_type="r21d_rgb"):
    a = str(tmp_path / "a.mp4")
    open(a, "wb").close()
    return main.make_parser().parse_args(["--feature_type", feature_type, "--video_paths", a,
                                          "--output_path", str(tmp_path / "out"), "--on_extraction", "save_numpy",
                                          *extra])


@pytest.mark.parametrize("name,stack", [("r2plus1d_18_16_kinetics", 16), ("r2plus1d_34_32_ig65m_ft_kinetics", 32),
                                        ("r2plus1d_34_8_ig65m_ft_kinetics", 8)])
def test_cli_model_defaults_and_overrides(tmp_path, name, stack):
    from video_features_b200.extract.extract_r21d import ExtractR21D
    ex = main.build_extractor(_args(tmp_path, "--model_name", name))
    assert isinstance(ex, ExtractR21D) and ex.model_name == name
    assert ex.stack_size == stack and ex.step_size == stack
    assert ex.output_path == os.path.join(str(tmp_path / "out"), "r21d_rgb")       # one feature type, as upstream
    ex = main.build_extractor(_args(tmp_path, "--model_name", name, "--stack_size", "12", "--step_size", "5"))
    assert ex.stack_size == 12 and ex.step_size == 5


def test_cli_model_name_default_and_refusals(tmp_path):
    from video_features_b200.utils import sanity_check
    args = _args(tmp_path)
    assert args.model_name is None
    ex = main.build_extractor(args)
    assert ex.model_name == "r2plus1d_18_16_kinetics" and ex.stack_size == 16 and ex.step_size == 16
    sanity_check(_args(tmp_path, "--model_name", "r2plus1d_34_8_ig65m_ft_kinetics"))
    for ft in ("i3d", "s3d", "resnet18"):
        sanity_check(_args(tmp_path, feature_type=ft))
        with pytest.raises(AssertionError, match=f"--model_name .* does not apply to {ft}"):
            sanity_check(_args(tmp_path, "--model_name", "r2plus1d_34_8_ig65m_ft_kinetics", feature_type=ft))
    with pytest.raises(SystemExit):                  # argparse: not one of the choices
        _args(tmp_path, "--model_name", "r2plus1d_34")
    args.model_name = "r2plus1d_50"
    with pytest.raises(ValueError, match="unknown model_name 'r2plus1d_50'"):
        main.build_extractor(args)


def test_weight_lookup_of_the_34_layer_models(tmp_path, monkeypatch):
    from video_features_b200.extract import extract_r21d
    monkeypatch.setenv("VF_CKPT_DIR", str(tmp_path / "none"))
    monkeypatch.setenv("TORCH_HOME", str(tmp_path / "th"))
    monkeypatch.setattr(extract_r21d, "_STATE_DICT", {})
    monkeypatch.setattr(extract_r21d, "_STATE_DICTS_34", {})
    name32, name8 = "r2plus1d_34_32_ig65m_ft_kinetics", "r2plus1d_34_8_ig65m_ft_kinetics"
    with pytest.raises(FileNotFoundError) as e:
        extract_r21d.load_r21d_34_weights(name32)
    msg = str(e.value)
    assert "r2plus1d_34_clip32*kinetics*.pth" in msg and str(tmp_path / "none") in msg
    assert os.path.join(str(tmp_path / "th"), "hub", "checkpoints") in msg
    # the release names, as recalled, match loosely; the 8- and 32-frame files are told apart
    d = tmp_path / "th" / "hub" / "checkpoints"
    d.mkdir(parents=True)
    sd = {f"layer{L}.{b}.conv1.0.0.weight": torch.full((1,), float(L)) for L, n in zip(range(1, 5), (3, 4, 6, 3))
          for b in range(n)}
    torch.save(dict(sd, tag=torch.ones(1) * 32), str(d / "r2plus1d_34_clip32_ft_kinetics_from_ig65m-ade133f1.pth"))
    torch.save(dict(sd, tag=torch.ones(1) * 8), str(d / "r2plus1d_34_clip8_ft_kinetics_from_ig65m-0aa0550b.pth"))
    assert float(extract_r21d.load_r21d_34_weights(name32)["tag"]) == 32
    assert float(extract_r21d.load_r21d_34_weights(name8)["tag"]) == 8
    # $VF_CKPT_DIR comes first, and a DataParallel prefix is fine
    (tmp_path / "none").mkdir()
    torch.save({"module." + k: v for k, v in dict(sd, tag=torch.ones(1) * 7).items()},
               str(tmp_path / "none" / "r2plus1d_34_clip8_kinetics.pth"))
    monkeypatch.setattr(extract_r21d, "_STATE_DICTS_34", {})
    assert float(extract_r21d.load_r21d_34_weights(name8)["module.tag"]) == 7
    # the 18-layer cache is untouched, and an r2plus1d_18 state dict under a 34-layer name is refused
    assert extract_r21d._STATE_DICT == {}
    torch.save(r21d_net.stand_in_state_dict(), str(tmp_path / "none" / "r2plus1d_34_clip32_kinetics.pth"))
    monkeypatch.setattr(extract_r21d, "_STATE_DICTS_34", {})
    with pytest.raises(ValueError, match=r"\(2, 2, 2, 2\) blocks in layer1..4, not R\(2\+1\)D-34's \(3, 4, 6, 3\)"):
        extract_r21d.load_r21d_34_weights(name32)

"""--show_pred without a GPU: the printer against the reference printer's own text (tests/golden/show_pred.npz), the
class-name lists against the reference's label maps, the oracle's logits paths against the reference modules, and the
CLI / extractor wiring."""
import contextlib
import io
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
VIDEO = os.path.join(ROOT, "tests", "golden", "v_GGSY1Qvo990.mp4")


@pytest.fixture(scope="module")
def golden():
    return np.load(os.path.join(ROOT, "tests", "golden", "show_pred.npz"))


def _printed(fn, *a, **kw):
    buf = io.StringIO()
    with contextlib.redirect_stdout(buf):
        fn(*a, **kw)
    return buf.getvalue()


def test_printer_matches_reference_text_on_kinetics(golden):
    from video_features_b200.utils import show_predictions_on_dataset
    text = _printed(show_predictions_on_dataset, torch.from_numpy(golden["kinetics_logits"]), "kinetics")
    assert text == str(golden["kinetics_text"])
    assert text.count("\n\n") == golden["kinetics_logits"].shape[0]


def test_printer_matches_reference_text_on_imagenet_with_its_lines(golden):
    """The package prints torchvision's (shorter) ImageNet names; with the reference's label lines the text is the
    reference's, byte for byte."""
    from video_features_b200.utils import show_predictions_on_dataset
    lines = [str(x) for x in golden["imagenet_labels"]]
    logits = torch.from_numpy(golden["imagenet_logits"])
    assert _printed(show_predictions_on_dataset, logits, "imagenet", classes=lines) == str(golden["imagenet_text"])
    ours = _printed(show_predictions_on_dataset, logits, "imagenet").splitlines()
    ref = str(golden["imagenet_text"]).splitlines()
    assert len(ours) == len(ref)
    for a, b in zip(ours, ref):                     # same logit and probability columns, name = first name of the line
        assert a.split(" ")[:2] == b.split(" ")[:2]


def test_printer_on_top_k_rows(golden):
    """print_top_predictions (the extractors' path) prints the same text from (idx, logit, prob) rows."""
    import torch.nn.functional as F
    from video_features_b200.utils import print_top_predictions
    lg = torch.from_numpy(golden["kinetics_logits"])
    p = F.softmax(lg, dim=-1)
    idx = torch.sort(p, dim=-1, descending=True, stable=True)[1][:, :5].to(torch.int32)
    text = _printed(print_top_predictions, idx, lg.gather(1, idx.long()), p.gather(1, idx.long()), "kinetics")
    assert text == str(golden["kinetics_text"])


def test_class_names_against_reference_label_maps(golden):
    from video_features_b200.utils import class_names
    assert class_names("kinetics") == [str(x) for x in golden["kinetics_labels"]]
    names, lines = class_names("imagenet"), [str(x) for x in golden["imagenet_labels"]]
    assert len(names) == len(lines) == 1000
    differ = {i: (a, b) for i, (a, b) in enumerate(zip(names, lines)) if a != b.split(", ")[0]}
    assert differ == {134: ("crane bird", "crane"), 639: ("maillot tank suit", "maillot, tank suit")}
    with pytest.raises(NotImplementedError):
        class_names("ucf101")


@pytest.mark.parametrize("mod,T", [("rgb", 16), ("flow", 16), ("rgb", 64), ("flow", 64)])
def test_i3d_oracle_logits_equal_reference_module(golden, mod, T):
    from oracle import class_heads
    from oracle.stand_in import state_dict
    cin = 3 if mod == "rgb" else 2
    x = torch.rand(1, cin, T, 224, 224, generator=torch.Generator().manual_seed(200 + T)) * 2 - 1
    sm, lg = class_heads.i3d_forward_logits(state_dict(f"i3d_{mod}.pt"), x)
    ref_lg, ref_sm = torch.from_numpy(golden[f"{mod}_T{T}_logits"]), torch.from_numpy(golden[f"{mod}_T{T}_softmax"])
    assert float((lg - ref_lg).norm() / ref_lg.norm()) < 1e-5
    assert float((sm - ref_sm).norm() / ref_sm.norm()) < 1e-5


def test_fc_oracle_logits_equal_torchvision():
    import torchvision
    from oracle import class_heads, r21d_net, resnet_net
    sd = resnet_net.stand_in_state_dict(18)
    net = torchvision.models.resnet18(weights=None).eval()
    net.load_state_dict(sd)
    x = resnet_net.calibration_images(0, 2)
    with torch.no_grad():
        ref = net(x)
    msd = {"module." + k: v for k, v in sd.items()}          # the prefix the trunk loaders accept
    assert float((class_heads.resnet_logits(msd, x, 18) - ref).norm() / ref.norm()) < 1e-5
    sdv = r21d_net.stand_in_state_dict()
    netv = torchvision.models.video.r2plus1d_18(weights=None).eval()
    netv.load_state_dict(sdv)
    xv = r21d_net.calibration_clips(0, 1, 8)
    with torch.no_grad():
        refv = netv(xv)
    assert float((class_heads.r21d_logits(sdv, xv) - refv).norm() / refv.norm()) < 1e-5


def test_cli_help_no_longer_says_not_built():
    r = subprocess.run([sys.executable, os.path.join(ROOT, "main.py"), "--help"], capture_output=True, text=True,
                       cwd=ROOT, timeout=120)
    assert r.returncode == 0
    assert "--show_pred" in r.stdout and "not built" not in r.stdout


def test_extractors_construct_with_show_pred(tmp_path):
    import main
    from video_features_b200.extract.extract_i3d import ExtractI3D
    from video_features_b200.extract.extract_r21d import ExtractR21D
    from video_features_b200.extract.extract_resnet import ExtractResNet
    common = ["--video_paths", VIDEO, "--output_path", str(tmp_path / "out"), "--tmp_path", str(tmp_path / "tmp"),
              "--show_pred"]
    for ft, cls in (("resnet50", ExtractResNet), ("r21d_rgb", ExtractR21D), ("i3d", ExtractI3D)):
        ex = main.build_extractor(main.make_parser().parse_args(["--feature_type", ft] + common))
        assert isinstance(ex, cls) and ex.show_pred is True


def test_missing_head_is_named_only_when_asked():
    """A checkpoint without fc.* loads the trunk as before; the head lookup names the missing key."""
    from video_features_b200.class_head import FC_KEYS, ClassHead
    with pytest.raises(KeyError, match="fc.weight"):
        ClassHead.from_state_dict({"conv1.weight": torch.zeros(1)}, FC_KEYS, 0, "resnet50 checkpoint")

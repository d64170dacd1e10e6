"""CLIP ViT-L/14 towers without a GPU: configuration inference and its refusals, the float64 reference against HF's
implementation at 224 and 336 px, the synthetic weights' layout, checkpoint lookup, the CLI, the emulation script."""
import argparse
import os
import subprocess
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import clip_vitl_ref  # noqa: E402
from video_features_b200 import synthetic_weights  # noqa: E402

TYPES = {"CLIP-ViT-L/14": ("ViT-L-14.pt", 224), "CLIP-ViT-L/14@336px": ("ViT-L-14-336px.pt", 336)}


@pytest.fixture(scope="module", params=[224, 336])
def sd(request):
    return synthetic_weights.clip_vit_l14_state_dict(0, n_px=request.param)


def test_synthetic_state_dict_has_openai_l14_keys_and_shapes(sd):
    n_px = sd["visual.positional_embedding"].shape[0] == 577 and 336 or 224
    T = (n_px // 14) ** 2 + 1
    expect = {"visual.class_embedding": (1024,), "visual.positional_embedding": (T, 1024), "visual.proj": (1024, 768),
              "visual.conv1.weight": (1024, 3, 14, 14), "visual.ln_pre.weight": (1024,), "visual.ln_pre.bias": (1024,),
              "visual.ln_post.weight": (1024,), "visual.ln_post.bias": (1024,)}
    for i in range(24):
        p = f"visual.transformer.resblocks.{i}."
        expect.update({p + "attn.in_proj_weight": (3072, 1024), p + "attn.in_proj_bias": (3072,),
                       p + "attn.out_proj.weight": (1024, 1024), p + "attn.out_proj.bias": (1024,),
                       p + "ln_1.weight": (1024,), p + "ln_1.bias": (1024,), p + "ln_2.weight": (1024,),
                       p + "ln_2.bias": (1024,), p + "mlp.c_fc.weight": (4096, 1024), p + "mlp.c_fc.bias": (4096,),
                       p + "mlp.c_proj.weight": (1024, 4096), p + "mlp.c_proj.bias": (1024,)})
    assert {k: tuple(v.shape) for k, v in sd.items()} == expect
    assert all(v.dtype == torch.float32 for v in sd.values())


def test_outlier_variant_plants_large_channels():
    plain = synthetic_weights.clip_vit_l14_state_dict(1)
    loud = synthetic_weights.clip_vit_l14_state_dict(1, outliers=True)
    assert plain["visual.ln_pre.bias"].abs().max() < 1 and loud["visual.ln_pre.bias"].abs().max() >= 60


def test_config_inference_for_both_towers(sd):
    cfg = clip_vitl_ref.config(sd)
    n_px = cfg["n_px"]
    assert n_px in (224, 336)
    assert cfg == dict(width=1024, patch=14, layers=24, heads=16, n_px=n_px, tokens=(n_px // 14) ** 2 + 1, embed=768)


def _create_message(numels):
    """vf_clip_vitl_create's inference and refusals run on the sizes alone, before any tensor is read or a device is
    touched: every name points at one placeholder float.  Returns the error text."""
    import ctypes as C

    import numpy as np
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
        check(lib().vf_clip_vitl_create(C.byref(h), arr, len(numels), 0, 1))
    return str(e.value)


@pytest.mark.parametrize("change, key", [
    ("width", "visual.class_embedding"),
    ("resblock", "visual.transformer.resblocks.7.attn.in_proj_weight"),
    ("grid", "visual.positional_embedding"),
    ("patch", "visual.conv1.weight"),
    ("embed", "visual.proj"),
])
def test_refusals_name_the_key(change, key):
    sd = {k: v.numel() for k, v in synthetic_weights.clip_vit_l14_state_dict(0).items()}
    if change == "width":
        sd["visual.class_embedding"] = 768
        sd["visual.conv1.weight"] = 768 * 3 * 14 * 14
    elif change == "resblock":
        for k in [k for k in sd if k.startswith("visual.transformer.resblocks.7.")]:
            del sd[k]
    elif change == "grid":
        sd["visual.positional_embedding"] = (16 * 15 + 1) * 1024
    elif change == "patch":
        sd["visual.conv1.weight"] = 1024 * 3 * 16 * 16
    else:
        sd["visual.proj"] = 1024 * 512
    msg = _create_message(sd)
    assert key in msg, msg


def test_ref_matches_hf_float64(sd):
    """The reference (fp64, no rounding) against HF CLIPVisionModelWithProjection at the same configuration."""
    tr = pytest.importorskip("transformers")
    cfg = clip_vitl_ref.config(sd)
    sd64 = {k: v.double() for k, v in sd.items()}
    hf = tr.CLIPVisionModelWithProjection(clip_vitl_ref.hf_config(sd)).eval().double()
    res = hf.load_state_dict(clip_vitl_ref.to_hf_state_dict(sd64), strict=False)
    assert not res.missing_keys
    x = torch.randn(1, 3, cfg["n_px"], cfg["n_px"], generator=torch.Generator().manual_seed(2), dtype=torch.float64)
    with torch.no_grad():
        y_hf = hf(pixel_values=x).image_embeds
    y = clip_vitl_ref.encode_image(sd64, x, dtype=torch.float64)
    assert y.shape == (1, 768)
    assert float((y - y_hf).norm() / y_hf.norm()) < 1e-6


def test_streamed_p_schedule_differs_from_softmax_by_fp16_p_only():
    g = torch.Generator().manual_seed(4)
    qkv = torch.randn(2, 200, 3 * 128, generator=g, dtype=torch.float64) * 3
    a = clip_vitl_ref.attention_core(qkv, 2, rounding={"p"}, key_block=64)
    b = clip_vitl_ref.attention_core(qkv, 2, rounding=frozenset())
    assert float((a - b).abs().max()) < 2e-3          # fp16 P only
    assert not torch.equal(a, clip_vitl_ref.attention_core(qkv, 2, rounding={"p"}, key_block=None))


@pytest.mark.parametrize("ftype", list(TYPES))
def test_not_found_error_names_the_checkpoint(ftype, monkeypatch, tmp_path):
    from video_features_b200.extract import extract_clip
    monkeypatch.delenv("VF_CLIP_CKPT", raising=False)
    monkeypatch.delenv("VF_CLIP_SYNTHETIC", raising=False)
    monkeypatch.setenv("HOME", str(tmp_path))
    with pytest.raises(FileNotFoundError) as e:
        extract_clip.load_clip_state_dict(ftype)
    assert TYPES[ftype][0] in str(e.value) and os.path.join(str(tmp_path), ".cache/clip") in str(e.value)


@pytest.mark.parametrize("ftype", list(TYPES))
def test_synthetic_env_selects_l14_weights(ftype, monkeypatch):
    from video_features_b200.extract import extract_clip
    monkeypatch.setenv("VF_CLIP_SYNTHETIC", "2:outliers")
    sd = extract_clip.load_clip_state_dict(ftype)
    assert clip_vitl_ref.config(sd)["n_px"] == TYPES[ftype][1]
    ref = synthetic_weights.clip_vit_l14_state_dict(2, True, n_px=TYPES[ftype][1])
    assert torch.equal(sd["visual.ln_pre.bias"], ref["visual.ln_pre.bias"])


def test_cli_supports_both_types():
    import main
    for t in TYPES:
        assert t in main.SUPPORTED
        args = main.make_parser().parse_args(["--feature_type", t, "--video_paths", "x.mp4"])
        assert args.feature_type == t


def test_extractor_routes_both_types_to_the_vitl_engine(monkeypatch):
    from video_features_b200.extract import extract_clip
    made = []
    monkeypatch.setattr(extract_clip, "ClipViTLEngine", lambda sd, device: made.append(clip_vitl_ref.config(sd)) or "e")
    monkeypatch.setenv("VF_CLIP_SYNTHETIC", "0")
    for t, (_, n_px) in TYPES.items():
        a = argparse.Namespace(feature_type=t, extraction_fps=None, extract_method="uni_12", on_extraction="print",
                               video_paths=[os.path.join(ROOT, "tests", "golden", "v_GGSY1Qvo990.mp4")],
                               file_with_video_paths=None, video_dir=None, output_path="out", output_direct=False)
        ex = extract_clip.ExtractCLIP(a, external_call=True)
        assert ex._engine(torch.device("cuda", 0)) == "e"
        assert made[-1]["n_px"] == n_px


def test_emulation_script_runs_tiny():
    r = subprocess.run([sys.executable, os.path.join(ROOT, "scripts", "precision", "emulate_clip_vitl.py"), "--tiny"],
                       capture_output=True, text=True, cwd=ROOT, timeout=600)
    assert r.returncode == 0, r.stderr
    assert "plain" in r.stdout and "outliers" in r.stdout

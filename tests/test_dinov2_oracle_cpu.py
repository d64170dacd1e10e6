"""oracle/dinov2_net.py against HF's independent DINOv2 implementations (``Dinov2Model`` for the plain hub models,
``Dinov2WithRegistersModel`` for the _reg ones), its 224-px positional table against HF's interpolation, and its
transform against torchvision's preset on PIL images."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import dinov2_net as D

pytest.importorskip("transformers")

# (model, blocks): S and B at full depth, L and g at full width with 2 blocks (g covers SwiGLU)
CASES = [(n + r, depth) for n, depth in (("dinov2_vits14", None), ("dinov2_vitb14", None), ("dinov2_vitl14", 2),
                                         ("dinov2_vitg14", 2)) for r in ("", "_reg")]


@pytest.mark.parametrize("name,depth", CASES)
def test_fp32_oracle_matches_hf(name, depth):
    sd = D.stand_in_state_dict(name, depth=depth)
    x = D.calibration_frames(4, 3)
    hf = D.hf_model(sd)
    with torch.no_grad():
        want = hf(pixel_values=x).pooler_output
        got = D.forward(D.prepare(sd, torch.float32), x)
        got64 = D.forward(D.prepare(sd), x.double())
    rel = ((got.double() - want.double()).norm(dim=1) / want.double().norm(dim=1)).max().item()
    assert rel < 2e-6, rel
    rel64 = ((got64 - want.double()).norm(dim=1) / got64.norm(dim=1)).max().item()
    assert rel64 < 2e-6, rel64


def test_reg_table_is_hfs_interpolation():
    from transformers import Dinov2WithRegistersConfig
    from transformers.models.dinov2_with_registers.modeling_dinov2_with_registers import Dinov2WithRegistersEmbeddings
    sd = D.stand_in_state_dict("dinov2_vitb14_reg", depth=1)
    cfg = Dinov2WithRegistersConfig(hidden_size=768, image_size=518, patch_size=14, num_register_tokens=4)
    emb = Dinov2WithRegistersEmbeddings(cfg)
    emb.position_embeddings.data.copy_(sd["pos_embed"])
    with torch.no_grad():
        want = emb.interpolate_pos_encoding(torch.zeros(1, 257, 768), 224, 224)[0]
    assert torch.equal(D.pos_table_224(sd["pos_embed"], True), want)


@pytest.mark.parametrize("name", ["dinov2_vits14", "dinov2_vitg14_reg"])
def test_engine_wrapper_table_equals_the_oracle(name):
    from video_features_b200.dinov2_engine import pos_table_224, state_dict_with_table
    sd = D.stand_in_state_dict(name, depth=1)
    reg = name.endswith("_reg")
    assert torch.equal(pos_table_224(sd["pos_embed"], reg), D.pos_table_224(sd["pos_embed"], reg))
    assert torch.equal(state_dict_with_table(sd)["pos_embed_224"], D.pos_table_224(sd["pos_embed"], reg))


def test_plain_table_needs_the_offset():
    """The plain hub models scale by (16 + 0.1) / 37; asking for size (16, 16) (HF's Dinov2Model) gives another table."""
    pe = D.stand_in_state_dict("dinov2_vits14", depth=1)["pos_embed"]
    ours = D.pos_table_224(pe, False)
    grid = pe[:, 1:].reshape(1, 37, 37, -1).permute(0, 3, 1, 2)
    sized = F.interpolate(grid, size=(16, 16), mode="bicubic", align_corners=False)
    sized = torch.cat([pe[0, :1], sized.permute(0, 2, 3, 1).reshape(256, -1)])
    assert torch.equal(ours[0], sized[0])
    diff = ((ours[1:] - sized[1:]).norm() / sized[1:].norm()).item()
    assert diff > 1e-2, diff


@pytest.mark.parametrize("h,w", [(240, 320), (256, 256), (480, 360), (200, 300), (720, 1280)])
def test_transform_equals_the_torchvision_preset(h, w):
    g = np.random.default_rng(h * w)
    rgb = g.integers(0, 256, (h, w, 3), dtype=np.uint8)
    got, want = D.transform(rgb), D.transform_torchvision(rgb)
    assert got.shape == (3, 224, 224)
    assert torch.equal(got, want)


def test_shape_inference_and_flops():
    for name in D.MODELS:
        d, depth, ffn, reg = D.shape_of(name)
        sd = D.stand_in_state_dict(name, depth=1)
        assert D.config(sd) == (d, 1, d // 64, ffn, reg)
        assert sd["pos_embed"].shape == (1, 1 + 37 * 37, d)
    gf = [D.flops(n)["gemm"] / 1e9 for n in ("dinov2_vits14", "dinov2_vitb14", "dinov2_vitl14", "dinov2_vitg14")]
    assert [round(v) for v in gf] == [11, 44, 156, 583], gf

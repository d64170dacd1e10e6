"""The DINOv2 engine against the float64 oracle (oracle/dinov2_net.py) for all eight stand-ins: the features against
the exact forward (tests/dinov2_bars.py FEATURES, under the project's 1e-3); the embedding, every 4th block and the head
through the debug taps against the oracle of the declared rounding; every 4th block alone on the oracle's own stream;
a lost lo half at the embedding and in the blocks; the u8 entry against the f32 entry,
graph replay against eager, chunked calls; the SwiGLU kernel and the attention at 261 tokens against float64."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from dinov2_bars import BARS, BLOCK_SEPARATION, FEATURES, PROJECT, SEPARATION
from oracle import dinov2_net as D

pytestmark = pytest.mark.gpu

ATTN_BAR = (2e-3, 4e-3)
SWIGLU_BAR = 4.9e-4           # one fp16 rounding (2^-11) of values computed in fp32


def _errors(y, ref):
    """(worst per-frame rel-L2, worst per-frame max-abs / max) over the leading dimension."""
    y, ref = y.double().flatten(1), ref.double().flatten(1)
    rel = ((y - ref).norm(dim=1) / ref.norm(dim=1)).max().item()
    mx = ((y - ref).abs().amax(dim=1) / ref.abs().amax(dim=1)).max().item()
    return rel, mx


def _under(e, bar):
    return e[0] <= bar[0] and e[1] <= bar[1]


def _block_updates(eng, taps):
    """Worst (rel-L2, max-abs / max) of the residual update of every 4th block but the last (which updates the class
    rows only), each run alone by the engine on the oracle's own stream, against the oracle's update."""
    worst = (0.0, 0.0)
    for i in range(0, eng.depth - 1, 4):
        xin = taps["embed"] if i == 0 else taps[f"block{i - 1}"]
        got = eng.debug_blocks(xin.float(), i, i + 1).double() - xin
        e = _errors(got, taps[f"block{i}"] - xin)
        worst = max(worst[0], e[0]), max(worst[1], e[1])
    return worst


@pytest.fixture(scope="module", params=list(D.MODELS))
def model(request):
    from video_features_b200.dinov2_engine import DINOv2Engine
    name = request.param
    sd = D.stand_in_state_dict(name)
    eng = DINOv2Engine(sd, 0, max_frames=4)
    sd64 = D.prepare(sd, torch.float64, "cuda")
    yield name, sd, sd64, eng
    eng.close()
    torch.cuda.empty_cache()


def test_engine_vs_float64(cuda_device, model):
    name, sd, sd64, eng = model
    d, depth, ffn, reg = D.shape_of(name)
    assert (eng.out_dim, eng.depth, eng.heads, eng.tokens, eng.registers, eng.ffn) == \
        (d, depth, d // 64, 257 + (4 if reg else 0), 4 if reg else 0, ffn)
    x = D.calibration_frames(1, 3).cuda()
    y = eng.encode_f32(x)
    assert tuple(y.shape) == (3, d)
    with torch.no_grad():
        declared = D.forward_engine(sd64, x.double())
        exact = D.forward(sd64, x.double())
    e_decl, e_exact = _errors(y, declared), _errors(y, exact)
    print(f"\n{name}: vs declared {e_decl[0]:.2e}/{e_decl[1]:.2e}, vs exact {e_exact[0]:.2e}/{e_exact[1]:.2e}")
    assert _under(e_exact, FEATURES[d]) and _under(e_exact, PROJECT), e_exact


def test_taps_vs_declared_rounding(cuda_device, model):
    """The embedding, the stream after every 4th block (the engine's own chain) and the head against the float64 oracle
    of the declared rounding."""
    name, sd, sd64, eng = model
    x = D.calibration_frames(2, 2).cuda()
    taps = {}
    with torch.no_grad():
        ref = D.forward_engine(sd64, x.double(), taps)
    depth = eng.depth
    got = eng.debug_embed_f32(x)
    worst = {"embed": _errors(got, taps["embed"])}
    worst["blocks"] = (0.0, 0.0)
    for l0 in range(0, depth, 4):
        l1 = min(l0 + 4, depth)
        got = eng.debug_blocks(got, l0, l1)
        e = _errors(got, taps[f"block{l1 - 1}"])
        worst["blocks"] = max(worst["blocks"][0], e[0]), max(worst["blocks"][1], e[1])
    # the head alone on the oracle's stream: only its own arithmetic
    head = eng.debug_head(taps[f"block{depth - 1}"].float())
    worst["head"] = _errors(head, ref)
    worst["block"] = _block_updates(eng, taps)
    print(f"\n{name}: " + ", ".join(f"{k} {r:.2e}/{m:.2e}" for k, (r, m) in worst.items()))
    assert _under(worst["embed"], BARS["embed"]), worst["embed"]
    assert _under(worst["blocks"], BARS["blocks"]), worst["blocks"]
    assert _under(worst["head"], BARS["head"]), worst["head"]
    assert _under(worst["block"], BARS["block"]), worst["block"]


@pytest.mark.parametrize("name", ["dinov2_vits14", "dinov2_vitg14_reg"])
def test_lost_lo_half_fails_the_bar(cuda_device, name):
    """The engine with every weight pre-rounded to fp16 (so W_lo is zero) misses the embedding bar by SEPARATION and the
    one-block bar by BLOCK_SEPARATION (rel-L2); its features are printed against the exact forward (fp16 weights cost
    about as much as every fp16 activation together, DESIGN.md §4.17)."""
    from video_features_b200.dinov2_engine import DINOv2Engine
    sd = D.stand_in_state_dict(name)
    w16 = {k: (v.half().float() if k.endswith(".weight") and v.dim() >= 2 else v) for k, v in sd.items()}
    eng = DINOv2Engine(w16, 0, max_frames=4)
    x = D.calibration_frames(1, 3).cuda()
    y = eng.encode_f32(x)
    emb = eng.debug_embed_f32(x)
    sd64 = D.prepare(sd, torch.float64, "cuda")
    taps = {}
    with torch.no_grad():
        exact = D.forward(sd64, x.double())
        emb_ref = D.embed(sd64, x.double(), D.ENGINE_FP16)
        D.forward_engine(sd64, D.calibration_frames(2, 2).cuda().double(), taps)
    blk = _block_updates(eng, taps)
    eng.close()
    e, ee = _errors(y, exact), _errors(emb, emb_ref)
    print(f"\n{name} fp16 weights: embed {ee[0]:.2e}/{ee[1]:.2e}, one block {blk[0]:.2e}/{blk[1]:.2e}, features vs "
          f"exact {e[0]:.2e}/{e[1]:.2e}")
    bar = BARS["embed"]
    assert ee[0] >= SEPARATION * bar[0] and ee[1] >= SEPARATION * bar[1], ee
    assert blk[0] >= BLOCK_SEPARATION * BARS["block"][0], blk
    del sd64
    torch.cuda.empty_cache()


def _frames_u8(n, h, w, seed):
    g = torch.Generator().manual_seed(seed)
    low = torch.rand(n, 3, 6, 8, generator=g)
    img = F.interpolate(low, size=(h, w), mode="bilinear", align_corners=False) * 200 + 40 * torch.rand(n, 3, h, w, generator=g)
    return img.round().clamp(0, 255).to(torch.uint8).permute(0, 2, 3, 1).contiguous()


def test_u8_entry_equals_f32_entry_and_the_preset(cuda_device):
    """The fused transform: identical bits to the f32 entry fed by the oracle's PIL transform (Pillow-exact resize),
    on frame sizes that resize up, down and not at all."""
    from video_features_b200.dinov2_engine import DINOv2Engine
    eng = DINOv2Engine(D.stand_in_state_dict("dinov2_vits14_reg"), 0, max_frames=4)
    for (h, w) in [(240, 320), (256, 256), (480, 360), (200, 300)]:
        bgr = _frames_u8(3, h, w, h + w)
        y8 = eng.encode_u8(bgr.cuda())
        x = torch.stack([D.transform(f[:, :, [2, 1, 0]].numpy()) for f in bgr]).cuda()
        y32 = eng.encode_f32(x)
        torch.cuda.synchronize()
        assert torch.equal(y8, y32), (h, w, (y8 - y32).abs().max().item())
        e8 = eng.debug_embed_u8(bgr.cuda())
        e32 = eng.debug_embed_f32(x)
        assert torch.equal(e8, e32), (h, w)
    eng.close()


def test_graph_replay_and_chunks_equal_eager(cuda_device, monkeypatch):
    """A captured graph replays the eager bits; a call larger than max_frames equals its frames run chunk by chunk."""
    from video_features_b200.dinov2_engine import DINOv2Engine
    sd = D.stand_in_state_dict("dinov2_vitb14")
    x = D.calibration_frames(3, 7).cuda()
    eng = DINOv2Engine(sd, 0, max_frames=4)
    first = eng.encode_f32(x[:4])                     # captures the 4-frame graph and replays it
    second = eng.encode_f32(x[:4])                    # replays
    third = eng.encode_f32(x[:4])
    whole = eng.encode_f32(x)                         # 7 frames: chunks of 4 and 3
    parts = torch.cat([eng.encode_f32(x[:4]), eng.encode_f32(x[4:])])
    torch.cuda.synchronize()
    assert torch.equal(first, second) and torch.equal(first, third)
    assert torch.equal(whole, parts)
    eng.close()
    monkeypatch.setenv("VF_NO_GRAPH", "1")
    eng = DINOv2Engine(sd, 0, max_frames=4)
    eager = eng.encode_f32(x[:4])
    torch.cuda.synchronize()
    assert torch.equal(eager, first)
    eng.close()


@pytest.mark.parametrize("rows,hidden", [(261, 4096), (5, 64)])
def test_swiglu_kernel_vs_float64(cuda_device, rows, hidden):
    from video_features_b200.dinov2_engine import swiglu
    g = torch.Generator().manual_seed(rows)
    ab = (torch.randn(rows, 2 * hidden, generator=g) * 3).cuda()
    out = swiglu(ab)
    a, b = ab.double().chunk(2, dim=-1)
    ref = F.silu(a) * b
    err = ((out.double() - ref).abs() / ref.abs().clamp_min(1e-3)).max().item()
    assert err <= SWIGLU_BAR, err
    assert torch.isfinite(out).all()


@pytest.mark.parametrize("heads", [6, 24])
def test_attention_261_tokens_vs_float64(cuda_device, heads):
    from video_features_b200.dinov2_engine import attention
    g = torch.Generator().manual_seed(heads)
    n, S = 3, 261
    qkv = (torch.randn(n, S, 3 * heads * 64, generator=g) * 1.5).half().cuda()
    out = attention(qkv, heads)
    q, k, v = (t.double().view(n, S, heads, 64).transpose(1, 2) for t in qkv.split(heads * 64, dim=-1))
    ref = (torch.softmax(q @ k.transpose(-1, -2) / 8, dim=-1) @ v).transpose(1, 2).reshape(n, S, heads * 64)
    e = _errors(out.reshape(n * S, -1), ref.reshape(n * S, -1))
    assert _under(e, ATTN_BAR), e


def test_refusals_name_the_key(cuda_device):
    from video_features_b200._lib import VfError
    from video_features_b200.dinov2_engine import DINOv2Engine
    sd = dict(D.stand_in_state_dict("dinov2_vits14"))
    sd["blocks.0.attn.proj.weight"] = torch.zeros(384, 383)
    with pytest.raises(VfError, match="blocks.0.attn.proj.weight"):
        DINOv2Engine(sd, 0, max_frames=1)

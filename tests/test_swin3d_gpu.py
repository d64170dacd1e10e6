"""The Swin3D engine against the float64 oracle (oracle/swin3d_net.py) at every read_stage tap and at the features,
for the t / s / b stand-ins at T = 32 (no temporal padding), 17 (T' = 9 padded to 16 with a temporal shift) and 10
(T' = 5: a clamped window and no temporal shift), several clips per call; the u8 entry against the f32 entry, graph
replay against eager, the window-attention kernel alone against float64, and the GELU epilogue against erf GELU."""
import numpy as np
import pytest
import torch

import attention_ref as A
from oracle import swin3d_net as S
from swin3d_bars import BARS, SEPARATION

pytestmark = pytest.mark.gpu

ATTN_BAR = (2e-3, 4e-3)
GELU_BAR = 1e-6


def _errors(y, ref):
    """(worst per-clip rel-L2, worst per-clip max-abs / max) over the leading dimension."""
    y, ref = y.double().flatten(1), ref.double().flatten(1)
    rel = ((y - ref).norm(dim=1) / ref.norm(dim=1)).max().item()
    mx = ((y - ref).abs().amax(dim=1) / ref.abs().amax(dim=1)).max().item()
    return rel, mx


@pytest.fixture(scope="module", params=["swin3d_t", "swin3d_s", "swin3d_b"])
def model(request):
    from video_features_b200.swin3d_engine import Swin3DEngine
    name = request.param
    sd = S.stand_in_state_dict(name)
    eng = Swin3DEngine(sd, 0, max_clips=2, max_T=32)
    sd64 = {k: (v.double() if v.is_floating_point() else v).cuda() for k, v in sd.items()}
    yield name, sd, sd64, eng
    eng.close()


@pytest.mark.parametrize("T", [32, 17, 10])
def test_engine_vs_float64(cuda_device, model, T):
    name, sd, sd64, eng = model
    x = S.calibration_clips(1, 3, T).cuda()            # 3 clips: one call of 2 + 1 (the stages hold the last chunk)
    y = eng.forward_f32(x)
    dim = 8 * S.MODELS[name][0]
    assert tuple(y.shape) == (3, dim)
    with torch.no_grad():
        ref, taps = S.forward(sd64, x.double(), taps=True)
    worst = {}
    worst["features"] = _errors(y, ref)
    for i, st in enumerate(S.STAGES):
        got = eng.read_stage(i)
        want = taps[st][2:]                            # the last chunk: clip 2
        assert got.shape == want.shape, (st, got.shape, want.shape)
        worst[st] = _errors(got, want)
    print(f"\n{name} T={T}: " + ", ".join(f"{k} {r:.2e}/{m:.2e}" for k, (r, m) in worst.items()))
    for k, (r, m) in worst.items():
        assert r <= BARS[k][0] and m <= BARS[k][1], (k, r, m)


def test_u8_entry_equals_f32_entry(cuda_device):
    from video_features_b200.swin3d_engine import Swin3DEngine
    sd = S.stand_in_state_dict("swin3d_t")
    eng = Swin3DEngine(sd, 0, max_clips=2, max_T=17)
    g = torch.Generator().manual_seed(11)
    for hw in [(240, 320), (360, 270)]:
        bgr = torch.randint(0, 256, (24,) + hw + (3,), dtype=torch.uint8, generator=g)
        starts, T = [0, 5, 7], 17
        yu = eng.forward_u8(bgr.cuda(), starts, T)
        rgb = bgr.numpy()[..., ::-1].copy()
        x = torch.stack([S.transform(rgb[s:s + T]) for s in starts]).cuda()
        yf = eng.forward_f32(x)
        assert torch.equal(yu, yf), hw
    eng.close()


def test_graph_replay_equals_eager(cuda_device, monkeypatch):
    from video_features_b200.swin3d_engine import Swin3DEngine
    sd = S.stand_in_state_dict("swin3d_t")
    x = S.calibration_clips(2, 2, 17).cuda()
    eng = Swin3DEngine(sd, 0, max_clips=2, max_T=17)
    first, second, third = eng.forward_f32(x), eng.forward_f32(x), eng.forward_f32(x)    # captured, then replayed
    eng.close()
    monkeypatch.setenv("VF_NO_GRAPH", "1")
    eager_eng = Swin3DEngine(sd, 0, max_clips=2, max_T=17)
    eager = eager_eng.forward_f32(x)
    eager_eng.close()
    assert torch.equal(first, second) and torch.equal(second, third) and torch.equal(third, eager)


def attention_ref(qkv, bias, table, shifted):
    """float64 window attention from a qkv matrix (n, T', H, W, 3C): the oracle's windowing, padded positions taking the
    qkv bias as their q / k / v (a zero row after norm1), q scaled by 32^-0.5, bias, -100 mask, softmax."""
    return A.swin3d(qkv, bias, table, shifted, rounding=False, key_block=None)


# (C, T', H = W): every stage's (heads, spatial extent) at an unpadded, a padded and a clamped T'
ATTN_CASES = [(c, tq, s) for c, s in [(96, 56), (192, 28), (384, 14), (768, 7), (128, 56), (1024, 7)]
              for tq in (16, 9, 5)]


@pytest.mark.parametrize("shifted", [False, True])
@pytest.mark.parametrize("C,Tq,S_", ATTN_CASES)
def test_window_attention_vs_float64(cuda_device, C, Tq, S_, shifted):
    from video_features_b200.swin3d_engine import window_attention
    g = torch.Generator().manual_seed(C * 100 + Tq * 10 + S_ + shifted)
    n = 2 if S_ >= 28 else 3
    qkv = (torch.randn(n, Tq, S_, S_, 3 * C, generator=g) * 1.5).half()
    bias = torch.randn(3 * C, generator=g) * 0.5
    table = torch.randn(2535, C // 32, generator=g)
    y = window_attention(qkv.cuda(), bias.cuda(), table.cuda(), shifted)
    ref = attention_ref(qkv.cuda(), bias.half().float().cuda(), table.cuda(), shifted)
    rel, mx = _errors(y, ref)
    assert rel <= ATTN_BAR[0] and mx <= ATTN_BAR[1], (rel, mx)


def test_gelu_epilogue_vs_erf(cuda_device):
    from video_features_b200 import ops
    from video_features_b200._lib import VF_ACT_GELU
    g = torch.Generator().manual_seed(3)
    a = (torch.randn(1000, 384, generator=g) * 0.2).half()
    b = (torch.randn(1536, 384, generator=g) * 0.2).half()
    bias = torch.randn(1536, generator=g) * 0.5
    for out_f32 in (True, False):
        y = ops.gemm_f16(a.cuda(), b.cuda(), bias.cuda(), None, VF_ACT_GELU, out_f32).double().cpu()
        z = a.double() @ b.double().T + bias.double()
        ref = 0.5 * z * (1 + torch.erf(z / np.sqrt(2)))
        err = (y - ref).abs().max().item() / ref.abs().max().item()
        assert err <= (GELU_BAR if out_f32 else 1e-3), (out_f32, err)
        assert (y - ref).abs().max().item() <= (1e-5 if out_f32 else 2e-2)


def test_refuses_other_shapes(cuda_device):
    from video_features_b200._lib import VfError
    from video_features_b200.swin3d_engine import Swin3DEngine
    sd = S.stand_in_state_dict("swin3d_t")
    bad = {k: v for k, v in sd.items() if not k.startswith("features.4.5.")}
    with pytest.raises(VfError, match="features.4"):
        Swin3DEngine(bad, 0, max_clips=1, max_T=8)
    bad = dict(sd)
    bad["features.0.0.attn.relative_position_bias_table"] = torch.zeros(100, 3)
    with pytest.raises(VfError, match="relative_position_bias_table"):
        Swin3DEngine(bad, 0, max_clips=1, max_T=8)
    prefixed = {"module." + k: v for k, v in sd.items()}
    eng = Swin3DEngine(prefixed, 0, max_clips=1, max_T=8)
    assert eng.out_dim == 768 and eng.depths == (2, 2, 6, 2)
    eng.close()


@pytest.mark.parametrize("name", ["swin3d_t", "swin3d_b"])
def test_lost_lo_half_fails_the_bar(cuda_device, name):
    """Control: every GEMM weight rounded to one fp16 value (its lo half zero, as a lost W_lo half or pass would leave
    it) puts the features over the bar by SEPARATION."""
    from video_features_b200.swin3d_engine import Swin3DEngine
    sd = S.stand_in_state_dict(name)
    gemm_w = [k for k in sd if k.endswith("weight") and sd[k].dim() >= 2 and "bias_table" not in k and k != "head.weight"]
    assert len(gemm_w) == 1 + sum(4 * d for d in S.MODELS[name][1]) + 3     # patch embed, blocks, reductions
    hi = {k: (v.half().float() if k in gemm_w else v) for k, v in sd.items()}
    eng = Swin3DEngine(hi, 0, max_clips=2, max_T=10)
    x = S.calibration_clips(1, 2, 10).cuda()
    y = eng.forward_f32(x)
    eng.close()
    with torch.no_grad():
        ref = S.forward({k: (v.double() if v.is_floating_point() else v).cuda() for k, v in sd.items()}, x.double())
    rel, mx = _errors(y, ref)
    print(f"\n{name} fp16 weights: features {rel:.2e} / {mx:.2e}")
    assert rel >= SEPARATION * BARS["features"][0] and mx >= SEPARATION * BARS["features"][1], (rel, mx)

"""The DINOv2, Swin3D, MViT and CLIP text attention kernels on hard inputs against the float64 references of their
declared rounding (tests/attention_ref.py): scores in the tens to hundreds, one dominant key per row placed where the
online softmax has to rescale late (either side of a key-block boundary, the last block, the last shared-memory chunk,
a register token, the padded positions of a window), the Swin3D shift mask and bias table competing with the scores,
MViT's rel-pos terms in the tens, and rows made identical on purpose.  Every case first asserts that its inputs are
hard; each prints its error against its bar.  Also the DINOv2 SwiGLU kernel on inputs where expf(-a) overflows.

Each error is (worst rel-L2, worst max-abs / max) over the leading dimension (frames, clips, prompts)."""
import pytest
import torch
import torch.nn.functional as F

import attention_ref as A
import clip_text_bars
import dinov2_bars
import mvit_bars
import swin3d_bars
from test_dinov2_gpu import SWIGLU_BAR

pytestmark = pytest.mark.gpu


def _errors(y, ref):
    y, ref = y.double().flatten(1), ref.double().flatten(1)
    rel = ((y - ref).norm(dim=1) / ref.norm(dim=1)).max().item()
    mx = ((y - ref).abs().amax(dim=1) / ref.abs().amax(dim=1)).max().item()
    return rel, mx


def _check(name, got, want, bar):
    assert torch.isfinite(got.float()).all(), name
    e = _errors(got, want)
    print(f"\n{name}: {e[0]:.2e} / {e[1]:.2e}  (bar {bar[0]:.1e} / {bar[1]:.1e})")
    assert e[0] <= bar[0] and e[1] <= bar[1], (name, e)


# --------------------------------------------------------------------------------------------------------- DINOv2

@pytest.mark.parametrize("heads", [6, 12, 16, 24])
@pytest.mark.parametrize("S", [257, 261])
def test_dinov2_attention(cuda_device, S, heads):
    """257 tokens (no registers: the last key alone in its 64-key block) and 261 (4 registers), every released head
    count; random frames and hard ones, and a frame of identical rows whose outputs must be bit-equal."""
    from video_features_b200.dinov2_engine import attention
    qkv, keys = A.dinov2_hard(S, heads, 1000 * heads + S)
    g = torch.Generator().manual_seed(S + heads)
    rnd = (torch.randn(3, S, 3 * heads * 64, generator=g) * 1.5).half().cuda()
    qkv = qkv.cuda()
    s = A.dinov2_scores(qkv[:-1], heads)
    for f, key in enumerate(keys):
        dominant = torch.zeros(S, dtype=torch.bool, device=s.device)
        dominant[key] = True
        hit, med = A.hardness(s[f], dominant)
        assert hit >= 0.1 and med > 15.0, (key, hit, med)
    assert s.amax().item() > 200.0
    got = attention(qkv, heads)
    _check(f"dinov2 S={S} heads={heads} random", attention(rnd, heads), A.dinov2(rnd, heads),
           dinov2_bars.BARS["attention"])
    _check(f"dinov2 S={S} heads={heads} hard (keys {keys}, identical rows)", got, A.dinov2(qkv, heads),
           dinov2_bars.BARS["attention hard"])
    assert torch.equal(got[-1], got[-1, :1].expand(S, -1)), "identical rows give identical outputs"


# --------------------------------------------------------------------------------------------------------- Swin3D

# (C, T', H = W): every stage's (heads, spatial extent) at an unpadded, a padded and a clamped T'
SWIN_CASES = [(c, tq, s) for c, s in [(96, 56), (192, 28), (384, 14), (768, 7), (128, 56), (1024, 7)]
              for tq in (16, 9, 5)]


@pytest.mark.parametrize("shifted", [False, True])
@pytest.mark.parametrize("C,Tq,S_", SWIN_CASES)
def test_swin3d_window_attention(cuda_device, C, Tq, S_, shifted):
    from video_features_b200.swin3d_engine import window_attention
    n = 2 if S_ >= 28 else 3
    qkv, bias, table = A.swin3d_hard(n, C, Tq, S_, shifted, C * 100 + Tq * 10 + S_ + shifted)
    qkv, bias, table = qkv.cuda(), bias.cuda(), table.cuda()
    hit, med, cross = A.swin3d_stats(qkv, bias, table, shifted)
    assert hit >= 0.1 and med > 15.0, (hit, med)
    if A.SwinWindows((Tq, S_, S_), shifted).region is not None:
        assert cross > 100.0, cross
    y = window_attention(qkv, bias, table, shifted)
    _check(f"swin3d C={C} T'={Tq} {S_}x{S_} shifted={shifted} (hit {hit:.2f}, cross-region max {cross:.0f})", y,
           A.swin3d(qkv, bias, table, shifted), swin3d_bars.BARS["attention hard"])


# ----------------------------------------------------------------------------------------------------------- MViT

# every block geometry of both variants: (q extent, kv extent, heads); 1569 keys take four 416-key chunks
MVIT_CASES = [(56, 7, 1), (28, 14, 2), (28, 7, 2), (14, 14, 4), (14, 7, 4), (7, 14, 8), (7, 7, 8)]


@pytest.mark.parametrize("v2", [False, True])
@pytest.mark.parametrize("S,K,heads", MVIT_CASES)
def test_mvit_pool_attention(cuda_device, S, K, heads, v2):
    from video_features_b200.mvit_engine import pool_attention
    q, k, v, rel = A.mvit_hard(S, K, heads, v2, S * 10 + K * 1000 + heads + 100 * v2, "cuda")
    nk = k.shape[1]
    hit, med, last_block, last_chunk = A.mvit_stats(q, k, S, K, heads, rel)
    assert hit >= 0.1 and med > 15.0 and last_block > 0.0, (hit, med, last_block)
    if nk > A.MV_MAX_KEYS:
        assert last_chunk > 0.0, last_chunk
    if v2:
        rb = A.mvit_add(A.mvit_heads(q, heads), (8, S, S), (8, K, K), tuple(r.double() for r in rel), nk)
        assert rb.abs().amax().item() > 20.0
    y = pool_attention(q, k, v, (8, S, S), (8, K, K), rel, resid=v2)
    want = A.mvit(A.mvit_heads(q, heads), A.mvit_heads(k, heads), A.mvit_heads(v, heads), (8, S, S), (8, K, K),
                  tuple(r.double() for r in rel) if rel else None, resid=v2)
    want = want.transpose(1, 2).reshape(y.shape)
    _check(f"mvit q {S} kv {K} ({nk} keys) heads {heads} v2 {v2} (hit {hit:.2f}, max in the last block "
           f"{last_block:.3f}, last chunk {last_chunk:.3f})", y, want, mvit_bars.BARS["attention hard"])


# ------------------------------------------------------------------------------------------------------ CLIP text

@pytest.mark.parametrize("heads", [8, 10, 12])
def test_clip_text_attention(cuda_device, heads):
    """Key 0 a sink at scores in the hundreds, or each row's last key dominant; every prompt length S gives the rows
    of the full 77-row call bit for bit."""
    from video_features_b200.clip_text_engine import attention
    qkv = A.clip_text_hard(16, heads, heads)
    (hit0, med0), (hitl, medl), top = A.clip_text_stats(qkv.cuda(), heads)
    assert hit0 >= 0.1 and med0 > 15.0 and hitl >= 0.1 and medl > 15.0 and top > 200.0, (hit0, med0, hitl, medl, top)
    full = attention(qkv.cuda(), heads)
    for S in (1, 2, 33, 64, 65, 77):
        part = qkv[:, :S].contiguous().cuda()
        out = attention(part, heads)
        _check(f"clip text heads={heads} S={S}", out, A.clip_text(part, heads), clip_text_bars.ATTENTION_HARD)
        assert torch.equal(out, full[:, :S]), S              # row i's bits do not depend on the rows after it


# --------------------------------------------------------------------------------------------------------- SwiGLU

@pytest.mark.parametrize("rows", [257, 261])
def test_swiglu_where_exp_overflows(cuda_device, rows):
    """a spread over [-120, 120] (expf(-a) overflows below -88.7), b up to +-50: finite everywhere, exactly +-0 for
    a <= -100, a b within one fp16 rounding for a >= 20 (silu(a) = a to fp32 precision), SWIGLU_BAR elsewhere."""
    from video_features_b200.dinov2_engine import swiglu
    hidden = 1024
    g = torch.Generator().manual_seed(rows)
    a = torch.linspace(-120.0, 120.0, rows * hidden)[torch.randperm(rows * hidden, generator=g)].view(rows, hidden)
    b = (torch.rand(rows, hidden, generator=g) * 2 - 1) * 50.0
    out = swiglu(torch.cat([a, b], dim=1).cuda()).cpu().double()
    a, b = a.double(), b.double()
    assert torch.isfinite(out).all()
    low, high = a <= -100.0, a >= 20.0
    assert low.any() and high.any()
    assert (out[low] == 0).all()
    ab = (a * b)[high]
    assert ((out[high] - ab).abs() <= ab.abs() * 2.0 ** -11 + 2.0 ** -25).all()
    mid = ~(low | high)
    ref = F.silu(a) * b
    err = ((out - ref).abs() / ref.abs().clamp_min(1e-3))[mid].max().item()
    print(f"\nswiglu rows={rows}: {err:.2e} (bar {SWIGLU_BAR:.1e})")
    assert err <= SWIGLU_BAR, err

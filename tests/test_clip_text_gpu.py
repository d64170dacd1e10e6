"""The CLIP text tower (csrc/clip_text.cu) against float64: the causal attention kernel alone, every block and the
whole tower against the declared-rounding oracle (oracle/clip_text.py) at the three released geometries, and the
zero-shot head (row normalisation + classifier head) against float64 logits."""
import math

import pytest
import torch

from clip_text_bars import ATTENTION_ATOL, ATTENTION_REL, BLOCK, FEATURES, LOGITS
from oracle import clip_text as T
from video_features_b200 import synthetic_weights
from video_features_b200.class_head import ClassHead
from video_features_b200.clip_text_engine import ClipTextEngine, ZeroShotHead, attention, l2_normalize_rows

pytestmark = pytest.mark.gpu

VOCAB = 1000
GEOMETRIES = [(512, 1024), (640, 640), (768, 768)]


def _prompts(n, seed, lo=6, hi=21):
    g = torch.Generator().manual_seed(seed)
    tokens = torch.zeros(n, 77, dtype=torch.int32)
    for b in range(n):
        k = int(torch.randint(lo, hi, (1,), generator=g))
        tokens[b, 0] = VOCAB - 2
        tokens[b, 1:k - 1] = torch.randint(0, VOCAB - 2, (k - 2,), generator=g)
        tokens[b, k - 1] = VOCAB - 1
    return tokens


def _attention64(qkv, heads):
    q, k, v = qkv.double().chunk(3, -1)
    return T._causal_attention(q, k, v, heads)


@pytest.mark.parametrize("heads", [8, 10, 12])
def test_attention_against_float64_and_length_independent(cuda_device, heads):
    g = torch.Generator().manual_seed(heads)
    n, W = 37, heads * 64
    qkv = (torch.randn(n, 77, 3 * W, generator=g) * 1.5).half()
    full = attention(qkv.to(cuda_device), heads).cpu()
    for S in (1, 2, 7, 63, 64, 65, 77):
        out = attention(qkv[:, :S].contiguous().to(cuda_device), heads).cpu()
        ref = _attention64(qkv[:, :S], heads)
        excess = ((out.double() - ref).abs() - ATTENTION_REL * ref.abs()).max().item()
        assert excess < ATTENTION_ATOL, (S, excess)
        assert torch.equal(out, full[:, :S]), S          # row i's bits do not depend on the rows after it


def test_attention_refuses_long_rows(cuda_device):
    with pytest.raises(RuntimeError, match="rows must be 1..77"):
        attention(torch.zeros(1, 78, 3 * 512, dtype=torch.float16, device=cuda_device), 8)


def _rel_rows(a, b):
    return ((a.double() - b).norm(dim=-1) / b.norm(dim=-1)).max().item()


@pytest.mark.parametrize("width,embed", GEOMETRIES)
def test_tower_block_by_block_and_end_to_end(cuda_device, width, embed):
    sd = synthetic_weights.clip_text_state_dict(width, width, embed, VOCAB)
    eng = ClipTextEngine(sd, cuda_device.index or 0)
    assert (eng.width, eng.heads, eng.layers, eng.context, eng.embed, eng.vocab) == (width, width // 64, 12, 77,
                                                                                    embed, VOCAB)
    tokens = _prompts(48, width)
    ref, streams = T.encode_text_declared(sd, tokens, taps=True)
    for i in range(12):
        got = eng.blocks(streams[i].float().to(cuda_device), i, 1).cpu()
        assert _rel_rows(got, T.block(sd, i, streams[i])) < BLOCK, i
    t = eng.encode(tokens.numpy()).cpu()
    assert (t.double().norm(dim=1) - 1).abs().max().item() < 1e-6
    err = (t.double() - ref).norm(dim=1).max().item()
    assert err < FEATURES, err
    # the length cut: the same prompts among longer ones (a larger L), and in chunks of a small workspace
    longer = torch.cat([tokens, _prompts(4, 7, 60, 78)])
    t2 = eng.encode(longer.numpy()).cpu()[:48]
    assert (t2.double() - ref).norm(dim=1).max().item() < FEATURES
    small = ClipTextEngine(sd, cuda_device.index or 0, max_rows=100)
    assert (small.encode(tokens.numpy()).cpu().double() - ref).norm(dim=1).max().item() < FEATURES


def test_tower_refuses_other_geometries_and_ids(cuda_device):
    sd = synthetic_weights.clip_text_state_dict(0, 512, 512, VOCAB, layers=12)
    bad = dict(sd, **{"ln_final.weight": torch.ones(1024), "ln_final.bias": torch.zeros(1024)})
    with pytest.raises(RuntimeError, match="text width 1024"):
        ClipTextEngine(bad, cuda_device.index or 0)
    few = {k: v for k, v in sd.items() if not k.startswith("transformer.resblocks.11.")}
    with pytest.raises(RuntimeError, match="11 blocks"):
        ClipTextEngine(few, cuda_device.index or 0)
    eng = ClipTextEngine(sd, cuda_device.index or 0)
    tokens = _prompts(2, 0)
    tokens[1, 3] = VOCAB
    with pytest.raises(RuntimeError, match="outside the vocabulary"):
        eng.encode(tokens.numpy())


def test_zero_shot_head_against_float64(cuda_device):
    g = torch.Generator().manual_seed(5)
    img = torch.randn(53, 512, generator=g) * 3
    text = torch.randn(400, 512, generator=g).double()
    text = text / text.norm(dim=1, keepdim=True)
    dev = img.to(cuda_device)
    normed = l2_normalize_rows(dev)
    assert torch.equal(dev.cpu(), img)                                   # the caller's features are untouched
    ref_n = img.double() / img.double().norm(dim=1, keepdim=True)
    assert (normed.cpu().double() - ref_n).abs().max().item() < 1e-6
    head = ClassHead((100.0 * text).float(), torch.zeros(400), cuda_device.index or 0)
    logits = head.forward(normed, 5)[0].cpu().double()
    ref = 100.0 * ref_n @ text.t()
    assert (logits - ref).abs().max().item() < 1e-3


@pytest.mark.parametrize("n_prompts", [3, 400])
def test_zero_shot_head_end_to_end(cuda_device, n_prompts):
    sd = synthetic_weights.clip_text_state_dict(2, 512, 512, VOCAB)
    sd["logit_scale"] = torch.tensor(math.log(80.0))                    # CLIP4Clip-style: not ln 100
    tokens = _prompts(n_prompts, 11)
    zs = ZeroShotHead(sd, tokens.numpy(), cuda_device.index or 0)
    img = torch.randn(17, 512, generator=torch.Generator().manual_seed(3))
    _, _, idx, tl, _ = zs.forward(img.to(cuda_device), 5)
    ref = T.zero_shot_logits(sd, img, T.encode_text_declared(sd, tokens))
    assert idx.shape == (17, min(5, n_prompts))
    got = tl.cpu().double()
    assert (got - ref.gather(1, idx.cpu().long())).abs().max().item() < LOGITS
    top = ref.topk(idx.shape[1], dim=1).values
    assert (got - top).abs().max().item() < LOGITS

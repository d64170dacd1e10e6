"""The references of tests/test_attention_hard_gpu.py (tests/attention_ref.py) without a GPU: their block sizes are
the kernels', each adapter equals its oracle's exact attention when nothing is rounded, each hard-input generator meets
its own preconditions, and each named defect moves the reference by SEPARATION times the bar that has to catch it
(the CLIP text kernel has no key blocks, mask constant or rel-pos term, so none of them applies to it)."""
import os
import re

import pytest
import torch

import attention_ref as A
import clip_vitl_ref
import dinov2_bars
import mvit_bars
import swin3d_bars
from oracle import clip_text as T
from oracle import mvit_net as M
from oracle import swin3d_net as SW

CSRC = os.path.join(A.ROOT, "video_features_b200", "csrc")
EXACT = 1e-12


def _errors(y, ref):
    y, ref = y.double().flatten(1), ref.double().flatten(1)
    rel = ((y - ref).norm(dim=1) / ref.norm(dim=1)).max().item()
    mx = ((y - ref).abs().amax(dim=1) / ref.abs().amax(dim=1)).max().item()
    return rel, mx


def _max_rel(y, ref):
    return ((y - ref).abs().max() / ref.abs().max()).item()


def _constant(src, name):
    text = open(os.path.join(CSRC, src)).read()
    return int(re.search(rf"\b{name} = (\d+)", text).group(1))


def test_block_sizes_are_the_kernels():
    assert A.DINOV2_KEY_BLOCK == _constant("clip_vitl_kernels.cu", "AL_KB") == clip_vitl_ref.KEY_BLOCK
    assert A.SWIN_KEY_BLOCK == _constant("swin3d_kernels.cu", "WA_KB")
    assert A.MVIT_KEY_BLOCK == _constant("mvit_kernels.cu", "MA_KB")
    assert A.MV_MAX_KEYS == _constant("mvit_kernels.h", "MV_MAX_KEYS")


# ------------------------------------------------------------------------------------------------------ equivalence

@pytest.mark.parametrize("S", [65, 257, 261])
def test_dinov2_equals_exact_attention(S):
    g = torch.Generator().manual_seed(S)
    qkv = (torch.randn(2, S, 3 * 384, generator=g) * 3).half()
    want = clip_vitl_ref.attention_core(qkv.double(), 6, rounding=frozenset())
    for kb in (S, A.DINOV2_KEY_BLOCK):
        e = _max_rel(A.dinov2(qkv, 6, rounding=False, key_block=kb), want)
        print(f"\ndinov2 S={S} key_block={kb} vs exact: {e:.1e}")
        assert e <= EXACT
    # at the declared rounding the streamed schedule is clip_vitl_ref's
    got = A.dinov2(qkv, 6)
    ref = clip_vitl_ref.attention_core(qkv.double(), 6, rounding=frozenset({"p", "att"}), key_block=64)
    assert _max_rel(got, ref) <= 2.0 ** -11


@pytest.mark.parametrize("shifted", [False, True])
@pytest.mark.parametrize("C,Tq,S_", [(96, 9, 14), (192, 16, 14), (384, 5, 7)])
def test_swin3d_equals_the_oracle_window_attention(C, Tq, S_, shifted):
    """S.window_attention with an identity projection on x, against the adapter on qkv = x W^T + b (a padded position
    is a zero row after norm1: its q / k / v are b)."""
    g = torch.Generator().manual_seed(C + Tq + S_)
    heads = C // 32
    x = torch.randn(2, Tq, S_, S_, C, generator=g, dtype=torch.float64)
    w = torch.randn(3 * C, C, generator=g, dtype=torch.float64) * C ** -0.5 * 2
    b = torch.randn(3 * C, generator=g, dtype=torch.float64)
    table = torch.randn(2535, heads, generator=g, dtype=torch.float64) * 3
    sd = {"p.qkv.weight": w, "p.qkv.bias": b, "p.proj.weight": torch.eye(C, dtype=torch.float64),
          "p.proj.bias": torch.zeros(C, dtype=torch.float64), "p.relative_position_bias_table": table}
    want = SW.window_attention(sd, "p", x, heads, shifted)
    qkv = x @ w.T + b
    for kb in (None, A.SWIN_KEY_BLOCK):
        e = _max_rel(A.swin3d(qkv, b, table, shifted, rounding=False, key_block=kb), want)
        print(f"\nswin3d C={C} T'={Tq} {S_}x{S_} shifted={shifted} key_block={kb} vs oracle: {e:.1e}")
        assert e <= EXACT


@pytest.mark.parametrize("v2", [False, True])
@pytest.mark.parametrize("S,K,heads", [(7, 14, 2), (14, 7, 1)])
def test_mvit_equals_the_oracle_attention(S, K, heads, v2):
    g = torch.Generator().manual_seed(S + K + v2)
    nq, nk = 1 + 8 * S * S, 1 + 8 * K * K
    q, k, v = (torch.randn(2, heads, n, 96, generator=g, dtype=torch.float64) * 2 for n in (nq, nk, nk))
    sp = 2 * max(S, K) - 1
    rel = tuple(torch.randn(r, 96, generator=g, dtype=torch.float64) * 0.3 for r in (sp, sp, 15)) if v2 else None
    want = M.attention(q, k, v, (8, S, S), (8, K, K), rel, resid=v2)
    for kb in (None, A.MVIT_KEY_BLOCK):
        e = _max_rel(A.mvit(q, k, v, (8, S, S), (8, K, K), rel, v2, rounding=False, key_block=kb), want)
        print(f"\nmvit q {S} kv {K} ({nk} keys) v2 {v2} key_block={kb} vs oracle: {e:.1e}")
        assert e <= EXACT


def test_mvit_chunks_restart_the_blocks():
    """416 is a whole number of 32-key blocks, so the chunks leave the schedule as plain 32-key blocks; a chunk that is
    not (100) restarts the blocks, and P rounded relative to a different running max shows."""
    g = torch.Generator().manual_seed(1)
    q, k, v = (torch.randn(1, 1, n, 96, generator=g, dtype=torch.float64) * 3 for n in (40, 1569, 1569))
    kw = dict(scale=96 ** -0.5, key_block=32)
    plain = A.attention(q, k, v, **kw)
    assert torch.equal(A.attention(q, k, v, chunk=A.MV_MAX_KEYS, **kw), plain)
    assert not torch.equal(A.attention(q, k, v, chunk=100, **kw), plain)


@pytest.mark.parametrize("L", [1, 2, 33, 77])
def test_clip_text_equals_the_oracle_attention(L):
    g = torch.Generator().manual_seed(L)
    qkv = torch.randn(3, L, 3 * 512, generator=g, dtype=torch.float64) * 3
    want = T._causal_attention(*qkv.chunk(3, -1), 8)
    e = _max_rel(A.clip_text(qkv, 8, rounding=False), want)
    print(f"\nclip text L={L} vs oracle: {e:.1e}")
    assert e <= EXACT


# ---------------------------------------------------------------------------------------------------------- hardness

@pytest.mark.parametrize("S", [257, 261])
def test_dinov2_inputs_are_hard(S):
    qkv, keys = A.dinov2_hard(S, 6, 1)
    assert keys[-1] == (2 if S == 261 else S - 1)
    s = A.dinov2_scores(qkv[:-1], 6)
    for f, key in enumerate(keys):
        dominant = torch.zeros(S, dtype=torch.bool)
        dominant[key] = True
        hit, med = A.hardness(s[f], dominant)
        print(f"\ndinov2 S={S} key {key}: hit {hit:.2f}, median row max {med:.0f}")
        assert hit >= 0.1 and med > 15.0
    assert (qkv[-1] == qkv[-1, :1]).all()


@pytest.mark.parametrize("C,Tq,S_,shifted", [(96, 9, 14, True), (768, 16, 7, True), (384, 5, 14, True),
                                              (192, 9, 14, False)])
def test_swin3d_inputs_are_hard(C, Tq, S_, shifted):
    qkv, bias, table = A.swin3d_hard(2, C, Tq, S_, shifted, 7)
    hit, med, cross = A.swin3d_stats(qkv, bias, table, shifted)
    print(f"\nswin3d C={C} T'={Tq} {S_}x{S_} shifted={shifted}: hit {hit:.2f}, median row max {med:.0f}, "
          f"cross-region max {cross:.0f}")
    assert hit >= 0.1 and med > 15.0 and table.abs().max() > 19.0
    assert cross > 100.0 if shifted else cross == -float("inf")


@pytest.mark.parametrize("S,K,heads,v2", [(7, 14, 8, True), (14, 7, 4, True), (7, 7, 8, False)])
def test_mvit_inputs_are_hard(S, K, heads, v2):
    q, k, _, rel = A.mvit_hard(S, K, heads, v2, 5)
    hit, med, last_block, last_chunk = A.mvit_stats(q, k, S, K, heads, rel)
    print(f"\nmvit q {S} kv {K} v2 {v2}: hit {hit:.2f}, median row max {med:.0f}, max in the last block "
          f"{last_block:.3f}, in the last chunk {last_chunk:.3f}")
    assert hit >= 0.1 and med > 15.0 and last_block > 0.0 and last_chunk > 0.0
    if v2:
        rb = A.mvit_add(A.mvit_heads(q, heads), (8, S, S), (8, K, K), tuple(r.double() for r in rel), k.shape[1])
        assert rb.abs().amax().item() > 20.0


def test_clip_text_inputs_are_hard():
    (hit0, med0), (hitl, medl), top = A.clip_text_stats(A.clip_text_hard(16, 8, 8), 8)
    print(f"\nclip text: sink hit {hit0:.2f} median {med0:.0f}, last key hit {hitl:.2f} median {medl:.0f}, "
          f"top {top:.0f}")
    assert hit0 >= 0.1 and med0 > 15.0 and hitl >= 0.1 and medl > 15.0 and top > 200.0


# ---------------------------------------------------------------------------------------------------------- controls

def _separates(name, moved, bar):
    sep = max(moved[0] / bar[0], moved[1] / bar[1])
    print(f"\ncontrol {name}: moves the reference {moved[0]:.2e} / {moved[1]:.2e}, {sep:.0f}x the bar")
    assert sep >= A.SEPARATION, (name, moved, bar)


def test_dinov2_controls():
    qkv, _ = A.dinov2_hard(257, 6, 1)
    ref = A.dinov2(qkv, 6)
    _separates("dinov2 no_rescale", _errors(A.dinov2(qkv, 6, defects=("no_rescale",)), ref),
               dinov2_bars.BARS["attention hard"])


@pytest.mark.parametrize("C,Tq,S_", [(96, 9, 14), (768, 16, 7)])
def test_swin3d_controls(C, Tq, S_):
    qkv, bias, table = A.swin3d_hard(2, C, Tq, S_, True, 7)
    ref = A.swin3d(qkv, bias, table, True)
    for d in ("mask_in_log2_units", "no_rescale"):
        _separates(f"swin3d C={C} T'={Tq} {d}", _errors(A.swin3d(qkv, bias, table, True, defects=(d,)), ref),
                   swin3d_bars.BARS["attention hard"])


@pytest.mark.parametrize("S,K,heads,v2", [(7, 14, 8, True), (7, 7, 8, False)])
def test_mvit_controls(S, K, heads, v2):
    q, k, v, rel = A.mvit_hard(S, K, heads, v2, 5)
    args = (A.mvit_heads(q, heads), A.mvit_heads(k, heads), A.mvit_heads(v, heads), (8, S, S), (8, K, K),
            tuple(r.double() for r in rel) if rel else None, v2)
    ref = A.mvit(*args)
    for d in ("no_rescale",) + (("relpos_scaled",) if v2 else ()):
        _separates(f"mvit q {S} kv {K} v2 {v2} {d}", _errors(A.mvit(*args, defects=(d,)), ref),
                   mvit_bars.BARS["attention hard"])


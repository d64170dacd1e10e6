"""float64 references of the streamed attention kernels at their declared rounding, and the hard inputs that test them
(tests/test_attention_hard_gpu.py on the GPU, tests/test_attention_hard_cpu.py for the reference, the inputs and the
controls).

``attention`` is softmax(q k^T * scale + add + mask) v in float64.  With ``key_block`` set it takes the kernels' online
softmax: the keys in blocks of ``key_block`` (the blocks restart at every ``chunk`` keys, the shared-memory chunks of
the MViT kernel), a running max m and sum l per row; each block's P = exp(s - m), m already raised to the block's max,
is rounded to fp16 (``round_p``) before P.V, l sums the unrounded P, and the accumulated output and l are rescaled by
exp(m_old - m_new) when the max grows; 1 / l is applied to the unrounded output.  Without ``key_block`` it is one pass
over every key (P relative to the row max), the CLIP text kernel's two-pass softmax.

The adapters give each kernel's inputs and declared rounding (P and the output fp16, both with ``rounding``):
  dinov2    vitl_attention_kernel (csrc/clip_vitl_kernels.cu), 64-key blocks, scale 1 / 8
  swin3d    window_attention_kernel (csrc/swin3d_kernels.cu), 64-key blocks within a window, the bias table and the
            -100 shift mask; padded positions take fp16(bias_qkv) as k and v
  mvit      pool_attention_kernel (csrc/mvit_kernels.cu), 32-key blocks in chunks of MV_MAX_KEYS, the rel-pos terms of
            the unscaled q on token rows and columns, + q on token rows
  clip_text attention_kernel (csrc/clip_text_kernels.cu), causal, two fp32 passes, P not rounded

Named defects, each a plausible kernel bug, for the controls (``defects``):
  mask_in_log2_units  the -100 mask added after the scores are taken to log2 units: -100 ln 2 in natural units
  no_rescale          the accumulated output not rescaled when the running max grows
  relpos_scaled       the additive term taken from the scaled q (the rel-pos term times the scale)
"""
from __future__ import annotations

import math
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import mvit_net as M  # noqa: E402
from oracle import swin3d_net as SW  # noqa: E402

DINOV2_KEY_BLOCK = 64       # AL_KB, csrc/clip_vitl_kernels.cu
SWIN_KEY_BLOCK = 64         # WA_KB, csrc/swin3d_kernels.cu
MVIT_KEY_BLOCK = 32         # MA_KB, csrc/mvit_kernels.cu
MV_MAX_KEYS = 416           # csrc/mvit_kernels.h: keys per shared-memory chunk
DEFECTS = ("mask_in_log2_units", "no_rescale", "relpos_scaled")
# a named defect must move the reference by at least this factor times the kernel's bar (in one of the two measures)
SEPARATION = 3.0


def r16(t: torch.Tensor) -> torch.Tensor:
    return t.half().to(t.dtype)


def scores(q, k, scale, add=None, mask=None, defects=()):
    """The scores in natural units, with the additive term and the mask as the defects place them."""
    s = (q @ k.transpose(-1, -2)) * scale
    if add is not None:
        s = s + (add * scale if "relpos_scaled" in defects else add)
    if mask is not None:
        s = s + (mask * math.log(2.0) if "mask_in_log2_units" in defects else mask)
    return s


def attention(q, k, v, add=None, mask=None, *, scale, key_block=None, chunk=None, round_p=True, defects=()):
    """q (..., Sq, d), k / v (..., Sk, d) float64; add / mask broadcast to (..., Sq, Sk) -> (..., Sq, d) unrounded."""
    assert set(defects) <= set(DEFECTS), defects
    s = scores(q, k, scale, add, mask, defects)
    Sk = s.shape[-1]
    if not key_block:
        p = torch.exp(s - s.amax(-1, keepdim=True))
        return (r16(p) if round_p else p) @ v / p.sum(-1, keepdim=True)
    chunk = chunk or Sk
    m = torch.full(s.shape[:-1] + (1,), -math.inf, dtype=s.dtype, device=s.device)
    l = torch.zeros_like(m)
    o = torch.zeros(s.shape[:-1] + (v.shape[-1],), dtype=s.dtype, device=s.device)
    for c0 in range(0, Sk, chunk):
        for b0 in range(c0, min(c0 + chunk, Sk), key_block):
            b1 = min(b0 + key_block, c0 + chunk, Sk)
            sb = s[..., b0:b1]
            mn = torch.maximum(m, sb.amax(-1, keepdim=True))
            carry = torch.exp(m - mn)
            e = torch.exp(sb - mn)
            l = l * carry + e.sum(-1, keepdim=True)
            o = (o if "no_rescale" in defects else o * carry) + (r16(e) if round_p else e) @ v[..., b0:b1, :]
            m = mn
    return o / l


# ---------------------------------------------------------------------------------------------------------- adapters

def _heads(t, heads, hd):
    n, S, _ = t.shape
    return t.double().view(n, S, heads, hd).transpose(1, 2)


def _concat(o):
    n, h, S, d = o.shape
    return o.transpose(1, 2).reshape(n, S, h * d)


def dinov2(qkv, heads, *, rounding=True, key_block=DINOV2_KEY_BLOCK, defects=()):
    """qkv (n, S, 3 heads 64) -> (n, S, heads 64) float64."""
    q, k, v = (_heads(t, heads, 64) for t in qkv.split(heads * 64, -1))
    o = _concat(attention(q, k, v, scale=0.125, key_block=key_block, round_p=rounding, defects=defects))
    return r16(o) if rounding else o


class SwinWindows:
    """The window partition of a (n, T', H, W, X) map as window_attention_kernel makes it: padded to whole windows,
    rolled back by the shift, windows of ``vol`` positions t-major.  ``real`` marks the positions inside (T', H, W),
    ``region`` is each position's shift region (None unshifted)."""

    def __init__(self, size, shifted, device="cpu"):
        self.size = tuple(size)
        self.win, self.sh = SW.window_and_shift(self.size, shifted)
        self.pad = [(self.win[i] - self.size[i] % self.win[i]) % self.win[i] for i in range(3)]
        self.padded = tuple(self.size[i] + self.pad[i] for i in range(3))
        self.grid = tuple(self.padded[i] // self.win[i] for i in range(3))
        self.nw = self.grid[0] * self.grid[1] * self.grid[2]
        self.vol = self.win[0] * self.win[1] * self.win[2]
        real = torch.zeros(self.padded, dtype=torch.bool)
        real[:self.size[0], :self.size[1], :self.size[2]] = True
        self.real = self.part(real[None, ..., None])[0, ..., 0]                       # (nw, vol)
        self.region = None
        if sum(self.sh):
            reg = SW.region_ids(self.padded, self.win, self.sh)                     # in rolled coordinates already
            self.region = self._split(reg[None, ..., None])[0, ..., 0].to(device)  # (nw, vol)

    def _split(self, x):
        n, c = x.shape[0], x.shape[-1]
        (gt, gh, gw), (wt, wh, ww) = self.grid, self.win
        x = x.reshape(n, gt, wt, gh, wh, gw, ww, c).permute(0, 1, 3, 5, 2, 4, 6, 7)
        return x.reshape(n, self.nw, self.vol, c)

    def part(self, x, fill=None):
        """(n, T', H, W, X) or already padded -> (n, nw, vol, X); padded positions take ``fill`` (X,) (zero if None)."""
        if tuple(x.shape[1:4]) != self.padded:
            base = torch.zeros((x.shape[0],) + self.padded + (x.shape[-1],), dtype=x.dtype, device=x.device)
            if fill is not None:
                base[:] = fill
            base[:, :self.size[0], :self.size[1], :self.size[2]] = x
            x = base
        if sum(self.sh):
            x = torch.roll(x, shifts=tuple(-s for s in self.sh), dims=(1, 2, 3))
        return self._split(x)

    def merge(self, y):
        """(n, nw, vol, X) -> (n, T', H, W, X)."""
        n, c = y.shape[0], y.shape[-1]
        (gt, gh, gw), (wt, wh, ww) = self.grid, self.win
        y = y.reshape(n, gt, gh, gw, wt, wh, ww, c).permute(0, 1, 4, 2, 5, 3, 6, 7).reshape((n,) + self.padded + (c,))
        if sum(self.sh):
            y = torch.roll(y, shifts=tuple(self.sh), dims=(1, 2, 3))
        return y[:, :self.size[0], :self.size[1], :self.size[2]]

    def mask(self, dtype=torch.float64):
        """(nw, 1, vol, vol): -100 where query and key lie in different shift regions; None unshifted."""
        if self.region is None:
            return None
        return torch.where(self.region[:, None, :, None] != self.region[:, None, None, :], -100.0, 0.0).to(dtype)

    def table_term(self, table):
        """(heads, vol, vol) from the (2535, heads) relative-position bias table."""
        idx = SW.bias_index(self.win).reshape(-1).to(table.device)
        return table.double()[idx].view(self.vol, self.vol, -1).permute(2, 0, 1)


def swin3d_qkv(qkv, bias, shifted, *, rounding=True):
    """q, k, v (n, nw, heads, vol, 32) float64 of a (n, T', H, W, 3C) qkv map, and its SwinWindows; padded positions
    take bias_qkv (fp16-rounded with ``rounding``, as the kernel stores them), a zero row after norm1."""
    n, t, h, w, c3 = qkv.shape
    win = SwinWindows((t, h, w), shifted, qkv.device)
    b = bias.double().to(qkv.device)
    x = win.part(qkv.double(), r16(b) if rounding else b)
    x = x.view(n, win.nw, win.vol, 3, c3 // 96, 32).permute(3, 0, 1, 4, 2, 5)
    return x[0], x[1], x[2], win


def swin3d(qkv, bias, table, shifted, *, rounding=True, key_block=SWIN_KEY_BLOCK, defects=()):
    """qkv (n, T', H, W, 3C) fp16, bias_qkv (3C,), table (2535, C / 32) -> (n, T', H, W, C) float64."""
    q, k, v, win = swin3d_qkv(qkv, bias, shifted, rounding=rounding)
    o = attention(q, k, v, win.table_term(table), win.mask(), scale=32 ** -0.5, key_block=key_block,
                  round_p=rounding, defects=defects)                                 # (n, nw, heads, vol, 32)
    n, nw, heads, vol, _ = o.shape
    y = win.merge(o.permute(0, 1, 3, 2, 4).reshape(n, nw, vol, heads * 32))
    return r16(y) if rounding else y


def mvit_add(q, q_thw, k_thw, rel, nk):
    """The rel-pos term (B, heads, Nq, Nk) of M.attention: on token rows and columns only, from the unscaled q."""
    add = torch.zeros(q.shape[:-1] + (nk,), dtype=q.dtype, device=q.device)
    add[:, :, 1:, 1:] = M.rel_bias(q, q_thw, k_thw, *rel)
    return add


def mvit(q, k, v, q_thw, k_thw, rel=None, resid=False, *, rounding=True, key_block=MVIT_KEY_BLOCK, chunk=MV_MAX_KEYS,
         defects=()):
    """M.attention's arguments: q (B, heads, Nq, 96), k / v (B, heads, Nk, 96) float64 -> (B, heads, Nq, 96)."""
    add = mvit_add(q, q_thw, k_thw, rel, k.shape[2]) if rel is not None else None
    o = attention(q, k, v, add, scale=M.HEAD_DIM ** -0.5, key_block=key_block, chunk=chunk, round_p=rounding,
                  defects=defects)
    if resid:
        o[:, :, 1:] += q[:, :, 1:]
    return r16(o) if rounding else o


def causal_mask(L, device="cpu"):
    return torch.zeros(L, L, dtype=torch.float64, device=device).masked_fill(
        torch.ones(L, L, dtype=torch.bool, device=device).triu(1), -math.inf)


def clip_text(qkv, heads, *, rounding=True):
    """qkv (n, L, 3 heads 64) -> (n, L, heads 64) float64: causal, P unrounded, the output fp16 with ``rounding``."""
    q, k, v = (_heads(t, heads, 64) for t in qkv.split(heads * 64, -1))
    o = _concat(attention(q, k, v, mask=causal_mask(qkv.shape[1], qkv.device), scale=0.125, round_p=False))
    return r16(o) if rounding else o


# ------------------------------------------------------------------------------------------------------ hard inputs

def hardness(s, dominant, valid=None):
    """(fraction of rows whose max is a dominant key, median row max) of scores s (..., Sq, Sk); ``dominant`` a bool
    (..., Sq or 1, Sk) marking the dominant keys of each row, ``valid`` a bool (..., Sq) of the rows that count."""
    top = s.argmax(-1, keepdim=True)
    hit = torch.gather(dominant.expand_as(s), -1, top)[..., 0]
    mx = s.amax(-1)
    if valid is not None:
        valid = valid.expand_as(hit)
        hit, mx = hit[valid], mx[valid]
    return hit.double().mean().item(), mx.median().item()


def dinov2_hard(S, heads, seed):
    """Frames of scores in the tens to hundreds: q and k scaled 3 .. 6 (scores grow with the square) and one key row
    4x, so that the max of many rows falls on it: key 0, 63 and 64 (either side of the first block boundary), S - 1
    (alone in its block at 257) and, with registers (261), register token 2.  The last frame: every row the same.
    -> (qkv (n, S, 3 heads 64) fp16, the dominant key of each frame but the last)."""
    g = torch.Generator().manual_seed(seed)
    keys = [0, 63, 64, S - 1] + ([2] if S == 261 else [])
    scale = (3.0, 4.0, 5.0, 6.0, 4.0)
    D = heads * 64
    qkv = torch.randn(len(keys) + 1, S, 3 * D, generator=g)
    for f, key in enumerate(keys):
        qkv[f, :, :2 * D] *= scale[f]
        qkv[f, key, D:2 * D] *= 4.0
    qkv[-1, :, :2 * D] *= 4.0
    qkv[-1] = qkv[-1, 7].clone()
    return qkv.half(), keys


def dinov2_scores(qkv, heads):
    q, k, _ = (_heads(t, heads, 64) for t in qkv.split(heads * 64, -1))
    return scores(q, k, 0.125)


def swin3d_hard(n, C, Tq, S, shifted, seed):
    """A (n, T', S, S, 3C) qkv map of scores in the tens to hundreds (q and k scaled 3), the last key in partition order
    of every window scaled 8 (scores across shift regions pass 100, so that the -100 mask competes with them), a bias
    table uniform in [-20, 20], and a bias_qkv whose k part is as large as a dominant key's, so that where T' is padded
    the padded positions' keys (fp16(bias_qkv)) dominate too.  -> (qkv fp16, bias (3C,) fp32, table (2535, C / 32))."""
    g = torch.Generator().manual_seed(seed)
    qkv = torch.randn(n, Tq, S, S, 3 * C, generator=g)
    qkv[..., :2 * C] *= 3.0
    win = SwinWindows((Tq, S, S), shifted)
    last = torch.zeros(win.nw, win.vol, 1)
    last[:, -1] = 1.0
    last = win.merge(last[None].expand(1, -1, -1, -1))[0, ..., 0].bool()             # (T', S, S)
    qkv[:, last, C:2 * C] *= 8.0
    bias = torch.randn(3 * C, generator=g) * 0.5
    bias[C:2 * C] = torch.randn(C, generator=g) * 24.0
    table = (torch.rand(2535, C // 32, generator=g) * 2 - 1) * 20.0
    return qkv.half(), bias, table


def swin3d_stats(qkv, bias, table, shifted):
    """(fraction of the real query rows whose max is a dominant key -- the last in partition order, or a padded
    position's --, their median row max, the largest score across shift regions before the mask)."""
    q, k, _, win = swin3d_qkv(qkv, bias, shifted)
    s = scores(q, k, 32 ** -0.5, win.table_term(table).to(q.device))           # (n, nw, heads, vol, vol)
    mask = win.mask()
    cross = s[(mask != 0).expand_as(s)].max().item() if mask is not None else -math.inf
    if mask is not None:
        s = s + mask
    dominant = ~win.real.to(s.device)
    dominant[:, -1] = True
    hit, med = hardness(s, dominant[None, :, None, None, :], win.real.to(s.device)[None, :, None, :])
    return hit, med, cross


def mvit_dominant_keys(nk, n):
    """Per clip: the last key (the last 32-key block, and at 1569 keys alone in it and in the last chunk), a key in the
    last block (393 keys) or in the middle of the last chunk (1569 keys: chunk 3 holds keys 1248 .. 1568), the class
    token key."""
    return [nk - 1, nk - 9 if nk <= MV_MAX_KEYS else 1300, 0][:n]


def mvit_hard(S, K, heads, v2, seed, device="cpu"):
    """Pooling-attention inputs with scores in the tens: q and k scaled 3, one key row per clip 8x
    (mvit_dominant_keys), v2's rel-pos tables scaled 0.5 (terms of tens from the unscaled q).  q is a column slice of
    qkv rows at S = 56 (v1's unpooled q), contiguous otherwise.  -> (q, k, v fp16 (n, 1 + N, heads 96), rel or None)."""
    g = torch.Generator().manual_seed(seed)
    c, n = heads * 96, 2 if S >= 28 else 3
    nq, nk = 1 + 8 * S * S, 1 + 8 * K * K
    qkv = (torch.randn(n, nq, 3 * c, generator=g) * 3.0).half().to(device)
    q = qkv[..., :c] if S == 56 else qkv[..., :c].contiguous()
    k = torch.randn(n, nk, c, generator=g) * 3.0
    for b, key in enumerate(mvit_dominant_keys(nk, n)):
        k[b, key] *= 8.0
    v = torch.randn(n, nk, c, generator=g)
    rel = None
    if v2:
        sp = 2 * max(S, K) - 1
        rel = tuple((torch.randn(r, 96, generator=g) * 0.5).to(device) for r in (sp, sp, 15))
    return q, k.half().to(device), v.half().to(device), rel


def mvit_heads(t, heads):
    return t.double().reshape(t.shape[0], t.shape[1], heads, 96).transpose(1, 2)


def mvit_stats(q, k, S, K, heads, rel):
    """(hit fraction of each clip's dominant key, median row max, fraction of rows whose max lies in the last 32-key
    block, the same for the last chunk) over the scores with the rel-pos term."""
    qh, kh = mvit_heads(q, heads), mvit_heads(k, heads)
    nk = kh.shape[2]
    add = mvit_add(qh, (8, S, S), (8, K, K), tuple(r.double().to(q.device) for r in rel), nk) if rel else None
    s = scores(qh, kh, M.HEAD_DIM ** -0.5, add)
    dominant = torch.zeros(s.shape[0], 1, 1, nk, dtype=torch.bool, device=s.device)
    for b, key in enumerate(mvit_dominant_keys(nk, s.shape[0])):
        dominant[b, 0, 0, key] = True
    hit, med = hardness(s, dominant)
    top = s.argmax(-1)
    last_block = (top >= (nk - 1) // MVIT_KEY_BLOCK * MVIT_KEY_BLOCK).double().mean().item()
    last_chunk = (top >= (nk - 1) // MV_MAX_KEYS * MV_MAX_KEYS).double().mean().item()
    return hit, med, last_block, last_chunk


def clip_text_hard(n, heads, seed):
    """(n, 77, 3 heads 64) fp16: the first half of the prompts with key 0 a sink (k0 along a direction every q shares,
    at strengths 1 .. 25: scores from about 8, where it competes, to several hundred), the second half with every key
    near 1.5x its own query (each row's last key dominant, at scores near 50)."""
    g = torch.Generator().manual_seed(seed)
    W, L = heads * 64, 77
    qkv = torch.randn(n, L, 3 * W, generator=g)
    h = n // 2
    u = torch.randn(W, generator=g)
    qkv[:h, :, :W] += u
    strength = torch.linspace(1.0, 25.0, h)
    qkv[:h, 0, W:2 * W] = strength[:, None] * u
    qkv[h:, :, :W] *= 2.0
    qkv[h:, :, W:2 * W] = 1.5 * qkv[h:, :, :W] + 0.5 * qkv[h:, :, W:2 * W]
    return qkv.half()


def clip_text_stats(qkv, heads):
    """((hit fraction of key 0, median row max) of the sink prompts, the same of each row's last key in the others,
    the largest score)."""
    q, k, _ = (_heads(t, heads, 64) for t in qkv.split(heads * 64, -1))
    L = q.shape[2]
    s = scores(q, k, 0.125, mask=causal_mask(L, q.device))
    h = q.shape[0] // 2
    sink = torch.zeros(L, dtype=torch.bool, device=s.device)
    sink[0] = True
    last = torch.eye(L, dtype=torch.bool, device=s.device)
    return hardness(s[:h, :, 1:], sink), hardness(s[h:, :, 1:], last[1:]), s.amax().item()   # row 0 sees key 0 only

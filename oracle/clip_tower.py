"""fp32 CPU restatement of the CLIP ViT image tower -- test oracle only -- and, below it, the same tower in any float
dtype with the engine's declared fp16 rounding (``encode_image(..., dtype=torch.float64, declared_rounding=True)``, and its
pieces ``embed`` / ``block`` / ``head``), what tests/test_clip_float64_gpu.py holds the engine to.

The reference runs ``model.encode_image(frames)`` (models/CLIP/extract_clip.py:128)
on a model returned by ``clip.load("ViT-B/32")`` (extract_clip.py:47).  ``clip`` is
openai/CLIP (third-party, un-vendored, version unpinned by the reference; weights
fetched at run time) -- absent offline.  This file restates the published algorithm
of ``clip/model.py``: ``VisionTransformer.forward``, ``ResidualAttentionBlock``,
``LayerNorm`` (fp32 compute), ``QuickGELU`` and ``CLIP.encode_image``; the state-dict
keys are openai's (``visual.*``) so a user-supplied real checkpoint loads unchanged.

PARITY UNPINNED versus the reference itself (no reference test or golden vector
touches this boundary and neither the package nor its weights can be obtained here).
It IS pinned against an independent implementation of the same math: HF
``transformers.CLIPVisionModelWithProjection`` (tests/test_oracle_clip.py).
"""
from __future__ import annotations

import math
from collections import OrderedDict
from typing import Dict

import torch
import torch.nn.functional as F

# ViT-B/32 hyper-parameters (clip/model.py: build_model for "ViT-B/32")
WIDTH = 768
LAYERS = 12
HEADS = 12
PATCH = 32
RES = 224
GRID = RES // PATCH            # 7
TOKENS = GRID * GRID + 1       # 50
MLP = 4 * WIDTH                # 3072
EMBED = 512
LN_EPS = 1e-5


def synthetic_state_dict(seed: int = 0, dtype=torch.float32, patch: int = PATCH) -> "OrderedDict[str, torch.Tensor]":
    """Seeded synthetic weights in openai's ``visual.*`` key layout.

    Scales follow clip/model.py (VisionTransformer.__init__: ``scale = width**-0.5``
    for class/positional embedding and proj; CLIP.initialize_parameters:
    attn_std = width**-0.5, proj_std = width**-0.5 * (2*layers)**-0.5,
    fc_std = (2*width)**-0.5) so activations have realistic magnitudes.  LayerNorm
    gains/biases and linear biases are perturbed so every term of the forward is
    exercised by parity tests.
    """
    g = torch.Generator().manual_seed(seed)

    def rn(*shape, std=1.0):
        return torch.randn(*shape, generator=g, dtype=torch.float32) * std

    scale = WIDTH ** -0.5
    attn_std = WIDTH ** -0.5
    proj_std = (WIDTH ** -0.5) * ((2 * LAYERS) ** -0.5)
    fc_std = (2 * WIDTH) ** -0.5
    sd: "OrderedDict[str, torch.Tensor]" = OrderedDict()
    sd["visual.class_embedding"] = rn(WIDTH, std=scale)
    sd["visual.positional_embedding"] = rn((RES // patch) ** 2 + 1, WIDTH, std=scale)
    sd["visual.proj"] = rn(WIDTH, EMBED, std=scale)
    sd["visual.conv1.weight"] = rn(WIDTH, 3, patch, patch, std=(3 * patch * patch) ** -0.5)
    for name in ("ln_pre", "ln_post"):
        sd[f"visual.{name}.weight"] = 1.0 + rn(WIDTH, std=0.1)
        sd[f"visual.{name}.bias"] = rn(WIDTH, std=0.05)
    for i in range(LAYERS):
        p = f"visual.transformer.resblocks.{i}."
        sd[p + "attn.in_proj_weight"] = rn(3 * WIDTH, WIDTH, std=attn_std)
        sd[p + "attn.in_proj_bias"] = rn(3 * WIDTH, std=0.02)
        sd[p + "attn.out_proj.weight"] = rn(WIDTH, WIDTH, std=proj_std)
        sd[p + "attn.out_proj.bias"] = rn(WIDTH, std=0.02)
        sd[p + "ln_1.weight"] = 1.0 + rn(WIDTH, std=0.1)
        sd[p + "ln_1.bias"] = rn(WIDTH, std=0.05)
        sd[p + "mlp.c_fc.weight"] = rn(MLP, WIDTH, std=fc_std)
        sd[p + "mlp.c_fc.bias"] = rn(MLP, std=0.02)
        sd[p + "mlp.c_proj.weight"] = rn(WIDTH, MLP, std=proj_std)
        sd[p + "mlp.c_proj.bias"] = rn(WIDTH, std=0.02)
        sd[p + "ln_2.weight"] = 1.0 + rn(WIDTH, std=0.1)
        sd[p + "ln_2.bias"] = rn(WIDTH, std=0.05)
    return OrderedDict((k, v.to(dtype)) for k, v in sd.items())


def _ln(x: torch.Tensor, w: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    # clip/model.py LayerNorm: compute in fp32, cast back to the input dtype.
    return F.layer_norm(x.float(), (x.shape[-1],), w.float(), b.float(), LN_EPS).to(x.dtype)


def _quick_gelu(x: torch.Tensor) -> torch.Tensor:
    # clip/model.py QuickGELU
    return x * torch.sigmoid(1.702 * x)


def _attention(x: torch.Tensor, w_in, b_in, w_out, b_out) -> torch.Tensor:
    """nn.MultiheadAttention(width, heads) self-attention, no mask, batch-first here.

    q is scaled by head_dim**-0.5 before q@k^T (torch MHA semantics, what
    ResidualAttentionBlock.attention calls with need_weights=False).
    """
    B, S, D = x.shape
    hd = D // HEADS
    qkv = F.linear(x, w_in, b_in)                      # (B,S,3D) = cat(q,k,v)
    q, k, v = qkv.split(D, dim=-1)
    q = q.view(B, S, HEADS, hd).transpose(1, 2) * (hd ** -0.5)
    k = k.view(B, S, HEADS, hd).transpose(1, 2)
    v = v.view(B, S, HEADS, hd).transpose(1, 2)
    att = torch.softmax(q @ k.transpose(-1, -2), dim=-1)
    o = (att @ v).transpose(1, 2).reshape(B, S, D)
    return F.linear(o, w_out, b_out)


@torch.no_grad()
def encode_image(sd: Dict[str, torch.Tensor], frames: torch.Tensor, *, return_hidden: bool = False, dtype=None,
                 declared_rounding: bool = False):
    """``CLIP.encode_image`` == ``VisionTransformer.forward``.

    ``dtype`` (e.g. torch.float64) runs the restatement built from ``embed`` / ``block`` / ``head`` below in that dtype;
    ``declared_rounding`` rounds to fp16 there exactly what the engine holds in fp16 (``DECLARED``).

    frames: (B,3,224,224) float, already normalised (output of the CLIP transform).
    returns (B,512) in the weight dtype.  No L2 normalisation (the reference saves
    the raw projection, extract_clip.py:128-131).
    """
    if dtype is not None or declared_rounding:
        assert not return_hidden
        return encode_image_declared(sd, frames, dtype=dtype or torch.float64, declared_rounding=declared_rounding)
    w = sd["visual.conv1.weight"]
    x = frames.to(w.dtype)
    patch = w.shape[-1]                                          # 32 (ViT-B/32) or 16 (ViT-B/16): conv stride == kernel
    x = F.conv2d(x, w, None, stride=patch)                       # (B,768,7,7) / (B,768,14,14)
    x = x.reshape(x.shape[0], x.shape[1], -1).permute(0, 2, 1)   # (B,49|196,768) row-major grid
    cls = sd["visual.class_embedding"].to(x.dtype).expand(x.shape[0], 1, -1)
    x = torch.cat([cls, x], dim=1) + sd["visual.positional_embedding"].to(x.dtype)
    x = _ln(x, sd["visual.ln_pre.weight"], sd["visual.ln_pre.bias"])
    hidden = [x]
    for i in range(LAYERS):
        p = f"visual.transformer.resblocks.{i}."
        h = _ln(x, sd[p + "ln_1.weight"], sd[p + "ln_1.bias"])
        x = x + _attention(h, sd[p + "attn.in_proj_weight"], sd[p + "attn.in_proj_bias"],
                           sd[p + "attn.out_proj.weight"], sd[p + "attn.out_proj.bias"])
        h = _ln(x, sd[p + "ln_2.weight"], sd[p + "ln_2.bias"])
        h = _quick_gelu(F.linear(h, sd[p + "mlp.c_fc.weight"], sd[p + "mlp.c_fc.bias"]))
        x = x + F.linear(h, sd[p + "mlp.c_proj.weight"], sd[p + "mlp.c_proj.bias"])
        hidden.append(x)
    x = _ln(x[:, 0, :], sd["visual.ln_post.weight"], sd["visual.ln_post.bias"])
    out = x @ sd["visual.proj"]
    return (out, hidden) if return_hidden else out


# ---- the tower with the engine's declared rounding --------------------------------------------------------------
# The tensors the engine (csrc/clip.cu) holds in fp16, read off its code; a reference that rounds exactly these to fp16
# and keeps everything else (residual stream, LayerNorm statistics, scores, softmax sums, biases, positional embedding)
# in float64 differs from the engine by fp32 accumulation order, intrinsic error and 1-ulp flips of those roundings.
#   weights  conv1, in_proj, out_proj, c_fc, c_proj, proj                    (upload_f16)
#   patches  the patch matrix = the transformed frames                       (clip_patchify_*_kernel)
#   ln       the outputs of ln_1, ln_2 and ln_post (ln_pre writes the fp32 stream)   (add_layernorm768_kernel)
#   qkv      q, k, v after the bias                                          (GEMM epilogue / qkv_attention_kernel staging)
#   p        the softmax probabilities before P.V: normalised at 50 tokens (attention50_kernel, attention_unit),
#            un-normalised exp(s - running max) in two key halves at 197 (attention_long_kernel, whose 1 / sum stays fp32)
#   att      the attention output before the out-projection
#   mlp      the MLP hidden layer after QuickGELU
#   y_o/y_m  the out-projection's / c_proj's result as an fp16 increment: VF_CLIP_RESID=y (both) or mix (y_o) only
# Two more names exist for the separation tests and are part of no engine path: resid (the residual stream after each
# add) and scores (q k^T / 8).
DECLARED = frozenset({"weights", "patches", "ln", "qkv", "p", "att", "mlp"})
RESID_ROUNDING = {"acc": frozenset(), "mix": frozenset({"y_o"}), "y": frozenset({"y_o", "y_m"})}
LONG_KEY_SPLIT = 112           # attention_long_kernel: 13 key tiles of 16, the first (13 + 1) / 2 = 7 in the first half


def _r16(t: torch.Tensor) -> torch.Tensor:
    return t.half().to(t.dtype)


def _rounding(declared_rounding, rounding):
    return frozenset(rounding) if rounding is not None else (DECLARED if declared_rounding else frozenset())


def _rw(w: torch.Tensor, r, dtype) -> torch.Tensor:
    w = w.to(dtype)
    return _r16(w) if "weights" in r else w


def _ln_d(x, w, b, eps):
    mu = x.mean(-1, keepdim=True)
    var = ((x - mu) ** 2).mean(-1, keepdim=True)
    return (x - mu) / torch.sqrt(var + eps) * w.to(x.dtype) + b.to(x.dtype)


def embed(sd, frames, *, dtype=torch.float64, declared_rounding=False, rounding=None, eps=LN_EPS):
    """frames (B,3,224,224) -> the residual stream after ln_pre, (B, tokens, 768)."""
    r = _rounding(declared_rounding, rounding)
    w = _rw(sd["visual.conv1.weight"], r, dtype)
    x = frames.to(dtype)
    if "patches" in r:
        x = _r16(x)
    x = F.conv2d(x, w, None, stride=w.shape[-1])
    x = x.reshape(x.shape[0], x.shape[1], -1).permute(0, 2, 1)
    cls = sd["visual.class_embedding"].to(dtype).expand(x.shape[0], 1, -1)
    x = torch.cat([cls, x], dim=1) + sd["visual.positional_embedding"].to(dtype)
    return _ln_d(x, sd["visual.ln_pre.weight"], sd["visual.ln_pre.bias"], eps)


def attention_core(qkv, *, rounding=DECLARED):
    """qkv (B,S,2304) = cat(q, k, v) after the bias -> concat_heads(softmax(q k^T / 8) v), (B,S,768), with the roundings
    named in `rounding` (qkv, scores, p, att).  More than 64 tokens: the two-half form of attention_long_kernel."""
    r = rounding
    B, S, D3 = qkv.shape
    D = D3 // 3
    hd = D // HEADS
    if "qkv" in r:
        qkv = _r16(qkv)
    q, k, v = (t.view(B, S, HEADS, hd).transpose(1, 2) for t in qkv.split(D, dim=-1))
    s = (q @ k.transpose(-1, -2)) * (hd ** -0.5)
    if "scores" in r:
        s = _r16(s)
    if S <= 64 or "p" not in r:
        p = torch.softmax(s, dim=-1)
        if "p" in r:
            p = _r16(p)
        o = p @ v
    else:
        c = LONG_KEY_SPLIT
        m1 = s[..., :c].amax(-1, keepdim=True)
        m = s.amax(-1, keepdim=True)
        e1, e2 = torch.exp(s[..., :c] - m1), torch.exp(s[..., c:] - m)
        carry = torch.exp(m1 - m)
        o = ((_r16(e1) @ v[..., :c, :]) * carry + _r16(e2) @ v[..., c:, :]) / (e1.sum(-1, keepdim=True) * carry
                                                                               + e2.sum(-1, keepdim=True))
    o = o.transpose(1, 2).reshape(B, S, D)
    return _r16(o) if "att" in r else o


def block(sd, i, x, *, declared_rounding=False, rounding=None, resid="acc", eps=LN_EPS, gelu=1.702):
    """Resblock i on the residual stream x (B, tokens, 768), in x's dtype.  ``resid``: the engine's VF_CLIP_RESID form
    (its fp16 increments are part of the declared rounding of that form)."""
    r = _rounding(declared_rounding, rounding)
    if declared_rounding and rounding is None:
        r = r | RESID_ROUNDING[resid]
    dt = x.dtype
    p = f"visual.transformer.resblocks.{i}."

    def rnd(t, name):
        return _r16(t) if name in r else t

    h = rnd(_ln_d(x, sd[p + "ln_1.weight"], sd[p + "ln_1.bias"], eps), "ln")
    qkv = F.linear(h, _rw(sd[p + "attn.in_proj_weight"], r, dt), sd[p + "attn.in_proj_bias"].to(dt))
    att = attention_core(qkv, rounding=r)
    y = F.linear(att, _rw(sd[p + "attn.out_proj.weight"], r, dt), sd[p + "attn.out_proj.bias"].to(dt))
    x = rnd(x + rnd(y, "y_o"), "resid")
    h = rnd(_ln_d(x, sd[p + "ln_2.weight"], sd[p + "ln_2.bias"], eps), "ln")
    h = F.linear(h, _rw(sd[p + "mlp.c_fc.weight"], r, dt), sd[p + "mlp.c_fc.bias"].to(dt))
    h = rnd(h * torch.sigmoid(gelu * h), "mlp")
    y = F.linear(h, _rw(sd[p + "mlp.c_proj.weight"], r, dt), sd[p + "mlp.c_proj.bias"].to(dt))
    return rnd(x + rnd(y, "y_m"), "resid")


def head(sd, x_cls, *, declared_rounding=False, rounding=None, eps=LN_EPS):
    """ln_post + projection on class-token rows x_cls (B, 768) -> (B, 512)."""
    r = _rounding(declared_rounding, rounding)
    h = _ln_d(x_cls, sd["visual.ln_post.weight"], sd["visual.ln_post.bias"], eps)
    if "ln" in r:
        h = _r16(h)
    return h @ _rw(sd["visual.proj"], r, x_cls.dtype)


@torch.no_grad()
def encode_image_declared(sd, frames, *, dtype=torch.float64, declared_rounding=True, rounding=None, resid="acc",
                          eps=LN_EPS, gelu=1.702):
    """The tower from embed / block / head (what ``encode_image(dtype=...)`` runs)."""
    kw = dict(declared_rounding=declared_rounding, rounding=rounding, eps=eps)
    x = embed(sd, frames, dtype=dtype, **kw)
    for i in range(LAYERS):
        x = block(sd, i, x, resid=resid, gelu=gelu, **kw)
    return head(sd, x[:, 0, :], **kw)


def to_hf_state_dict(sd: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
    """Remap openai ``visual.*`` keys to HF CLIPVisionModelWithProjection keys
    (SURVEY.md Appendix E) -- used only to pin this oracle against HF's code."""
    out = {}
    out["vision_model.embeddings.patch_embedding.weight"] = sd["visual.conv1.weight"]
    out["vision_model.embeddings.class_embedding"] = sd["visual.class_embedding"]
    out["vision_model.embeddings.position_embedding.weight"] = sd["visual.positional_embedding"]
    out["vision_model.pre_layrnorm.weight"] = sd["visual.ln_pre.weight"]
    out["vision_model.pre_layrnorm.bias"] = sd["visual.ln_pre.bias"]
    out["vision_model.post_layernorm.weight"] = sd["visual.ln_post.weight"]
    out["vision_model.post_layernorm.bias"] = sd["visual.ln_post.bias"]
    out["visual_projection.weight"] = sd["visual.proj"].t().contiguous()
    for i in range(LAYERS):
        p = f"visual.transformer.resblocks.{i}."
        h = f"vision_model.encoder.layers.{i}."
        wq, wk, wv = sd[p + "attn.in_proj_weight"].split(WIDTH, dim=0)
        bq, bk, bv = sd[p + "attn.in_proj_bias"].split(WIDTH, dim=0)
        for n, wt, bs in (("q", wq, bq), ("k", wk, bk), ("v", wv, bv)):
            out[h + f"self_attn.{n}_proj.weight"] = wt
            out[h + f"self_attn.{n}_proj.bias"] = bs
        out[h + "self_attn.out_proj.weight"] = sd[p + "attn.out_proj.weight"]
        out[h + "self_attn.out_proj.bias"] = sd[p + "attn.out_proj.bias"]
        out[h + "layer_norm1.weight"] = sd[p + "ln_1.weight"]
        out[h + "layer_norm1.bias"] = sd[p + "ln_1.bias"]
        out[h + "layer_norm2.weight"] = sd[p + "ln_2.weight"]
        out[h + "layer_norm2.bias"] = sd[p + "ln_2.bias"]
        out[h + "mlp.fc1.weight"] = sd[p + "mlp.c_fc.weight"]
        out[h + "mlp.fc1.bias"] = sd[p + "mlp.c_fc.bias"]
        out[h + "mlp.fc2.weight"] = sd[p + "mlp.c_proj.weight"]
        out[h + "mlp.fc2.bias"] = sd[p + "mlp.c_proj.bias"]
    return out


FLOP_PER_FRAME = 231_211_008 + 12 * 715_468_800 + 786_432   # SURVEY.md App. E (8.818 GFLOP)

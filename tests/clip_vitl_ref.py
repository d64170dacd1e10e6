"""Reference for the CLIP ViT-L/14 towers (csrc/clip_vitl.cu): openai/CLIP's ``VisionTransformer.forward`` with width,
patch, depth, heads, resolution and output width read from the state dict as ``clip.model.build_model`` does, in any
float dtype, optionally with the engine's declared fp16 rounding.

oracle/clip_tower.py fixes the ViT-B shape in module constants (12 heads in its attention, 12 layers in its tower and its
HF remap); its shape-free pieces -- ``embed``, ``head``, the LayerNorm and the fp16 rounding -- are reused here unchanged,
and the pieces that depend on the shape are restated with the shape read from the weights.

Declared rounding (``DECLARED`` of oracle/clip_tower.py): weights, patches, the ln_1 / ln_2 / ln_post outputs, q / k / v,
P, the attention output and the MLP hidden layer.  P is the streamed kernel's: with ``key_block=64`` the keys are taken
in blocks of 64 with a running max m and sum l, each block contributes fp16(exp(s - m_block)) . V, and the accumulated
output and sum are rescaled by exp(m_old - m_new) when the max grows; 1 / l is applied to the unrounded output.
"""
from __future__ import annotations

import math
import os
import sys
from typing import Dict

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import clip_tower  # noqa: E402
from oracle.clip_tower import DECLARED, LN_EPS, _ln_d, _r16, _rw  # noqa: E402

KEY_BLOCK = 64          # vitl_attention_kernel: keys per streamed block


def config(sd: Dict[str, torch.Tensor]) -> dict:
    """clip.model.build_model's inference for a ViT tower."""
    w = sd["visual.conv1.weight"]
    width, patch = int(w.shape[0]), int(w.shape[-1])
    layers = 0
    while f"visual.transformer.resblocks.{layers}.attn.in_proj_weight" in sd:
        layers += 1
    grid = round((sd["visual.positional_embedding"].shape[0] - 1) ** 0.5)
    return dict(width=width, patch=patch, layers=layers, heads=width // 64, n_px=patch * grid,
                tokens=grid * grid + 1, embed=int(sd["visual.proj"].shape[1]))


def attention_core(qkv: torch.Tensor, heads: int, *, rounding=DECLARED, key_block=KEY_BLOCK) -> torch.Tensor:
    """qkv (B, S, 3D) = cat(q, k, v) after the bias -> concat_heads(softmax(q k^T / sqrt(hd)) v), (B, S, D), with the
    roundings named in `rounding`.  With "p" rounded and key_block set, the streamed schedule of the kernel."""
    r = rounding
    B, S, D3 = qkv.shape
    D = D3 // 3
    hd = D // heads
    if "qkv" in r:
        qkv = _r16(qkv)
    q, k, v = (t.view(B, S, heads, hd).transpose(1, 2) for t in qkv.split(D, dim=-1))
    s = (q @ k.transpose(-1, -2)) * (hd ** -0.5)
    if "p" not in r or not key_block:
        p = torch.softmax(s, dim=-1)
        o = (_r16(p) if "p" in r else p) @ v
    else:
        m = torch.full(s.shape[:-1] + (1,), -math.inf, dtype=s.dtype, device=s.device)
        l = torch.zeros_like(m)
        o = torch.zeros(s.shape[:-1] + (hd,), dtype=s.dtype, device=s.device)
        for b0 in range(0, S, key_block):
            sb = s[..., b0:b0 + key_block]
            mn = torch.maximum(m, sb.amax(-1, keepdim=True))
            carry = torch.exp(m - mn)
            e = torch.exp(sb - mn)
            l = l * carry + e.sum(-1, keepdim=True)
            o = o * carry + _r16(e) @ v[..., b0:b0 + key_block, :]
            m = mn
        o = o / l
    o = o.transpose(1, 2).reshape(B, S, D)
    return _r16(o) if "att" in r else o


def block(sd, i, x, heads, *, declared_rounding=False, rounding=None, key_block=KEY_BLOCK, eps=LN_EPS):
    """Resblock i on the residual stream x (B, tokens, width), in x's dtype."""
    r = frozenset(rounding) if rounding is not None else (DECLARED if declared_rounding else frozenset())
    dt = x.dtype
    p = f"visual.transformer.resblocks.{i}."

    def rnd(t, name):
        return _r16(t) if name in r else t

    h = rnd(_ln_d(x, sd[p + "ln_1.weight"], sd[p + "ln_1.bias"], eps), "ln")
    qkv = F.linear(h, _rw(sd[p + "attn.in_proj_weight"], r, dt), sd[p + "attn.in_proj_bias"].to(dt))
    att = attention_core(qkv, heads, rounding=r, key_block=key_block)
    x = x + F.linear(att, _rw(sd[p + "attn.out_proj.weight"], r, dt), sd[p + "attn.out_proj.bias"].to(dt))
    h = rnd(_ln_d(x, sd[p + "ln_2.weight"], sd[p + "ln_2.bias"], eps), "ln")
    h = F.linear(h, _rw(sd[p + "mlp.c_fc.weight"], r, dt), sd[p + "mlp.c_fc.bias"].to(dt))
    h = rnd(h * torch.sigmoid(1.702 * h), "mlp")
    return x + F.linear(h, _rw(sd[p + "mlp.c_proj.weight"], r, dt), sd[p + "mlp.c_proj.bias"].to(dt))


def embed(sd, frames, *, dtype=torch.float64, declared_rounding=False, rounding=None):
    """frames (B, 3, n_px, n_px) -> the residual stream after ln_pre (B, tokens, width)."""
    return clip_tower.embed(sd, frames, dtype=dtype, declared_rounding=declared_rounding, rounding=rounding)


def head(sd, x_cls, *, declared_rounding=False, rounding=None):
    """ln_post + proj on class rows (B, width) -> (B, embed)."""
    return clip_tower.head(sd, x_cls, declared_rounding=declared_rounding, rounding=rounding)


@torch.no_grad()
def encode_image(sd, frames, *, dtype=torch.float32, declared_rounding=False, rounding=None, key_block=KEY_BLOCK):
    """``CLIP.encode_image``: frames (B, 3, n_px, n_px), already transformed -> (B, embed) in `dtype`.  Without
    rounding this is the fp32 (or float64) oracle; ``declared_rounding`` rounds what the engine holds in fp16."""
    cfg = config(sd)
    kw = dict(declared_rounding=declared_rounding, rounding=rounding)
    x = embed(sd, frames, dtype=dtype, **kw)
    for i in range(cfg["layers"]):
        x = block(sd, i, x, cfg["heads"], key_block=key_block, **kw)
    return head(sd, x[:, 0, :], **kw)


def to_hf_state_dict(sd: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
    """openai ``visual.*`` keys -> HF CLIPVisionModelWithProjection keys, width and depth taken from the weights."""
    cfg = config(sd)
    out = {
        "vision_model.embeddings.patch_embedding.weight": sd["visual.conv1.weight"],
        "vision_model.embeddings.class_embedding": sd["visual.class_embedding"],
        "vision_model.embeddings.position_embedding.weight": sd["visual.positional_embedding"],
        "vision_model.pre_layrnorm.weight": sd["visual.ln_pre.weight"],
        "vision_model.pre_layrnorm.bias": sd["visual.ln_pre.bias"],
        "vision_model.post_layernorm.weight": sd["visual.ln_post.weight"],
        "vision_model.post_layernorm.bias": sd["visual.ln_post.bias"],
        "visual_projection.weight": sd["visual.proj"].t().contiguous(),
    }
    for i in range(cfg["layers"]):
        p, h = f"visual.transformer.resblocks.{i}.", f"vision_model.encoder.layers.{i}."
        ws = sd[p + "attn.in_proj_weight"].split(cfg["width"], dim=0)
        bs = sd[p + "attn.in_proj_bias"].split(cfg["width"], dim=0)
        for n, wt, b in zip("qkv", ws, bs):
            out[h + f"self_attn.{n}_proj.weight"] = wt
            out[h + f"self_attn.{n}_proj.bias"] = b
        for a, b in (("attn.out_proj", "self_attn.out_proj"), ("ln_1", "layer_norm1"), ("ln_2", "layer_norm2"),
                     ("mlp.c_fc", "mlp.fc1"), ("mlp.c_proj", "mlp.fc2")):
            out[h + b + ".weight"] = sd[p + a + ".weight"]
            out[h + b + ".bias"] = sd[p + a + ".bias"]
    return out


def hf_config(sd: Dict[str, torch.Tensor]):
    """The HF CLIPVisionConfig of the tower the weights describe (quick_gelu, as openai's CLIP)."""
    import transformers
    cfg = config(sd)
    return transformers.CLIPVisionConfig(hidden_size=cfg["width"], intermediate_size=4 * cfg["width"],
                                         num_hidden_layers=cfg["layers"], num_attention_heads=cfg["heads"],
                                         patch_size=cfg["patch"], image_size=cfg["n_px"], projection_dim=cfg["embed"],
                                         hidden_act="quick_gelu")


# algorithmic GEMM FLOPs per frame (patch embedding, 24 blocks of QKV / out-proj / fc1 / fc2 on every token except the
# last block's out-proj and MLP on the class row, proj on the class row); attention adds 4 S^2 64 per head and block
def gemm_flops_per_frame(n_px: int) -> int:
    W, L, T = 1024, 24, (n_px // 14) ** 2 + 1
    patch = 2 * (T - 1) * 588 * W
    full = 2 * T * W * (3 * W + W + 4 * W + 4 * W)
    last = 2 * T * W * 3 * W + 2 * 1 * W * (W + 8 * W)
    return patch + (L - 1) * full + last + 2 * W * 768


def attention_flops_per_frame(n_px: int) -> int:
    T = (n_px // 14) ** 2 + 1
    return 24 * 16 * 4 * T * T * 64

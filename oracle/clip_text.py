"""CPU restatement of openai/CLIP's text tower (``CLIP.encode_text`` in ``clip/model.py``) -- test oracle only -- and,
below it, the same tower in float64 with the engine's declared rounding (``encode_text_declared`` and its pieces
``embed`` / ``block`` / ``pool``), what tests/test_clip_text_gpu.py holds csrc/clip_text.cu to.

``encode_text``: x = token_embedding[text] + positional_embedding; the resblocks under openai's causal mask (row i
attends to rows 0..i); ln_final; the row of the end-of-text token, found as ``text.argmax(-1)`` (the EOT id is the
largest id of the vocabulary), times ``text_projection``.  The geometry is read from the state dict as
``clip.build_model`` reads it.  Pinned against HF ``transformers.CLIPTextModelWithProjection``
(tests/test_clip_text_oracle_cpu.py).
"""
from __future__ import annotations

import math
from typing import Dict, Iterable

import torch
import torch.nn.functional as F

LN_EPS = 1e-5
HEAD_DIM = 64
GEMMS = ("qkv", "out", "fc1", "fc2", "proj")          # the five GEMMs of the tower, by weight


def config(sd: Dict[str, torch.Tensor]) -> dict:
    """clip.build_model's text geometry: width, heads, layers, context, embed, vocab."""
    width = sd["ln_final.weight"].shape[0]
    layers = len({k.split(".")[2] for k in sd if k.startswith("transformer.resblocks.")})
    return dict(width=width, heads=width // HEAD_DIM, layers=layers, context=sd["positional_embedding"].shape[0],
                embed=sd["text_projection"].shape[1], vocab=sd["token_embedding.weight"].shape[0])


def eot_positions(tokens: torch.Tensor) -> torch.Tensor:
    return torch.as_tensor(tokens).long().argmax(-1)


def _ln(x, w, b, eps=LN_EPS):
    return F.layer_norm(x, (x.shape[-1],), w.to(x.dtype), b.to(x.dtype), eps)


def _causal_attention(q, k, v, heads):
    """q, k, v: (B, L, W) -> (B, L, W); per head softmax(q k^T / 8 + causal mask) v."""
    B, L, W = q.shape
    sh = lambda t: t.view(B, L, heads, HEAD_DIM).transpose(1, 2)
    s = sh(q) @ sh(k).transpose(-1, -2) / math.sqrt(HEAD_DIM)
    mask = torch.ones(L, L, dtype=torch.bool).triu(1)
    s = s.masked_fill(mask, float("-inf"))
    return (s.softmax(-1) @ sh(v)).transpose(1, 2).reshape(B, L, W)


def encode_text(sd: Dict[str, torch.Tensor], tokens, *, dtype=torch.float32) -> torch.Tensor:
    """tokens (B, context) ids -> (B, embed) text features (not normalised), in ``dtype``."""
    cfg = config(sd)
    g = lambda k: sd[k].to(dtype)
    tokens = torch.as_tensor(tokens).long()
    x = g("token_embedding.weight")[tokens] + g("positional_embedding")[: tokens.shape[1]]
    for i in range(cfg["layers"]):
        p = f"transformer.resblocks.{i}."
        h = _ln(x, g(p + "ln_1.weight"), g(p + "ln_1.bias"))
        q, k, v = F.linear(h, g(p + "attn.in_proj_weight"), g(p + "attn.in_proj_bias")).chunk(3, -1)
        x = x + F.linear(_causal_attention(q, k, v, cfg["heads"]), g(p + "attn.out_proj.weight"),
                         g(p + "attn.out_proj.bias"))
        h = _ln(x, g(p + "ln_2.weight"), g(p + "ln_2.bias"))
        h = F.linear(h, g(p + "mlp.c_fc.weight"), g(p + "mlp.c_fc.bias"))
        x = x + F.linear(h * torch.sigmoid(1.702 * h), g(p + "mlp.c_proj.weight"), g(p + "mlp.c_proj.bias"))
    x = _ln(x, g("ln_final.weight"), g("ln_final.bias"))
    return x[torch.arange(x.shape[0]), eot_positions(tokens)] @ g("text_projection")


def to_hf_state_dict(sd: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
    """openai text keys -> ``CLIPTextModelWithProjection`` keys."""
    cfg = config(sd)
    out = {"text_model.embeddings.token_embedding.weight": sd["token_embedding.weight"],
           "text_model.embeddings.position_embedding.weight": sd["positional_embedding"],
           "text_model.final_layer_norm.weight": sd["ln_final.weight"],
           "text_model.final_layer_norm.bias": sd["ln_final.bias"],
           "text_projection.weight": sd["text_projection"].t().contiguous()}
    W = cfg["width"]
    for i in range(cfg["layers"]):
        p, q = f"transformer.resblocks.{i}.", f"text_model.encoder.layers.{i}."
        for j, n in enumerate("qkv"):
            out[q + f"self_attn.{n}_proj.weight"] = sd[p + "attn.in_proj_weight"][j * W:(j + 1) * W]
            out[q + f"self_attn.{n}_proj.bias"] = sd[p + "attn.in_proj_bias"][j * W:(j + 1) * W]
        for a, b in (("attn.out_proj", "self_attn.out_proj"), ("ln_1", "layer_norm1"), ("ln_2", "layer_norm2"),
                     ("mlp.c_fc", "mlp.fc1"), ("mlp.c_proj", "mlp.fc2")):
            out[q + b + ".weight"] = sd[p + a + ".weight"]
            out[q + b + ".bias"] = sd[p + a + ".bias"]
    return out


# ---------------------------------------------------------------- float64 with the declared rounding
#
# The engine's rounding (DESIGN §2, §4.16): every GEMM weight a split-fp16 pair (hi + lo: to float64 within 2^-22
# relative, taken as exact here); rounded to one fp16 value are the LayerNorm outputs (ln_1, ln_2, ln_final), q / k / v,
# the attention output and the fc1 output after QuickGELU.  The residual stream, the scores, softmax and P.V stay fp32
# (exact here).  ``fp16_weights`` names GEMMs whose weights are single fp16 values instead, and ``act=False`` leaves the
# activations unrounded: the knobs scripts/precision/emulate_clip_text.py turns.

def _r16(t: torch.Tensor) -> torch.Tensor:
    return t.to(torch.float16).to(t.dtype)


class Rounding:
    def __init__(self, act: bool = True, fp16_weights: Iterable[str] = ()):
        self.act, self.w16 = act, frozenset(fp16_weights)
        assert self.w16 <= set(GEMMS), self.w16

    def a(self, t):
        return _r16(t) if self.act else t

    def w(self, name, t):
        return _r16(t) if name in self.w16 else t


DECLARED = Rounding()


def _g(sd, k, dtype=torch.float64):
    return sd[k].to(dtype)


def embed(sd, tokens, L=None, *, dtype=torch.float64) -> torch.Tensor:
    """The residual stream entering block 0: (B, L, W) rows token_embedding[id] + positional_embedding."""
    tokens = torch.as_tensor(tokens).long()
    L = tokens.shape[1] if L is None else L
    return _g(sd, "token_embedding.weight", dtype)[tokens[:, :L]] + _g(sd, "positional_embedding", dtype)[:L]


def block(sd, i, x, *, rounding: Rounding = DECLARED) -> torch.Tensor:
    """Residual block i on the stream x (B, L, W) under causal attention."""
    r, p, dt = rounding, f"transformer.resblocks.{i}.", x.dtype
    heads = x.shape[-1] // HEAD_DIM
    h = r.a(_ln(x, _g(sd, p + "ln_1.weight", dt), _g(sd, p + "ln_1.bias", dt)))
    qkv = r.a(F.linear(h, r.w("qkv", _g(sd, p + "attn.in_proj_weight", dt)), _g(sd, p + "attn.in_proj_bias", dt)))
    att = r.a(_causal_attention(*qkv.chunk(3, -1), heads))
    x = x + F.linear(att, r.w("out", _g(sd, p + "attn.out_proj.weight", dt)), _g(sd, p + "attn.out_proj.bias", dt))
    h = r.a(_ln(x, _g(sd, p + "ln_2.weight", dt), _g(sd, p + "ln_2.bias", dt)))
    h = F.linear(h, r.w("fc1", _g(sd, p + "mlp.c_fc.weight", dt)), _g(sd, p + "mlp.c_fc.bias", dt))
    h = r.a(h * torch.sigmoid(1.702 * h))
    return x + F.linear(h, r.w("fc2", _g(sd, p + "mlp.c_proj.weight", dt)), _g(sd, p + "mlp.c_proj.bias", dt))


def pool(sd, x, tokens, *, rounding: Rounding = DECLARED) -> torch.Tensor:
    """The EOT row of each prompt through ln_final and text_projection, L2-normalised: (B, embed)."""
    r, dt = rounding, x.dtype
    rows = x[torch.arange(x.shape[0]), eot_positions(tokens)]
    h = r.a(_ln(rows, _g(sd, "ln_final.weight", dt), _g(sd, "ln_final.bias", dt)))
    t = h @ r.w("proj", _g(sd, "text_projection", dt))
    return t / t.norm(dim=-1, keepdim=True)


def encode_text_declared(sd, tokens, *, rounding: Rounding = DECLARED, dtype=torch.float64, taps: bool = False):
    """The whole tower on L = 1 + max EOT position rows: normalised (B, embed) features, and with ``taps`` also the
    stream after the embedding and after every block."""
    tokens = torch.as_tensor(tokens).long()
    L = int(eot_positions(tokens).max()) + 1
    x = embed(sd, tokens, L, dtype=dtype)
    streams = [x]
    for i in range(config(sd)["layers"]):
        x = block(sd, i, x, rounding=rounding)
        streams.append(x)
    t = pool(sd, x, tokens, rounding=rounding)
    return (t, streams) if taps else t


def zero_shot_logits(sd, image_feats: torch.Tensor, text_feats: torch.Tensor) -> torch.Tensor:
    """CLIP's logits_per_image: exp(logit_scale) * normalised image . normalised text (float64)."""
    im = image_feats.double()
    im = im / im.norm(dim=-1, keepdim=True)
    return math.exp(float(sd["logit_scale"])) * im @ text_feats.double().t()

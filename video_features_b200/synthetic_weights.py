"""Seeded synthetic weights in the layouts the engines load -- for benchmarks and tests on machines without the real
checkpoints (the reference downloads ViT-B-32.pt at run time, models/CLIP/extract_clip.py:47; there is no network
here).  ``VF_CLIP_SYNTHETIC=<seed>[:outliers]`` makes ``ExtractCLIP`` use them instead of a checkpoint file.
"""
from __future__ import annotations

import math
from collections import OrderedDict

import torch

WIDTH, LAYERS, TOKENS, PATCH, MLP, EMBED = 768, 12, 50, 32, 3072, 512


def clip_vit_b16_state_dict(seed: int = 0, outliers: bool = False) -> "OrderedDict[str, torch.Tensor]":
    """The same for the ViT-B/16 tower (16-pixel patches, 197 tokens)."""
    return clip_vit_b32_state_dict(seed, outliers, patch=16)


def clip_vit_b32_state_dict(seed: int = 0, outliers: bool = False, patch: int = PATCH) -> "OrderedDict[str, torch.Tensor]":
    """openai ``visual.*`` key layout, fp32 (see ``_vit_state_dict``)."""
    return _vit_state_dict(seed, outliers, WIDTH, LAYERS, patch, 224, EMBED)


def clip_vit_l14_state_dict(seed: int = 0, outliers: bool = False, n_px: int = 224) -> "OrderedDict[str, torch.Tensor]":
    """The same scheme at the ViT-L/14 shape: width 1024, 24 blocks, patch 14, ``n_px`` 224 (257 tokens) or 336 (577
    tokens), output 768."""
    return _vit_state_dict(seed, outliers, 1024, 24, 14, n_px, 768)


def _vit_state_dict(seed, outliers, WIDTH, LAYERS, patch, n_px, EMBED) -> "OrderedDict[str, torch.Tensor]":
    """openai ``visual.*`` key layout, fp32.  Initialisation scales are the ones openai/CLIP's
    ``initialize_parameters`` uses (width**-0.5 etc.), with perturbed LayerNorm gains / biases so that every term of the
    forward matters.

    ``outliers=True`` adds what trained ViT weights have and random ones lack: a handful of residual-stream
    channels that carry magnitudes of 50-200 through every block (set up by the positional embedding and fed by the
    projection biases), LayerNorm gains with a heavy tail (a few entries near 0.05, a few above 4), and a few large
    rows in the attention / MLP output projections.  This is the regime where fp16 storage of intermediate tensors is
    most at risk."""
    g = torch.Generator().manual_seed(seed)

    def rn(*shape, std=1.0):
        return torch.randn(*shape, generator=g, dtype=torch.float32) * std

    scale = WIDTH ** -0.5
    attn_std = WIDTH ** -0.5
    proj_std = (WIDTH ** -0.5) * ((2 * LAYERS) ** -0.5)
    fc_std = (2 * WIDTH) ** -0.5
    sd: "OrderedDict[str, torch.Tensor]" = OrderedDict()
    sd["visual.class_embedding"] = rn(WIDTH, std=scale)
    sd["visual.positional_embedding"] = rn((n_px // patch) ** 2 + 1, WIDTH, std=scale)
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
        sd[p + "mlp.c_fc.weight"] = rn(4 * WIDTH, WIDTH, std=fc_std)
        sd[p + "mlp.c_fc.bias"] = rn(4 * WIDTH, std=0.02)
        sd[p + "mlp.c_proj.weight"] = rn(WIDTH, 4 * WIDTH, std=proj_std)
        sd[p + "mlp.c_proj.bias"] = rn(WIDTH, std=0.02)
        sd[p + "ln_2.weight"] = 1.0 + rn(WIDTH, std=0.1)
        sd[p + "ln_2.bias"] = rn(WIDTH, std=0.05)
    if outliers:
        dims = torch.randperm(WIDTH, generator=g)[:6]
        sign = torch.tensor([1.0, -1.0, 1.0, -1.0, 1.0, -1.0])
        # ln_pre rescales whatever the embedding holds, so the outlier channels are planted in ln_pre's affine part:
        # the residual stream leaves ln_pre with +-(60..150) in these channels
        sd["visual.ln_pre.bias"][dims] = sign * (60.0 + 90.0 * torch.rand(6, generator=g))
        sd["visual.ln_pre.weight"][dims] = 8.0
        for i in range(LAYERS):
            p = f"visual.transformer.resblocks.{i}."
            for ln in ("ln_1", "ln_2"):
                w = sd[p + ln + ".weight"]
                w.mul_(torch.exp(rn(WIDTH, std=0.35)))                       # heavy-tailed gains
                w[dims[:3]] = 0.05 + 0.05 * torch.rand(3, generator=g)       # trained nets damp their outlier channels ...
                w[dims[3:]] = 3.0 + 2.0 * torch.rand(3, generator=g)         # ... or read them loudly
                sd[p + ln + ".bias"][dims] = rn(6, std=0.5)
            # the projections keep feeding the outlier channels (bias) and have a few loud rows
            sd[p + "attn.out_proj.bias"][dims] = sign * (1.0 + 2.0 * torch.rand(6, generator=g))
            sd[p + "mlp.c_proj.bias"][dims] = sign * (2.0 + 4.0 * torch.rand(6, generator=g))
            loud = torch.randperm(WIDTH, generator=g)[:4]
            sd[p + "attn.out_proj.weight"][loud] *= 6.0
            sd[p + "mlp.c_proj.weight"][loud] *= 6.0
        sd["visual.ln_post.weight"][dims] = 0.05
    return sd


def clip_text_state_dict(seed: int = 0, width: int = 512, embed: int = 512, vocab_size: int = 49408,
                         layers: int = LAYERS, context: int = 77) -> "OrderedDict[str, torch.Tensor]":
    """openai's text-tower keys (``token_embedding``, ``positional_embedding``, ``transformer.*``, ``ln_final``,
    ``text_projection``, ``logit_scale`` = ln 100), fp32, for ``--show_pred`` without a checkpoint.  ``vocab_size``
    must be the size of the BPE vocabulary the prompts are tokenized with.  Scales as openai's
    ``initialize_parameters``, with perturbed LayerNorms as ``_vit_state_dict``."""
    g = torch.Generator().manual_seed(seed + 1000)

    def rn(*shape, std=1.0):
        return torch.randn(*shape, generator=g, dtype=torch.float32) * std

    proj_std = (width ** -0.5) * ((2 * layers) ** -0.5)
    sd: "OrderedDict[str, torch.Tensor]" = OrderedDict()
    sd["token_embedding.weight"] = rn(vocab_size, width, std=0.02)
    sd["positional_embedding"] = rn(context, width, std=0.01)
    for i in range(layers):
        p = f"transformer.resblocks.{i}."
        sd[p + "attn.in_proj_weight"] = rn(3 * width, width, std=width ** -0.5)
        sd[p + "attn.in_proj_bias"] = rn(3 * width, std=0.02)
        sd[p + "attn.out_proj.weight"] = rn(width, width, std=proj_std)
        sd[p + "attn.out_proj.bias"] = rn(width, std=0.02)
        sd[p + "ln_1.weight"] = 1.0 + rn(width, std=0.1)
        sd[p + "ln_1.bias"] = rn(width, std=0.05)
        sd[p + "mlp.c_fc.weight"] = rn(4 * width, width, std=(2 * width) ** -0.5)
        sd[p + "mlp.c_fc.bias"] = rn(4 * width, std=0.02)
        sd[p + "mlp.c_proj.weight"] = rn(width, 4 * width, std=proj_std)
        sd[p + "mlp.c_proj.bias"] = rn(width, std=0.02)
        sd[p + "ln_2.weight"] = 1.0 + rn(width, std=0.1)
        sd[p + "ln_2.bias"] = rn(width, std=0.05)
    sd["ln_final.weight"] = 1.0 + rn(width, std=0.1)
    sd["ln_final.bias"] = rn(width, std=0.05)
    sd["text_projection"] = rn(width, embed, std=width ** -0.5)
    sd["logit_scale"] = torch.tensor(math.log(100.0))
    return sd


def parse_env(value: str):
    """``VF_CLIP_SYNTHETIC`` value -> (seed, outliers): "3", "3:outliers", "" (seed 0)."""
    head, _, tail = (value or "").partition(":")
    return int(head or 0), tail.strip().lower() == "outliers"

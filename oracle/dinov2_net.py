"""Plain-torch restatement of DINOv2's frame feature: ``torch.hub.load('facebookresearch/dinov2', name)(x)``, the class
token after the final ``norm``, for the four hub ViTs (S/14, B/14, L/14, g/14) with and without registers, at 224 px;
the hub's eval transform; the positional table the hub interpolates for 224 px; seeded stand-ins for the hub
checkpoints (they cannot be fetched offline).

Also the float64 forward with the engine's declared rounding (csrc/dinov2.cu): each tensor class in ``fp16`` is rounded
to one fp16 value where the engine rounds it, and LayerScale is folded into the GEMM epilogue as the engine folds it
(scale gamma, bias fp32(gamma * b)).  ``pos_table_224`` is the restatement the engine wrapper's own table
(video_features_b200/dinov2_engine.py) is tested equal to.
"""
import functools
import math

import numpy as np
import torch
import torch.nn.functional as F

IMAGENET_MEAN = [0.485, 0.456, 0.406]
IMAGENET_STD = [0.229, 0.224, 0.225]
RESIZE = 256
CROP = 224
PATCH = 14
GRID = CROP // PATCH                  # 16 x 16 patches at 224 px
HUB_GRID = 37                          # the checkpoints' 37 x 37 positional grid (518 px)
TOKENS = 1 + GRID * GRID               # 257, plus the registers
N_REG = 4
EPS = 1e-6
HEAD_DIM = 64
SWIGLU_HIDDEN = 4096                   # ViT-g/14's SwiGLUFFNFused: int(6144 * 2 / 3) rounded to a multiple of 8
INTERPOLATE_OFFSET = 0.1               # the plain hub models' interpolate_offset (the _reg models use 0)
# hub name -> (width, depth, feed-forward kind)
SHAPES = {"dinov2_vits14": (384, 12, "mlp"), "dinov2_vitb14": (768, 12, "mlp"), "dinov2_vitl14": (1024, 24, "mlp"),
          "dinov2_vitg14": (1536, 40, "swiglu")}
MODELS = tuple(SHAPES) + tuple(n + "_reg" for n in SHAPES)
# the engine's tensor classes (scripts/precision/emulate_dinov2.py): w weights, patch the patch rows, ln the outputs of
# norm1 / norm2, qkv q / k / v, p the softmax numerator P per 64-key block, att the attention output, hidden the FFN
# hidden layer (fc2 / w3's input), swiglu the w12 output (a, b) that the SwiGLU kernel reads
CLASSES = ("w", "patch", "ln", "qkv", "p", "att", "hidden", "swiglu")
KEY_BLOCK = 64                         # vitl_attention_kernel: keys per streamed block


def shape_of(name: str):
    """(width, depth, ffn kind, registers) of a feature type."""
    reg = name.endswith("_reg")
    d, depth, ffn = SHAPES[name[:-4] if reg else name]
    return d, depth, ffn, reg


def _plain(sd):
    if not any(k.startswith("module.") for k in sd):
        return sd
    return {k[7:] if k.startswith("module.") else k: v for k, v in sd.items()}


def config(sd):
    """(width, depth, heads, ffn kind, registers) from the weights, as vf_dinov2_create infers them."""
    sd = _plain(sd)
    d = sd["cls_token"].shape[-1]
    depth = 0
    while f"blocks.{depth}.norm1.weight" in sd:
        depth += 1
    ffn = "swiglu" if "blocks.0.mlp.w12.weight" in sd else "mlp"
    return d, depth, d // HEAD_DIM, ffn, "register_tokens" in sd


def pos_table_224(pos_embed: torch.Tensor, registers: bool) -> torch.Tensor:
    """The hub's ``interpolate_pos_encoding`` for a 224 x 224 input, in fp32 on the host: (1, 1 + 37 * 37, D) ->
    (257, D).  The plain models scale by (16 + 0.1) / 37 without antialiasing; the _reg models ask for size (16, 16)
    with antialiasing.  Row 0 (the class position) is kept as it is."""
    pe = pos_embed.detach().to("cpu", torch.float32).reshape(1, -1, pos_embed.shape[-1])
    d = pe.shape[-1]
    if pe.shape[1] != 1 + HUB_GRID * HUB_GRID:
        raise ValueError(f"pos_embed has {pe.shape[1]} rows, not 1 + 37 x 37")
    grid = pe[:, 1:].reshape(1, HUB_GRID, HUB_GRID, d).permute(0, 3, 1, 2)
    if registers:
        grid = F.interpolate(grid, mode="bicubic", antialias=True, size=(GRID, GRID))
    else:
        s = (GRID + INTERPOLATE_OFFSET) / HUB_GRID
        grid = F.interpolate(grid, mode="bicubic", antialias=False, scale_factor=(s, s))
    assert tuple(grid.shape[-2:]) == (GRID, GRID), grid.shape
    return torch.cat([pe[0, :1], grid.permute(0, 2, 3, 1).reshape(GRID * GRID, d)]).contiguous()


# ---- transform
def transform(rgb_u8) -> torch.Tensor:
    """(H, W, 3) uint8 RGB -> (3, 224, 224) fp32: Resize(256, BICUBIC) on the PIL image, CenterCrop(224), ToTensor,
    Normalize (ImageNet), as the hub's eval preset, with Pillow doing the resize."""
    from PIL import Image
    img = Image.fromarray(np.ascontiguousarray(rgb_u8))
    w, h = img.size
    short, long = (w, h) if w <= h else (h, w)
    nl = int(RESIZE * long / short)
    size = (RESIZE, nl) if w <= h else (nl, RESIZE)
    if size != (w, h):
        img = img.resize(size, Image.BICUBIC)
    a = np.asarray(img)
    i, j = int(round((a.shape[0] - CROP) / 2.0)), int(round((a.shape[1] - CROP) / 2.0))
    x = torch.from_numpy(a[i:i + CROP, j:j + CROP].copy()).permute(2, 0, 1).to(torch.float32) / 255
    return (x - torch.tensor(IMAGENET_MEAN).view(3, 1, 1)) / torch.tensor(IMAGENET_STD).view(3, 1, 1)


def transform_torchvision(rgb_u8) -> torch.Tensor:
    """The preset itself (torchvision on a PIL image)."""
    import torchvision.transforms as T
    from PIL import Image
    tf = T.Compose([T.Resize(RESIZE, interpolation=T.InterpolationMode.BICUBIC), T.CenterCrop(CROP), T.ToTensor(),
                    T.Normalize(mean=IMAGENET_MEAN, std=IMAGENET_STD)])
    return tf(Image.fromarray(np.ascontiguousarray(rgb_u8)))


# ---- forward
def _r16(x):
    return x.to(torch.float16).to(x.dtype)


def _q(x, cls, fp16):
    return _r16(x) if cls in fp16 else x


def _attention(qkv, heads, fp16):
    """softmax(q k^T / 8) v per head on qkv (B, S, 3D); with "p" rounded, the kernel's streamed schedule: per 64-key
    block fp16(exp(s - running max)) . V, rescaled as the max grows, 1 / sum applied to the unrounded output."""
    B, S, D3 = qkv.shape
    D = D3 // 3
    q, k, v = (t.view(B, S, heads, HEAD_DIM).transpose(1, 2) for t in qkv.split(D, dim=-1))
    s = (q @ k.transpose(-1, -2)) * 0.125
    if "p" not in fp16:
        o = torch.softmax(s, dim=-1) @ v
    else:
        m = torch.full(s.shape[:-1] + (1,), -math.inf, dtype=s.dtype, device=s.device)
        l = torch.zeros_like(m)
        o = torch.zeros(s.shape[:-1] + (HEAD_DIM,), dtype=s.dtype, device=s.device)
        for b0 in range(0, S, KEY_BLOCK):
            sb = s[..., b0:b0 + KEY_BLOCK]
            mn = torch.maximum(m, sb.amax(-1, keepdim=True))
            carry = torch.exp(m - mn)
            e = torch.exp(sb - mn)
            l = l * carry + e.sum(-1, keepdim=True)
            o = o * carry + _r16(e) @ v[..., b0:b0 + KEY_BLOCK, :]
            m = mn
        o = o / l
    return o.transpose(1, 2).reshape(B, S, D)


def _ln(sd, p, x):
    return F.layer_norm(x, x.shape[-1:], sd[p + ".weight"], sd[p + ".bias"], EPS)


def _ls_linear(sd, p, gamma, x, fp16, fold):
    """gamma * (x W^T + b): with ``fold`` as the engine's epilogue, acc * gamma + fp32(gamma * b)."""
    w = _q(sd[p + ".weight"], "w", fp16)
    g = sd[gamma]
    if fold:
        bias = (sd[gamma].float() * sd[p + ".bias"].float()).to(x.dtype)
        return (x @ w.T) * g + bias
    return g * F.linear(x, w, sd[p + ".bias"])


def _ffn(sd, p, x, ffn, fp16, fold):
    if ffn == "mlp":
        h = F.gelu(F.linear(x, _q(sd[p + ".mlp.fc1.weight"], "w", fp16), sd[p + ".mlp.fc1.bias"]))
        return _ls_linear(sd, p + ".mlp.fc2", p + ".ls2.gamma", _q(h, "hidden", fp16), fp16, fold)
    ab = F.linear(x, _q(sd[p + ".mlp.w12.weight"], "w", fp16), sd[p + ".mlp.w12.bias"])
    if fold:
        ab = ab.float().to(x.dtype)            # the w12 GEMM writes fp32
    a, b = _q(ab, "swiglu", fp16).chunk(2, dim=-1)
    return _ls_linear(sd, p + ".mlp.w3", p + ".ls2.gamma", _q(F.silu(a) * b, "hidden", fp16), fp16, fold)


def prepare(sd, dtype=torch.float64, device="cpu"):
    """The state dict in ``dtype`` on ``device`` without a "module." prefix, with "pos_224" (the 257-row table)."""
    sd = _plain(sd)
    out = {k: v.to(device, dtype) for k, v in sd.items() if torch.is_tensor(v) and v.is_floating_point()}
    out["pos_224"] = pos_table_224(sd["pos_embed"], "register_tokens" in sd).to(device, dtype)
    return out


def patch_rows(x):
    """(B, 3, 224, 224) -> (B, 256, 588) patch rows, column c * 196 + ky * 14 + kx (the conv weight's flattening)."""
    B = x.shape[0]
    return x.reshape(B, 3, GRID, PATCH, GRID, PATCH).permute(0, 2, 4, 1, 3, 5).reshape(B, GRID * GRID, 3 * PATCH * PATCH)


def embed(sd, x, fp16=()):
    """Normalised frames (B, 3, 224, 224) -> the residual stream before block 0 (B, tokens, D).  ``sd`` from prepare()."""
    d = sd["cls_token"].shape[-1]
    w = _q(sd["patch_embed.proj.weight"].reshape(d, -1), "w", fp16)
    emb = _q(patch_rows(x), "patch", fp16) @ w.T + sd["patch_embed.proj.bias"]
    pos = sd["pos_224"]
    B = x.shape[0]
    rows = [(sd["cls_token"].reshape(1, 1, d) + pos[:1]).expand(B, 1, d)]
    if "register_tokens" in sd:
        rows.append(sd["register_tokens"].reshape(1, -1, d).expand(B, -1, d))
    rows.append(emb + pos[1:])
    return torch.cat(rows, dim=1)


def block(sd, i, x, fp16=(), fold=False, last=False):
    """Block i on x (B, tokens, D); ``last``: the out-projection and the FFN on the class rows only (the rest of x is
    left as it was)."""
    d = x.shape[-1]
    heads, ffn = d // HEAD_DIM, ("swiglu" if f"blocks.{i}.mlp.w12.weight" in sd else "mlp")
    p = f"blocks.{i}"
    h = _q(_ln(sd, p + ".norm1", x), "ln", fp16)
    qkv = _q(F.linear(h, _q(sd[p + ".attn.qkv.weight"], "w", fp16), sd[p + ".attn.qkv.bias"]), "qkv", fp16)
    att = _q(_attention(qkv, heads, fp16), "att", fp16)
    if last:
        x = x.clone()
        c = x[:, :1] + _ls_linear(sd, p + ".attn.proj", p + ".ls1.gamma", att[:, :1], fp16, fold)
        c = c + _ffn(sd, p, _q(_ln(sd, p + ".norm2", c), "ln", fp16), ffn, fp16, fold)
        x[:, :1] = c
        return x
    x = x + _ls_linear(sd, p + ".attn.proj", p + ".ls1.gamma", att, fp16, fold)
    return x + _ffn(sd, p, _q(_ln(sd, p + ".norm2", x), "ln", fp16), ffn, fp16, fold)


def head(sd, x):
    """The final norm of the class rows of x (B, tokens, D) -> (B, D)."""
    return _ln(sd, "norm", x[:, 0])


def forward(sd, x, fp16=(), fold=False, taps=None):
    """Features (B, D) of normalised frames x (B, 3, 224, 224) in x's dtype.  ``sd`` from prepare().  ``fp16``: the
    tensor classes rounded to one fp16 value; ``fold``: LayerScale folded as the engine's epilogue does.  ``taps``: a
    dict that receives "embed" and "block{i}" (the stream after block i)."""
    y = embed(sd, x, fp16)
    if taps is not None:
        taps["embed"] = y
    depth = config(sd)[1]
    for i in range(depth):
        y = block(sd, i, y, fp16, fold, last=i == depth - 1)
        if taps is not None:
            taps[f"block{i}"] = y
    return head(sd, y)


# the engine's declared rounding: weights are split-fp16 pairs (exact to ~2^-22), the SwiGLU inputs fp32; every other
# class one fp16 value (scripts/precision/emulate_dinov2.py decides this)
ENGINE_FP16 = ("patch", "ln", "qkv", "p", "att", "hidden")


def forward_engine(sd, x, taps=None):
    """The float64 forward of the engine's declared rounding."""
    return forward(sd, x, ENGINE_FP16, True, taps)


# ---- HF cross-check
def to_hf_state_dict(sd):
    """The hub keys -> HF ``Dinov2Model`` / ``Dinov2WithRegistersModel`` keys (position_embeddings left out: the test
    sets them to the 257-row table so that HF does not interpolate)."""
    sd = _plain(sd)
    d, depth, _, ffn, reg = config(sd)
    out = {"embeddings.cls_token": sd["cls_token"], "embeddings.mask_token": sd.get("mask_token", torch.zeros(1, d)),
           "embeddings.patch_embeddings.projection.weight": sd["patch_embed.proj.weight"],
           "embeddings.patch_embeddings.projection.bias": sd["patch_embed.proj.bias"],
           "layernorm.weight": sd["norm.weight"], "layernorm.bias": sd["norm.bias"]}
    if reg:
        out["embeddings.register_tokens"] = sd["register_tokens"]
    for i in range(depth):
        p, q = f"blocks.{i}.", f"encoder.layer.{i}."
        for n in ("weight", "bias"):
            out[q + "norm1." + n] = sd[p + "norm1." + n]
            out[q + "norm2." + n] = sd[p + "norm2." + n]
            wq, wk, wv = sd[p + "attn.qkv." + n].chunk(3, dim=0)
            out[q + "attention.attention.query." + n] = wq
            out[q + "attention.attention.key." + n] = wk
            out[q + "attention.attention.value." + n] = wv
            out[q + "attention.output.dense." + n] = sd[p + "attn.proj." + n]
            if ffn == "mlp":
                out[q + "mlp.fc1." + n] = sd[p + "mlp.fc1." + n]
                out[q + "mlp.fc2." + n] = sd[p + "mlp.fc2." + n]
            else:
                out[q + "mlp.weights_in." + n] = sd[p + "mlp.w12." + n]
                out[q + "mlp.weights_out." + n] = sd[p + "mlp.w3." + n]
        out[q + "layer_scale1.lambda1"] = sd[p + "ls1.gamma"]
        out[q + "layer_scale2.lambda1"] = sd[p + "ls2.gamma"]
    return out


def hf_model(sd):
    """HF's implementation loaded with ``sd`` (fp32, eval), its position embeddings the 257-row 224-px table."""
    from transformers import Dinov2Config, Dinov2Model, Dinov2WithRegistersConfig, Dinov2WithRegistersModel
    sd = _plain(sd)
    d, depth, heads, ffn, reg = config(sd)
    kw = dict(hidden_size=d, num_hidden_layers=depth, num_attention_heads=heads, mlp_ratio=4, image_size=224,
              patch_size=PATCH, layer_norm_eps=EPS, use_swiglu_ffn=ffn == "swiglu", hidden_act="gelu",
              layerscale_value=1.0, attention_probs_dropout_prob=0.0, hidden_dropout_prob=0.0)
    if reg:
        model = Dinov2WithRegistersModel(Dinov2WithRegistersConfig(num_register_tokens=N_REG, **kw))
    else:
        model = Dinov2Model(Dinov2Config(**kw))
    hsd = {k: v.float() for k, v in to_hf_state_dict(sd).items()}
    hsd["embeddings.position_embeddings"] = pos_table_224(sd["pos_embed"], reg)[None]
    missing, unexpected = model.load_state_dict(hsd, strict=False)
    assert not unexpected and not missing, (missing, unexpected)
    return model.eval()


# ---- stand-ins
def _stand_in(name, seed, depth):
    d, full_depth, ffn, reg = shape_of(name)
    depth = full_depth if depth is None else depth
    g = torch.Generator().manual_seed(9100 + 17 * MODELS.index(name) + seed)

    def rn(*shape, std=1.0):
        return torch.randn(*shape, generator=g) * std

    def ru(*shape, lo, hi):
        return lo + (hi - lo) * torch.rand(*shape, generator=g)

    def ls(n):                            # trained LayerScale gains: mostly 0.05 .. 0.8, log-normal
        return torch.exp(rn(n, std=0.6) + math.log(0.2))

    sd = {"cls_token": rn(1, 1, d, std=0.5), "mask_token": torch.zeros(1, d),
          "patch_embed.proj.weight": rn(d, 3, PATCH, PATCH, std=(3 * PATCH * PATCH) ** -0.5),
          "patch_embed.proj.bias": rn(d, std=0.1)}
    # a smooth positional field plus noise; for the plain models, a few cells carry a large offset, so that a few
    # patch tokens have the high norm of the artifact tokens registers exist to remove
    low = rn(1, d, 6, 6, std=0.3)
    pos = F.interpolate(low, size=(HUB_GRID, HUB_GRID), mode="bicubic", align_corners=False) + rn(1, d, HUB_GRID, HUB_GRID, std=0.05)
    if not reg:
        for cy, cx in ((5, 7), (12, 30), (24, 18), (31, 4)):
            pos[0, :, cy - 1:cy + 2, cx - 1:cx + 2] += rn(d, 1, 1, std=3.0)
    pos = pos.permute(0, 2, 3, 1).reshape(1, HUB_GRID * HUB_GRID, d)
    sd["pos_embed"] = torch.cat([rn(1, 1, d, std=0.1), pos], dim=1)
    if reg:
        sd["register_tokens"] = rn(1, N_REG, d, std=0.5)
    for i in range(depth):
        p = f"blocks.{i}."
        sd[p + "norm1.weight"] = ru(d, lo=0.5, hi=1.5)
        sd[p + "norm1.bias"] = rn(d, std=0.1)
        sd[p + "attn.qkv.weight"] = rn(3 * d, d, std=d ** -0.5)
        sd[p + "attn.qkv.bias"] = rn(3 * d, std=0.1)
        sd[p + "attn.proj.weight"] = rn(d, d, std=d ** -0.5)
        sd[p + "attn.proj.bias"] = rn(d, std=0.1)
        sd[p + "ls1.gamma"] = ls(d)
        sd[p + "norm2.weight"] = ru(d, lo=0.5, hi=1.5)
        sd[p + "norm2.bias"] = rn(d, std=0.1)
        if ffn == "mlp":
            sd[p + "mlp.fc1.weight"] = rn(4 * d, d, std=d ** -0.5)
            sd[p + "mlp.fc1.bias"] = rn(4 * d, std=0.1)
            sd[p + "mlp.fc2.weight"] = rn(d, 4 * d, std=(4 * d) ** -0.5)
            sd[p + "mlp.fc2.bias"] = rn(d, std=0.1)
        else:
            sd[p + "mlp.w12.weight"] = rn(2 * SWIGLU_HIDDEN, d, std=d ** -0.5)
            sd[p + "mlp.w12.bias"] = rn(2 * SWIGLU_HIDDEN, std=0.1)
            sd[p + "mlp.w3.weight"] = rn(d, SWIGLU_HIDDEN, std=SWIGLU_HIDDEN ** -0.5)
            sd[p + "mlp.w3.bias"] = rn(d, std=0.1)
        sd[p + "ls2.gamma"] = ls(d)
    sd["norm.weight"] = ru(d, lo=0.5, hi=1.5)
    sd["norm.bias"] = rn(d, std=0.1)
    return sd


@functools.lru_cache(maxsize=2)
def _stand_in_cached(name, seed, depth):
    return _stand_in(name, seed, depth)


def stand_in_state_dict(name: str = "dinov2_vits14", seed: int = 0, depth: int = None):
    """Seeded stand-in for the hub checkpoint of ``name``: its keys and shapes (``depth`` blocks, default the model's);
    weights ~ N(0, 1 / fan_in), LayerNorm gains ~ U(0.5, 1.5), biases ~ N(0, 0.1), LayerScale gains log-normal around
    0.2; the plain models' positional grid has four 3 x 3 patches of large offsets (high-norm tokens).  Returns the
    cached dict itself (do not modify it)."""
    return _stand_in_cached(name, seed, depth)


def calibration_frames(seed: int = 0, n: int = 2) -> torch.Tensor:
    """n seeded normalised (3, 224, 224) frames: smooth random fields plus pixel noise, quantised to uint8 like decoded
    frames."""
    g = torch.Generator().manual_seed(6100 + seed)
    low = torch.rand(n, 3, 8, 8, generator=g)
    img = F.interpolate(low, size=(CROP, CROP), mode="bilinear", align_corners=False)
    img = (img * 0.8 + 0.2 * torch.rand(n, 3, CROP, CROP, generator=g)).mul(255).round().clamp(0, 255)
    return (img.div(255) - torch.tensor(IMAGENET_MEAN).view(3, 1, 1)) / torch.tensor(IMAGENET_STD).view(3, 1, 1)


# ---- work
def flops(name: str) -> dict:
    """Algorithmic work per frame at 224 px: GEMM FLOPs with every block on all tokens (patch embedding included), and
    the attention's (2 S^2 D for scores and 2 S^2 D for P.V per block)."""
    d, depth, ffn, reg = shape_of(name)
    S = TOKENS + (N_REG if reg else 0)
    hidden = 4 * d if ffn == "mlp" else SWIGLU_HIDDEN
    per_tok = 3 * d * d + d * d + (d * hidden + hidden * d if ffn == "mlp" else d * 2 * hidden + hidden * d)
    gemm = 2 * (GRID * GRID * d * 3 * PATCH * PATCH + depth * S * per_tok)
    return {"gemm": gemm, "attention": depth * 4 * S * S * d}


def executed_gemm_flops(name: str) -> int:
    """The GEMM FLOPs the engine executes per frame: split weights double every product, the patch rows are padded
    to 592 columns, and the last block's out-projection and FFN run on the class row only."""
    d, depth, ffn, reg = shape_of(name)
    S = TOKENS + (N_REG if reg else 0)
    hidden = 4 * d if ffn == "mlp" else SWIGLU_HIDDEN
    ffn_tok = d * hidden + hidden * d if ffn == "mlp" else d * 2 * hidden + hidden * d
    blocks = depth * S * 3 * d * d + ((depth - 1) * S + 1) * (d * d + ffn_tok)
    return 2 * 2 * (GRID * GRID * d * 592 + blocks)

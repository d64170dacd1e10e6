"""Plain-torch restatement of VideoMAE's clip feature: Hugging Face ``VideoMAEForVideoClassification`` (Kinetics-400
fine-tuned ViT-S / B / L, 16 frames at 224 px), the classifier's input ``fc_norm(last_hidden_state.mean(1))`` and the
classifier; the processor's PIL preset (``VideoMAEImageProcessorPil``); the fixed sinusoid table; seeded stand-ins in
the HF key layout (the checkpoints cannot be fetched offline).

``forward`` runs in the dtype of its inputs: float64 on float64 weights is the exact reference the engine's features
are held against.  ``preset`` is the processor restated: Pillow bilinear resize of the short side to 224, a crop at the
floor of half the margin (not torchvision's round), float64 rescale by 1 / 255 rounded to fp32, then Normalize in fp32.
"""
import functools

import numpy as np
import torch
import torch.nn.functional as F

T, CROP, TUBELET, PATCH = 16, 224, 2, 16
GRID = CROP // PATCH
TOKENS = (T // TUBELET) * GRID * GRID        # 1568
PK = 3 * TUBELET * PATCH * PATCH             # 1536
IMAGENET_MEAN = (0.485, 0.456, 0.406)
IMAGENET_STD = (0.229, 0.224, 0.225)
N_CLASSES = 400
# feature type -> (hidden size, depth, heads, MLP width)
SHAPES = {"videomae_vits16": (384, 12, 6, 1536), "videomae_vitb16": (768, 12, 12, 3072),
          "videomae_vitl16": (1024, 24, 16, 4096)}
LN_EPS = 1e-12          # VideoMAEConfig's layer_norm_eps default
FC_NORM_EPS = 1e-5      # fc_norm is nn.LayerNorm(hidden_size): torch's default eps


def config_dict(name: str = "videomae_vitb16", depth: int = None, **over) -> dict:
    """A config.json of the Kinetics shape of ``name`` (``depth`` layers, default the model's)."""
    d, L, h, f = SHAPES[name]
    cfg = {"hidden_size": d, "num_hidden_layers": L if depth is None else depth, "num_attention_heads": h,
           "intermediate_size": f, "hidden_act": "gelu", "layer_norm_eps": LN_EPS, "qkv_bias": True,
           "use_mean_pooling": True, "tubelet_size": TUBELET, "num_frames": T, "image_size": CROP,
           "patch_size": PATCH, "num_channels": 3, "num_labels": N_CLASSES}
    cfg.update(over)
    return cfg


def sinusoid_table(n_position: int = TOKENS, d_hid: int = 768) -> np.ndarray:
    """The table as VideoMAE's reference builds it: angles element by element in float64, sin / cos, rounded to fp32."""
    def angles(position):
        return [position / np.power(10000, 2 * (j // 2) / d_hid) for j in range(d_hid)]
    table = np.array([angles(p) for p in range(n_position)])
    table[:, 0::2] = np.sin(table[:, 0::2])
    table[:, 1::2] = np.cos(table[:, 1::2])
    return table.astype(np.float32)


# ---- the processor
def preset_frame(rgb_u8, mean=IMAGENET_MEAN, std=IMAGENET_STD) -> np.ndarray:
    """(H, W, 3) uint8 RGB -> (3, 224, 224) fp32: VideoMAEImageProcessorPil's resize (shortest edge 224, bilinear,
    long side int(224 * long / short)), center crop at ((h - 224) // 2, (w - 224) // 2), rescale, Normalize."""
    from PIL import Image
    img = Image.fromarray(np.ascontiguousarray(rgb_u8))
    w, h = img.size
    short, long = (w, h) if w <= h else (h, w)
    nl = int(CROP * long / short)
    size = (CROP, nl) if w <= h else (nl, CROP)
    if size != (w, h):
        img = img.resize(size, Image.BILINEAR)
    a = np.asarray(img).transpose(2, 0, 1)
    i, j = (a.shape[1] - CROP) // 2, (a.shape[2] - CROP) // 2
    x = (a[:, i:i + CROP, j:j + CROP].astype(np.float64) * (1 / 255)).astype(np.float32)
    m, s = np.array(mean, dtype=np.float32), np.array(std, dtype=np.float32)
    return ((x.T - m) / s).T


def preset_clip(bgr_u8, mean=IMAGENET_MEAN, std=IMAGENET_STD) -> torch.Tensor:
    """(16, H, W, 3) uint8 BGR decoded frames -> (16, 3, 224, 224) fp32 pixel_values."""
    return torch.from_numpy(np.stack([preset_frame(f[:, :, ::-1], mean, std) for f in bgr_u8]))


# ---- forward
def tubelets(x: torch.Tensor) -> torch.Tensor:
    """(n, 16, 3, 224, 224) -> (n, 1568, 1536): rows (t / 2, y, x), columns (c, dt, py, px)."""
    n = x.shape[0]
    x = x.reshape(n, T // TUBELET, TUBELET, 3, GRID, PATCH, GRID, PATCH)
    return x.permute(0, 1, 4, 6, 3, 2, 5, 7).reshape(n, TOKENS, PK)


def prepare(sd, dtype=torch.float64, device="cpu") -> dict:
    """The state dict in ``dtype`` on ``device``, qkv fused as the engine fuses it ([q | k | v], bias [q | 0 | v])."""
    p = {k: v.to(device, dtype) for k, v in sd.items() if torch.is_tensor(v) and v.is_floating_point()}
    i = 0
    while f"videomae.encoder.layer.{i}.layernorm_before.weight" in p:
        a = f"videomae.encoder.layer.{i}.attention.attention."
        p[a + "qkv.weight"] = torch.cat([p[a + "query.weight"], p[a + "key.weight"], p[a + "value.weight"]])
        qb = p.get(a + "q_bias")
        p[a + "qkv.bias"] = None if qb is None else torch.cat([qb, torch.zeros_like(qb), p[a + "v_bias"]])
        i += 1
    p["depth"] = i
    return p


# the engine's tensor classes (scripts/precision/emulate_videomae.py): w every GEMM weight, tube the tubelet rows, ln
# the layernorm_before / layernorm_after outputs, qkv q / k / v, p the softmax numerator P per 64-key block, att the
# attention output, hidden the MLP hidden layer
CLASSES = ("w", "tube", "ln", "qkv", "p", "att", "hidden")
ENGINE_FP16 = ("tube", "ln", "qkv", "p", "att", "hidden")     # csrc/videomae.cu: weights are split-fp16 pairs
KEY_BLOCK = 64                                                 # videomae_attention: keys per streamed block


def _q(x, cls, fp16):
    return x.to(torch.float16).to(x.dtype) if cls in fp16 else x


def _linear(x, w, b, fp16):
    return F.linear(x, _q(w, "w", fp16), b)


def _attention(q, k, v, fp16):
    """softmax(q k^T / 8) v; with "p" in fp16 the kernel's online softmax: per 64-key block P = exp(s - running max)
    rounded to fp16 before P.V, the sum of the unrounded P, the output rescaled as the max grows."""
    s = (q @ k.transpose(-1, -2)) * 0.125
    if "p" not in fp16:
        return torch.softmax(s, -1) @ v
    m = torch.full(s.shape[:-1] + (1,), -float("inf"), dtype=s.dtype, device=s.device)
    l = torch.zeros_like(m)
    o = torch.zeros(s.shape[:-1] + (v.shape[-1],), dtype=s.dtype, device=s.device)
    for b0 in range(0, s.shape[-1], KEY_BLOCK):
        sb = s[..., b0:b0 + KEY_BLOCK]
        mn = torch.maximum(m, sb.amax(-1, keepdim=True))
        carry, e = torch.exp(m - mn), torch.exp(sb - mn)
        l = l * carry + e.sum(-1, keepdim=True)
        o = o * carry + _q(e, "p", fp16) @ v[..., b0:b0 + KEY_BLOCK, :]
        m = mn
    return o / l


def embed(p, rows: torch.Tensor, fp16=()) -> torch.Tensor:
    """tubelet rows (n, 1568, 1536) -> (n, 1568, D): the Conv3d as a linear, + the sinusoid table."""
    w = p["videomae.embeddings.patch_embeddings.projection.weight"]
    d = w.shape[0]
    x = _linear(_q(rows, "tube", fp16), w.reshape(d, PK), p["videomae.embeddings.patch_embeddings.projection.bias"],
                fp16)
    return x + torch.from_numpy(sinusoid_table(TOKENS, d)).to(x)


def block(p, i: int, x: torch.Tensor, eps: float = LN_EPS, fp16=()) -> torch.Tensor:
    """One pre-LN block; ``fp16``: the tensor classes rounded to one fp16 value (none: the exact block)."""
    d = x.shape[-1]
    pre = f"videomae.encoder.layer.{i}."
    a = pre + "attention.attention."
    hh = _q(F.layer_norm(x, (d,), p[pre + "layernorm_before.weight"], p[pre + "layernorm_before.bias"], eps), "ln", fp16)
    qkv = _q(_linear(hh, p[a + "qkv.weight"], p[a + "qkv.bias"], fp16), "qkv", fp16)
    n, S, _ = qkv.shape
    q, k, v = (t.reshape(n, S, d // 64, 64).transpose(1, 2) for t in qkv.split(d, -1))
    att = _q(_attention(q, k, v, fp16).transpose(1, 2).reshape(n, S, d), "att", fp16)
    x = x + _linear(att, p[pre + "attention.output.dense.weight"], p[pre + "attention.output.dense.bias"], fp16)
    hh = _q(F.layer_norm(x, (d,), p[pre + "layernorm_after.weight"], p[pre + "layernorm_after.bias"], eps), "ln", fp16)
    hh = _q(F.gelu(_linear(hh, p[pre + "intermediate.dense.weight"], p[pre + "intermediate.dense.bias"], fp16)),
            "hidden", fp16)
    return x + _linear(hh, p[pre + "output.dense.weight"], p[pre + "output.dense.bias"], fp16)


def head(p, x: torch.Tensor) -> torch.Tensor:
    """fc_norm(mean over tokens) -> (n, D)."""
    return F.layer_norm(x.mean(1), (x.shape[-1],), p["fc_norm.weight"], p["fc_norm.bias"], FC_NORM_EPS)


def forward(p, x: torch.Tensor, eps: float = LN_EPS, fp16=()) -> torch.Tensor:
    """pixel_values (n, 16, 3, 224, 224) -> the feature (n, D), in x's dtype (``p`` from ``prepare``); ``fp16``: the
    tensor classes rounded to one fp16 value where the engine would round them (none: the exact forward)."""
    h = embed(p, tubelets(x), fp16)
    for i in range(p["depth"]):
        h = block(p, i, h, eps, fp16)
    return head(p, h)


def logits(p, feat: torch.Tensor) -> torch.Tensor:
    return F.linear(feat, p["classifier.weight"], p["classifier.bias"])


# ---- stand-ins
@functools.lru_cache(maxsize=8)
def _stand_in_cached(name, seed, depth):
    d, L, h, f = SHAPES[name]
    L = L if depth is None else depth
    g = torch.Generator().manual_seed(9100 + 17 * seed + d)

    def rn(*shape, std):
        return torch.randn(*shape, generator=g) * std

    def gain(n):
        return torch.rand(n, generator=g) + 0.5
    sd = {"videomae.embeddings.patch_embeddings.projection.weight": rn(d, 3, TUBELET, PATCH, PATCH, std=PK ** -0.5),
          "videomae.embeddings.patch_embeddings.projection.bias": rn(d, std=0.1)}
    for i in range(L):
        pre = f"videomae.encoder.layer.{i}."
        a = pre + "attention.attention."
        for k in ("query", "key", "value"):
            sd[a + k + ".weight"] = rn(d, d, std=d ** -0.5)
        sd[a + "q_bias"] = rn(d, std=0.1)
        sd[a + "v_bias"] = rn(d, std=0.1)
        sd[pre + "attention.output.dense.weight"] = rn(d, d, std=d ** -0.5)
        sd[pre + "attention.output.dense.bias"] = rn(d, std=0.1)
        sd[pre + "intermediate.dense.weight"] = rn(f, d, std=d ** -0.5)
        sd[pre + "intermediate.dense.bias"] = rn(f, std=0.1)
        sd[pre + "output.dense.weight"] = rn(d, f, std=f ** -0.5)
        sd[pre + "output.dense.bias"] = rn(d, std=0.1)
        for n in ("layernorm_before", "layernorm_after"):
            sd[pre + n + ".weight"] = gain(d)
            sd[pre + n + ".bias"] = rn(d, std=0.1)
    sd["fc_norm.weight"] = gain(d)
    sd["fc_norm.bias"] = rn(d, std=0.1)
    sd["classifier.weight"] = rn(N_CLASSES, d, std=d ** -0.5)
    sd["classifier.bias"] = rn(N_CLASSES, std=0.1)
    return sd


def stand_in_state_dict(name: str = "videomae_vitb16", seed: int = 0, depth: int = None) -> dict:
    """Seeded stand-in for the HF checkpoint of ``name`` (``depth`` layers, default the model's): weights
    ~ N(0, 1 / fan_in), LayerNorm gains ~ U(0.5, 1.5), biases ~ N(0, 0.1).  The cached dict itself (do not modify)."""
    return _stand_in_cached(name, seed, depth)


def calibration_clips(seed: int = 0, n: int = 1) -> torch.Tensor:
    """n seeded (16, 3, 224, 224) pixel_values: smooth moving random fields plus pixel noise, quantised to uint8 like
    decoded frames, normalised with ImageNet's statistics."""
    g = torch.Generator().manual_seed(6300 + seed)
    low = torch.rand(n * T, 3, 8, 8, generator=g)
    img = F.interpolate(low, size=(CROP, CROP), mode="bilinear", align_corners=False)
    img = (img * 0.8 + 0.2 * torch.rand(n * T, 3, CROP, CROP, generator=g)).mul(255).round().clamp(0, 255)
    x = (img.div(255) - torch.tensor(IMAGENET_MEAN).view(3, 1, 1)) / torch.tensor(IMAGENET_STD).view(3, 1, 1)
    return x.reshape(n, T, 3, CROP, CROP)


def flops(name: str) -> dict:
    """Algorithmic work per clip: GEMM FLOPs (tubelet embedding included) and the attention's (4 S^2 D per block)."""
    d, L, h, f = SHAPES[name]
    gemm = 2 * (TOKENS * PK * d + L * TOKENS * (4 * d * d + 2 * d * f))
    return {"gemm": gemm, "attention": L * 4 * TOKENS * TOKENS * d}

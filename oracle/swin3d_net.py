"""Plain-torch restatement of torchvision's Swin3D clip feature: ``torchvision.models.video.swin3d_{t,s,b}()`` in eval
mode without ``head``, ``flatten(avgpool(norm(features(patch_embed(x)))))``, the ``Swin3D_*_Weights.KINETICS400_V1``
clip transform, and seeded stand-ins for the Kinetics weights (the torchvision checkpoints cannot be fetched offline).
Test infrastructure (the checker), never imported by the product."""
import functools
import math

import numpy as np
import torch
import torch.nn.functional as F

from oracle.r21d_net import form_slices, resize_restated  # noqa: F401  (form_slices: the same full-stack slicing)

IMAGENET_MEAN = [0.485, 0.456, 0.406]          # the Swin3D presets normalise with ImageNet statistics
IMAGENET_STD = [0.229, 0.224, 0.225]
RESIZE = 256
CROP = 224
EPS = 1e-5
PATCH = (2, 4, 4)
WINDOW = (8, 7, 7)
HEAD_DIM = 32
HEAD_KEYS = ("head.weight", "head.bias")
# (embed dim, depths): torchvision's swin3d_t / _s / _b; heads = dim / 32 in every stage
MODELS = {"swin3d_t": (96, (2, 2, 6, 2)), "swin3d_s": (96, (2, 2, 18, 2)), "swin3d_b": (128, (2, 2, 18, 2))}
# vf_swin3d_read_stage ids 0..5
STAGES = ("embed", "stage1", "stage2", "stage3", "stage4", "norm")


def _plain(sd):
    """The state dict without a DataParallel "module." prefix."""
    if not any(k.startswith("module.") for k in sd):
        return sd
    return {k[7:] if k.startswith("module.") else k: v for k, v in sd.items()}


def config(sd):
    """(embed dim, depths) from the weights, as the engine infers them."""
    sd = _plain(sd)
    dim = sd["patch_embed.proj.weight"].shape[0]
    depths = []
    for s in range(4):
        d = 0
        while f"features.{2 * s}.{d}.norm1.weight" in sd:
            d += 1
        depths.append(d)
    return dim, tuple(depths)


def window_and_shift(size, shifted):
    """torchvision's _get_window_and_shift_size: a window dimension no smaller than the feature is clamped to it and
    its shift zeroed."""
    win, sh = list(WINDOW), [w // 2 if shifted else 0 for w in WINDOW]
    for i in range(3):
        if size[i] <= win[i]:
            win[i], sh[i] = size[i], 0
    return win, sh


def bias_index(win):
    """The relative-position index of a (possibly clamped) window, computed arithmetically with the full (8,7,7)
    window's strides: (dt + 7) * 169 + (dh + 6) * 13 + (dw + 6), tokens t-major.  Equals torchvision's
    ``relative_position_index[:vol, :vol]``."""
    t, h, w = np.meshgrid(np.arange(win[0]), np.arange(win[1]), np.arange(win[2]), indexing="ij")
    base = (t * 169 + h * 13 + w).reshape(-1)
    return torch.from_numpy(base[:, None] - base[None, :] + 7 * 169 + 6 * 13 + 6)


def region_ids(padded, win, sh):
    """The shift mask's region id of every padded position (torchvision's _compute_attention_mask_3d slices)."""
    ids = []
    for i in range(3):
        p = np.arange(padded[i])
        ids.append(np.where(p < padded[i] - win[i], 0, np.where(p < padded[i] - sh[i], 1, 2)))
    return torch.from_numpy(ids[0][:, None, None] * 9 + ids[1][None, :, None] * 3 + ids[2][None, None, :])


def window_attention(sd, p, x, heads, shifted):
    """ShiftedWindowAttention3d ``p`` (eval) on x (B, T, H, W, C), restated: pad after norm1, cyclic shift, windows,
    q scaled by head_dim ** -0.5, relative-position bias, -100 shift mask, softmax, proj, reverse."""
    b, t, h, w, c = x.shape
    win, sh = window_and_shift((t, h, w), shifted)
    pad = [(win[i] - (t, h, w)[i] % win[i]) % win[i] for i in range(3)]
    x = F.pad(x, (0, 0, 0, pad[2], 0, pad[1], 0, pad[0]))
    tp, hp, wp = x.shape[1:4]
    if sum(sh):
        x = torch.roll(x, shifts=(-sh[0], -sh[1], -sh[2]), dims=(1, 2, 3))
    nw = (tp // win[0]) * (hp // win[1]) * (wp // win[2])
    vol = win[0] * win[1] * win[2]
    x = x.view(b, tp // win[0], win[0], hp // win[1], win[1], wp // win[2], win[2], c)
    x = x.permute(0, 1, 3, 5, 2, 4, 6, 7).reshape(b * nw, vol, c)
    qkv = F.linear(x, sd[p + ".qkv.weight"], sd[p + ".qkv.bias"]).reshape(b * nw, vol, 3, heads, c // heads)
    q, k, v = qkv.permute(2, 0, 3, 1, 4)
    attn = (q * (c // heads) ** -0.5) @ k.transpose(-2, -1)
    table = sd[p + ".relative_position_bias_table"].to(x.dtype)
    attn = attn + table[bias_index(win).reshape(-1).to(x.device)].view(vol, vol, heads).permute(2, 0, 1)
    if sum(sh):
        reg = region_ids((tp, hp, wp), win, sh).to(x.device)
        reg = reg.view(tp // win[0], win[0], hp // win[1], win[1], wp // win[2], win[2])
        reg = reg.permute(0, 2, 4, 1, 3, 5).reshape(nw, vol)
        mask = torch.where(reg[:, None, :] != reg[:, :, None], -100.0, 0.0).to(x.dtype)
        attn = (attn.view(b, nw, heads, vol, vol) + mask[None, :, None]).view(b * nw, heads, vol, vol)
    x = (attn.softmax(-1) @ v).transpose(1, 2).reshape(b * nw, vol, c)
    x = F.linear(x, sd[p + ".proj.weight"], sd[p + ".proj.bias"])
    x = x.view(b, tp // win[0], hp // win[1], wp // win[2], win[0], win[1], win[2], c)
    x = x.permute(0, 1, 4, 2, 5, 3, 6, 7).reshape(b, tp, hp, wp, c)
    if sum(sh):
        x = torch.roll(x, shifts=(sh[0], sh[1], sh[2]), dims=(1, 2, 3))
    return x[:, :t, :h, :w]


def _ln(sd, p, x):
    return F.layer_norm(x, x.shape[-1:], sd[p + ".weight"].to(x.dtype), sd[p + ".bias"].to(x.dtype), EPS)


def block(sd, p, x, shifted):
    """SwinTransformerBlock ``p`` (eval): x + attn(norm1(x)), then + mlp(norm2(x)) (Linear, exact GELU, Linear)."""
    heads = x.shape[-1] // HEAD_DIM
    x = x + window_attention(sd, p + ".attn", _ln(sd, p + ".norm1", x), heads, shifted)
    y = F.gelu(F.linear(_ln(sd, p + ".norm2", x), sd[p + ".mlp.0.weight"], sd[p + ".mlp.0.bias"]))
    return x + F.linear(y, sd[p + ".mlp.3.weight"], sd[p + ".mlp.3.bias"])


def merge_rows(x):
    """PatchMerging's gather: x0..x3 = [0::2, 0::2], [1::2, 0::2], [0::2, 1::2], [1::2, 1::2] along (H, W)."""
    x = F.pad(x, (0, 0, 0, x.shape[-2] % 2, 0, x.shape[-3] % 2))
    return torch.cat([x[..., 0::2, 0::2, :], x[..., 1::2, 0::2, :], x[..., 0::2, 1::2, :], x[..., 1::2, 1::2, :]], -1)


def patch_merge(sd, p, x):
    return F.linear(_ln(sd, p + ".norm", merge_rows(x)), sd[p + ".reduction.weight"])


def embed(sd, x):
    """PatchEmbed3d: pad T to even (after Normalize: zero frames), Conv3d (2,4,4)/(2,4,4), channels last, LayerNorm."""
    sd = _plain(sd)
    x = F.pad(x, (0, 0, 0, 0, 0, x.shape[2] % 2))
    y = F.conv3d(x, sd["patch_embed.proj.weight"].to(x.dtype), sd["patch_embed.proj.bias"].to(x.dtype), stride=PATCH)
    return _ln(sd, "patch_embed.norm", y.permute(0, 2, 3, 4, 1))


def forward(sd, x, taps: bool = False):
    """x: (n, 3, T, 224, 224) normalised -> (n, C_out) features ``flatten(avgpool(norm(features(patch_embed(x)))))``;
    with ``taps`` also {stage name: activation (n, T', H', W', C)} (STAGES)."""
    sd = {k: v.to(x.dtype) if v.is_floating_point() else v for k, v in _plain(sd).items()}
    _, depths = config(sd)
    st = {}
    y = embed(sd, x)
    st["embed"] = y
    for s in range(4):
        for d in range(depths[s]):
            y = block(sd, f"features.{2 * s}.{d}", y, d % 2 == 1)
        st[f"stage{s + 1}"] = y
        if s < 3:
            y = patch_merge(sd, f"features.{2 * s + 1}", y)
    y = _ln(sd, "norm", y)
    st["norm"] = y
    f = y.mean(dim=(1, 2, 3))
    return (f, st) if taps else f


def logits(sd, feats):
    """head (Linear C_out -> 400) on the feature."""
    sd = _plain(sd)
    return feats @ sd[HEAD_KEYS[0]].to(feats.dtype).T + sd[HEAD_KEYS[1]].to(feats.dtype)


def flops(name: str, T: int = 32):
    """(window-attention GFLOP, total GFLOP) of one T-frame clip at 224 x 224, counted from shapes: every GEMM's
    2 M N K, and per window and head 2 * 2 * vol^2 * 32 (q.k^T and P.v) over the padded windows."""
    dim, depths = MODELS[name]
    tq = (T + 1) // 2
    att, gemm = 0.0, 2.0 * tq * 56 * 56 * 96 * dim
    for s in range(4):
        c, hw = dim * 2 ** s, 56 >> s
        rows = tq * hw * hw
        win, _ = window_and_shift((tq, hw, hw), False)
        tp = math.ceil(tq / win[0]) * win[0]
        att += depths[s] * 4.0 * (tp * hw * hw) * (win[0] * win[1] * win[2]) * c
        gemm += depths[s] * 2.0 * rows * c * (3 * c + c + 8 * c)
        if s < 3:
            gemm += 2.0 * (rows // 4) * 4 * c * 2 * c
    return att / 1e9, (att + gemm) / 1e9


# ---- the transform
def crop_offset(d: int, crop: int = CROP) -> int:
    """torchvision center_crop's offset: int(round((d - crop) / 2))."""
    return int(round((d - crop) / 2.0))


def resize_geometry(h: int, w: int):
    """Resize([256]): the short side to 256, the long side int(256 * long / short); a short side of 256 is kept."""
    short, long = (w, h) if w <= h else (h, w)
    if short == RESIZE:
        return h, w
    nl = int(RESIZE * long / short)
    return (nl, RESIZE) if w <= h else (RESIZE, nl)


def transform(rgb_u8) -> torch.Tensor:
    """(T, H, W, 3) uint8 RGB frames -> (3, T, 224, 224) fp32, Swin3D_*_Weights.KINETICS400_V1.transforms() restated:
    Resize([256]) bilinear without antialias on uint8 (float interpolation, round half to even), CenterCrop(224), /255,
    Normalize."""
    x = np.ascontiguousarray(np.asarray(rgb_u8).transpose(3, 0, 1, 2))          # (3, T, H, W)
    rh, rw = resize_geometry(x.shape[2], x.shape[3])
    if (rh, rw) != x.shape[2:]:
        x = np.rint(resize_restated(x.astype(np.float32), rh, rw)).astype(np.uint8)
    i, j = crop_offset(rh), crop_offset(rw)
    vid = torch.from_numpy(x[..., i:i + CROP, j:j + CROP].copy()).to(torch.float32) / 255
    shape = (-1, 1, 1, 1)
    return (vid - torch.as_tensor(IMAGENET_MEAN).reshape(shape)) / torch.as_tensor(IMAGENET_STD).reshape(shape)


def transform_torchvision(rgb_u8) -> torch.Tensor:
    """The preset itself on (T, H, W, 3) uint8 RGB frames -> (3, T, 224, 224)."""
    import torchvision
    vid = torch.as_tensor(np.asarray(rgb_u8)).permute(0, 3, 1, 2).contiguous()       # (T, C, H, W)
    return torchvision.models.video.Swin3D_T_Weights.KINETICS400_V1.transforms()(vid)


def calibration_clips(seed: int = 0, n: int = 2, T: int = 32) -> torch.Tensor:
    """n seeded normalised (3, T, 224, 224) clips: smooth random space-time fields plus pixel noise, quantised to uint8
    like decoded frames."""
    g = torch.Generator().manual_seed(5000 + seed)
    low = torch.rand(n, 3, 3, 8, 8, generator=g)
    clip = F.interpolate(low, size=(T, CROP, CROP), mode="trilinear", align_corners=False)
    clip = (clip * 0.8 + 0.2 * torch.rand(n, 3, T, CROP, CROP, generator=g)).mul(255).round().clamp(0, 255)
    shape = (-1, 1, 1, 1)
    return (clip.div(255) - torch.as_tensor(IMAGENET_MEAN).reshape(shape)) / torch.as_tensor(IMAGENET_STD).reshape(shape)


def torchvision_model(name: str):
    import torchvision
    return getattr(torchvision.models.video, name)(weights=None)


@functools.lru_cache(maxsize=None)
def _stand_in(name: str, seed: int):
    """The module's keys and shapes with values that keep every block's signal O(1) and its attention non-uniform."""
    with torch.random.fork_rng(devices=[]):
        torch.manual_seed(seed)
        net = torchvision_model(name)
    g = torch.Generator().manual_seed(6000 + seed)
    sd = {}
    for k, v in net.state_dict().items():
        if k.endswith("relative_position_index"):
            sd[k] = v.clone()
        elif k.endswith("relative_position_bias_table"):
            sd[k] = (torch.randn(v.shape, generator=g, dtype=torch.float64) * 0.5).float()
        elif ".norm" in k or k.startswith("norm.") or "norm1" in k or "norm2" in k:
            if k.endswith("weight"):
                sd[k] = (torch.rand(v.shape, generator=g, dtype=torch.float64) + 0.5).float()
            else:
                sd[k] = (torch.randn(v.shape, generator=g, dtype=torch.float64) * 0.1).float()
        elif k.endswith("weight"):
            fan_in = v[0].numel()
            sd[k] = (torch.randn(v.shape, generator=g, dtype=torch.float64) / math.sqrt(fan_in)).float()
        else:
            sd[k] = (torch.randn(v.shape, generator=g, dtype=torch.float64) * 0.1).float()
    return sd


def stand_in_state_dict(name: str = "swin3d_t", seed: int = 0):
    """Seeded stand-in for torchvision's ``{name}`` Kinetics-400 checkpoint: the module's keys and shapes;
    every weight ~ N(0, 1 / fan_in); LayerNorm gains ~ U(0.5, 1.5), LayerNorm and Linear biases ~ N(0, 0.1); relative
    position bias tables ~ N(0, 0.5); relative_position_index the module's buffer.  Returns a fresh copy."""
    return {k: v.clone() for k, v in _stand_in(name, seed).items()}

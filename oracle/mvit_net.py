"""Plain-torch restatement of torchvision's MViT clip feature: ``torchvision.models.video.mvit_v1_b()`` /
``mvit_v2_s()`` in eval mode without ``head``, ``norm(x)[:, 0]``, the ``MViT_*_Weights.KINETICS400_V1`` clip transform,
and seeded stand-ins for the Kinetics weights (the torchvision checkpoints cannot be fetched offline).  Test
infrastructure (the checker), never imported by the product."""
import functools
import math

import numpy as np
import torch
import torch.nn.functional as F

from oracle.swin3d_net import crop_offset, resize_geometry, resize_restated  # the same Resize([256]) / CenterCrop(224)

MEAN = 0.45                 # the MViT presets normalise every channel with (0.45, 0.225)
STD = 0.225
CROP = 224
T = 16                      # torchvision's position tables and min_temporal_size fix 16 x 224 x 224
EPS = 1e-6
HEAD_DIM = 96
HEAD_KEYS = ("head.1.weight", "head.1.bias")
MODELS = ("mvit_v1_b", "mvit_v2_s")
# torchvision's block settings: heads, input / output channels, q stride, kv stride (kernels 3 x 3 x 3 everywhere)
HEADS = (1, 2, 2, 4, 4, 4, 4, 4, 4, 4, 4, 4, 4, 4, 8, 8)
CHANNELS = {
    "mvit_v1_b": ((96, 192, 192, 384, 384, 384, 384, 384, 384, 384, 384, 384, 384, 384, 768, 768),
                  (192, 192, 384, 384, 384, 384, 384, 384, 384, 384, 384, 384, 384, 768, 768, 768)),
    "mvit_v2_s": ((96, 96, 192, 192, 384, 384, 384, 384, 384, 384, 384, 384, 384, 384, 384, 768),
                  (96, 192, 192, 384, 384, 384, 384, 384, 384, 384, 384, 384, 384, 384, 768, 768)),
}
STRIDE_Q = (1, 2, 1, 2, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 2, 1)
STRIDE_KV = (8, 4, 4, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 1, 1)
# vf_mvit_read_stage ids 0..5: stage s ends at the block before the next q stride
STAGES = ("embed", "stage1", "stage2", "stage3", "stage4", "norm")
STAGE_END = (0, 2, 13, 15)


def _plain(sd):
    """The state dict without a DataParallel "module." prefix."""
    if not any(k.startswith("module.") for k in sd):
        return sd
    return {k[7:] if k.startswith("module.") else k: v for k, v in sd.items()}


def config(sd):
    """The model name from the weights, as the engine infers it: v2 has relative-position tables, v1 absolute
    position embeddings."""
    sd = _plain(sd)
    if "blocks.0.attn.rel_pos_h" in sd:
        return "mvit_v2_s"
    if "pos_encoding.spatial_pos" in sd:
        return "mvit_v1_b"
    raise ValueError("neither an mvit_v1_b nor an mvit_v2_s state dict")


def pooled(s, stride):
    """Extent after a 3-tap conv / pool with padding 1 and this stride."""
    return (s - 1) // stride + 1


def _ln(sd, p, x):
    return F.layer_norm(x, (x.shape[-1],), sd[p + ".weight"], sd[p + ".bias"], EPS)


def head_pool(sd, p, x, thw, stride):
    """Pool ``p`` on x (B, heads, 1 + N, 96): depthwise Conv3d 3x3x3 / (1, s, s) pad 1 on the tokens, class token
    re-attached, then LayerNorm(96)."""
    b, nh, _, c = x.shape
    cls, tok = x[:, :, :1], x[:, :, 1:]
    tok = tok.transpose(2, 3).reshape((b * nh, c) + tuple(thw))
    tok = F.conv3d(tok, sd[p + ".pool.weight"], None, (1, stride, stride), 1, groups=c)
    t, h, w = tok.shape[2:]
    tok = tok.reshape(b, nh, c, -1).transpose(2, 3)
    return _ln(sd, p + ".norm_act.0", torch.cat((cls, tok), dim=2)), (t, h, w)


def rel_distances(qs, ks):
    """_add_rel_pos's ratio-scaled distance table (q extent qs, k extent ks), in its float32 arithmetic."""
    q_ratio, k_ratio = max(ks / qs, 1.0), max(qs / ks, 1.0)
    return (torch.arange(qs)[:, None] * q_ratio - (torch.arange(ks)[None, :] + (1.0 - ks)) * k_ratio).long()


def rel_bias(q, q_thw, k_thw, rel_h, rel_w, rel_t):
    """The decomposed relative-position bias (B, heads, Nq, Nk) on token rows / columns, from the unscaled q."""
    (qt, qh, qw), (kt, kh, kw) = q_thw, k_thw
    rh = rel_h[rel_distances(qh, kh).to(q.device)]          # (qh, kh, 96)
    rw = rel_w[rel_distances(qw, kw).to(q.device)]
    rt = rel_t[rel_distances(qt, kt).to(q.device)]
    b, nh, _, c = q.shape
    r = q[:, :, 1:].reshape(b, nh, qt, qh, qw, c)
    bh = torch.einsum("bythwc,hkc->bythwk", r, rh)
    bw = torch.einsum("bythwc,wkc->bythwk", r, rw)
    bt = torch.einsum("bythwc,tkc->bythwk", r, rt)
    return (bt[..., :, None, None] + bh[..., None, :, None] + bw[..., None, None, :]).reshape(
        b, nh, qt * qh * qw, kt * kh * kw)


def attention(q, k, v, q_thw=None, k_thw=None, rel=None, resid=False):
    """softmax(q k^T / sqrt(96) (+ rel-pos bias on token rows / columns)) v (+ q on token rows): q (B, heads, Nq, 96)."""
    attn = (q * HEAD_DIM ** -0.5) @ k.transpose(2, 3)
    if rel is not None:
        attn = attn.clone()
        attn[:, :, 1:, 1:] += rel_bias(q, q_thw, k_thw, *rel)
    x = attn.softmax(dim=-1) @ v
    if resid:
        x = x.clone()
        x[:, :, 1:] += q[:, :, 1:]
    return x


def block(sd, name, i, x, s_in):
    """MultiscaleBlock i (eval) on x (B, 1 + 8 s_in^2, C_in) -> (B, 1 + 8 s_q^2, C_out)."""
    p = f"blocks.{i}."
    v2 = name == "mvit_v2_s"
    cin, cout = CHANNELS[name][0][i], CHANNELS[name][1][i]
    ad, heads, sq, skv = (cout if v2 else cin), HEADS[i], STRIDE_Q[i], STRIDE_KV[i]
    thw = (T // 2, s_in, s_in)
    b, n, _ = x.shape
    xn1 = _ln(sd, p + "norm1", x)
    qkv = F.linear(xn1, sd[p + "attn.qkv.weight"], sd[p + "attn.qkv.bias"])
    q, k, v = qkv.reshape(b, n, 3, heads, HEAD_DIM).transpose(1, 3).unbind(dim=2)
    k, k_thw = head_pool(sd, p + "attn.pool_k", k, thw, skv)
    v, _ = head_pool(sd, p + "attn.pool_v", v, thw, skv)
    q_thw = thw
    if v2 or sq > 1:
        q, q_thw = head_pool(sd, p + "attn.pool_q", q, thw, sq)
    rel = (sd[p + "attn.rel_pos_h"], sd[p + "attn.rel_pos_w"], sd[p + "attn.rel_pos_t"]) if v2 else None
    a = attention(q, k, v, q_thw, k_thw, rel, resid=v2)
    a = F.linear(a.transpose(1, 2).reshape(b, -1, ad), sd[p + "attn.project.0.weight"], sd[p + "attn.project.0.bias"])
    skip = x
    if v2 and cin != cout:
        skip = F.linear(xn1, sd[p + "project.weight"], sd[p + "project.bias"])
    if sq > 1:
        skip = skip_pool(skip, thw)
    x = skip + a
    xn2 = _ln(sd, p + "norm2", x)
    if not v2 and cin != cout:
        x = F.linear(xn2, sd[p + "project.weight"], sd[p + "project.bias"])
    h = F.gelu(F.linear(xn2, sd[p + "mlp.0.weight"], sd[p + "mlp.0.bias"]))
    return x + F.linear(h, sd[p + "mlp.3.weight"], sd[p + "mlp.3.bias"]), pooled(s_in, sq)


def skip_pool(x, thw):
    """MaxPool3d((1,3,3), (1,2,2), (0,1,1)) of the tokens of x (B, 1 + N, C), class token passed through."""
    b, _, c = x.shape
    tok = x[:, 1:].transpose(1, 2).reshape((b, c) + tuple(thw))
    tok = F.max_pool3d(tok, (1, 3, 3), (1, 2, 2), (0, 1, 1)).reshape(b, c, -1).transpose(1, 2)
    return torch.cat((x[:, :1], tok), dim=1)


def embed(sd, x):
    """conv_proj (3,7,7)/(2,4,4) pad (1,3,3), tokens t-major, class token, and (v1) the position embeddings."""
    sd = _plain(sd)
    y = F.conv3d(x, sd["conv_proj.weight"], sd["conv_proj.bias"], (2, 4, 4), (1, 3, 3)).flatten(2).transpose(1, 2)
    y = torch.cat((sd["pos_encoding.class_token"].expand(y.shape[0], 1, -1), y), dim=1)
    if "pos_encoding.spatial_pos" in sd:
        pos = torch.repeat_interleave(sd["pos_encoding.temporal_pos"], 3136, dim=0) + sd["pos_encoding.spatial_pos"].repeat(
            T // 2, 1)
        y = y + torch.cat((sd["pos_encoding.class_pos"][None], pos))[None]
    return y


def forward(sd, x, taps: bool = False):
    """x: (n, 3, 16, 224, 224) normalised -> (n, 768) features ``norm(x)[:, 0]``; with ``taps`` also {stage name:
    activation (n, tokens, C)} (STAGES)."""
    sd = {k: v.to(x.dtype) if v.is_floating_point() else v for k, v in _plain(sd).items()}
    name = config(sd)
    st = {}
    y = embed(sd, x)
    st["embed"] = y
    s = 56
    for i in range(16):
        y, s = block(sd, name, i, y, s)
        if i in STAGE_END:
            st[f"stage{STAGE_END.index(i) + 1}"] = y
    y = _ln(sd, "norm", y)
    st["norm"] = y
    f = y[:, 0]
    return (f, st) if taps else f


def logits(sd, feats):
    """head.1 (Linear 768 -> 400) on the feature."""
    sd = _plain(sd)
    return feats @ sd[HEAD_KEYS[0]].to(feats.dtype).T + sd[HEAD_KEYS[1]].to(feats.dtype)


def flops(name: str):
    """(pooling-attention GFLOP, total GFLOP) of one 16-frame clip, counted from shapes: every GEMM's 2 M N K and per
    (clip, head) 2 * 2 * Nq * Nk * 96 (q.k^T and P.v); pooling convs, norms and rel-pos dots excluded."""
    cin_all, cout_all = CHANNELS[name]
    gemm = 2.0 * 8 * 3136 * 96 * 441
    att = 0.0
    s = 56
    for i in range(16):
        v2 = name == "mvit_v2_s"
        cin, cout = cin_all[i], cout_all[i]
        ad = cout if v2 else cin
        n_in, sq = 1 + 8 * s * s, pooled(s, STRIDE_Q[i])
        n_q, n_k = 1 + 8 * sq * sq, 1 + 8 * pooled(s, STRIDE_KV[i]) ** 2
        gemm += 2.0 * n_in * cin * 3 * ad + 2.0 * n_q * ad * ad + 2.0 * n_q * ad * 4 * ad + 2.0 * n_q * 4 * ad * cout
        if cin != cout:
            gemm += 2.0 * (n_in if v2 else n_q) * cin * cout
        att += 4.0 * n_q * n_k * ad
        s = sq
    return att / 1e9, (att + gemm) / 1e9


# ---- the transform
def transform(rgb_u8) -> torch.Tensor:
    """(16, H, W, 3) uint8 RGB frames -> (3, 16, 224, 224) fp32, MViT_*_Weights.KINETICS400_V1.transforms() restated:
    Resize([256]) bilinear without antialias on uint8 (float interpolation, round half to even), CenterCrop(224), /255,
    Normalize(0.45, 0.225)."""
    x = np.ascontiguousarray(np.asarray(rgb_u8).transpose(3, 0, 1, 2))          # (3, T, H, W)
    rh, rw = resize_geometry(x.shape[2], x.shape[3])
    if (rh, rw) != x.shape[2:]:
        x = np.rint(resize_restated(x.astype(np.float32), rh, rw)).astype(np.uint8)
    i, j = crop_offset(rh), crop_offset(rw)
    vid = torch.from_numpy(x[..., i:i + CROP, j:j + CROP].copy()).to(torch.float32) / 255
    return (vid - torch.tensor(MEAN, dtype=torch.float32)) / torch.tensor(STD, dtype=torch.float32)


def transform_torchvision(rgb_u8, name: str = "mvit_v2_s") -> torch.Tensor:
    """The preset itself on (T, H, W, 3) uint8 RGB frames -> (3, T, 224, 224)."""
    import torchvision
    weights = {"mvit_v1_b": torchvision.models.video.MViT_V1_B_Weights,
               "mvit_v2_s": torchvision.models.video.MViT_V2_S_Weights}[name]
    vid = torch.as_tensor(np.asarray(rgb_u8)).permute(0, 3, 1, 2).contiguous()       # (T, C, H, W)
    return weights.KINETICS400_V1.transforms()(vid)


def calibration_clips(seed: int = 0, n: int = 2) -> torch.Tensor:
    """n seeded normalised (3, 16, 224, 224) clips: smooth random space-time fields plus pixel noise, quantised to uint8
    like decoded frames."""
    g = torch.Generator().manual_seed(7000 + seed)
    low = torch.rand(n, 3, 3, 8, 8, generator=g)
    clip = F.interpolate(low, size=(T, CROP, CROP), mode="trilinear", align_corners=False)
    clip = (clip * 0.8 + 0.2 * torch.rand(n, 3, T, CROP, CROP, generator=g)).mul(255).round().clamp(0, 255)
    return (clip.div(255) - MEAN) / STD


def torchvision_model(name: str):
    import torchvision
    return getattr(torchvision.models.video, name)(weights=None)


@functools.lru_cache(maxsize=None)
def _stand_in(name: str, seed: int):
    """The module's keys and shapes with values that keep every block's signal O(1), its attention non-uniform and
    every position term large enough to matter."""
    with torch.random.fork_rng(devices=[]):
        torch.manual_seed(seed)
        net = torchvision_model(name)
    g = torch.Generator().manual_seed(8000 + seed)

    def randn(shape, std):
        return (torch.randn(shape, generator=g, dtype=torch.float64) * std).float()

    sd = {}
    for k, v in net.state_dict().items():
        if ".rel_pos_" in k:
            sd[k] = randn(v.shape, 0.05)
        elif k.startswith("pos_encoding."):
            sd[k] = randn(v.shape, 0.5 if k.endswith("_pos") else 1.0)
        elif "norm" in k:
            if k.endswith("weight"):
                sd[k] = (torch.rand(v.shape, generator=g, dtype=torch.float64) + 0.5).float()
            else:
                sd[k] = randn(v.shape, 0.1)
        elif k.endswith("weight"):
            sd[k] = randn(v.shape, 1.0 / math.sqrt(v[0].numel()))
        else:
            sd[k] = randn(v.shape, 0.1)
    return sd


def stand_in_state_dict(name: str = "mvit_v2_s", seed: int = 0):
    """Seeded stand-in for torchvision's ``{name}`` Kinetics-400 checkpoint: the module's keys and shapes; every weight
    (the pooling convs included) ~ N(0, 1 / fan_in); LayerNorm gains ~ U(0.5, 1.5), LayerNorm and Linear biases
    ~ N(0, 0.1); class token ~ N(0, 1), position embeddings ~ N(0, 0.5), rel-pos tables ~ N(0, 0.05) (torchvision's
    init zeroes or shrinks these, which would leave them untested).  Returns a fresh copy."""
    return {k: v.clone() for k, v in _stand_in(name, seed).items()}

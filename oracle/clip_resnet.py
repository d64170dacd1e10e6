"""Plain-torch restatement of the CLIP ResNet image towers (third-party openai/CLIP ``clip/model.py``: ModifiedResNet,
Bottleneck, AttentionPool2d, and build_model's configuration inference), and a calibrated seeded stand-in for their
weights.  Test infrastructure (the checker), never imported by the product.

Written from the published model code, without the clip package or an RN checkpoint to check against: the restatement is
checked piecewise -- its attention pool against torch.nn.MultiheadAttention, its transform against
oracle/clip_preprocess.py at 224 -- but the tower as a whole is not pinned by an independent implementation.

Keys are openai's ``visual.*``.  ``forward`` computes in the dtype of its input (float32 or float64)."""
import functools
import math

import torch
import torch.nn.functional as F

# name -> (blocks per stage, width, input resolution, output dim); clip.load's published towers
TOWERS = {"RN50": ((3, 4, 6, 3), 64, 224, 1024), "RN101": ((3, 4, 23, 3), 64, 224, 512),
          "RN50x4": ((4, 6, 10, 6), 80, 288, 640), "RN50x16": ((6, 8, 18, 8), 96, 384, 768)}
STAGES = ("stem", "layer1", "layer2", "layer3", "layer4", "tokens", "pre_cproj")     # vf_clip_rn_read_stage ids 0..6


def config(sd):
    """build_model's inference from shapes -> dict(layers, width, n_px, embed, heads, out_dim, tokens).  Every key the
    tower needs is then checked for presence and shape; a missing key raises KeyError, a mis-shaped one ValueError, both
    naming the key."""
    if "visual.layer1.0.conv1.weight" not in sd:
        raise KeyError("missing 'visual.layer1.0.conv1.weight'")
    if "visual.attnpool.positional_embedding" not in sd:
        raise KeyError("missing 'visual.attnpool.positional_embedding'")
    if "visual.attnpool.c_proj.weight" not in sd:
        raise KeyError("missing 'visual.attnpool.c_proj.weight'")
    layers = tuple(len({k.split(".")[2] for k in sd if k.startswith(f"visual.layer{L}.")}) for L in (1, 2, 3, 4))
    width = int(sd["visual.layer1.0.conv1.weight"].shape[0])
    side = round(math.sqrt(sd["visual.attnpool.positional_embedding"].shape[0] - 1))
    embed = width * 32
    cfg = dict(layers=layers, width=width, n_px=32 * side, embed=embed, heads=embed // 64,
               out_dim=int(sd["visual.attnpool.c_proj.weight"].shape[0]), tokens=side * side + 1)
    for k, shape in expected_shapes(cfg).items():
        if k not in sd:
            raise KeyError(f"missing '{k}'")
        if tuple(sd[k].shape) != shape:
            raise ValueError(f"'{k}' has shape {tuple(sd[k].shape)}, expected {shape}")
    return cfg


def _bn_shapes(p, c):
    return {f"{p}.{s}": (c,) for s in ("weight", "bias", "running_mean", "running_var")}


def expected_shapes(cfg):
    w, E = cfg["width"], cfg["embed"]
    out = {"visual.conv1.weight": (w // 2, 3, 3, 3), "visual.conv2.weight": (w // 2, w // 2, 3, 3),
           "visual.conv3.weight": (w, w // 2, 3, 3)}
    for i, c in ((1, w // 2), (2, w // 2), (3, w)):
        out.update(_bn_shapes(f"visual.bn{i}", c))
    cin = w
    for L, nb in enumerate(cfg["layers"]):
        planes = w << L
        for b in range(nb):
            p = f"visual.layer{L + 1}.{b}"
            ci = cin if b == 0 else 4 * planes
            out[p + ".conv1.weight"] = (planes, ci, 1, 1)
            out[p + ".conv2.weight"] = (planes, planes, 3, 3)
            out[p + ".conv3.weight"] = (4 * planes, planes, 1, 1)
            for i, c in ((1, planes), (2, planes), (3, 4 * planes)):
                out.update(_bn_shapes(f"{p}.bn{i}", c))
            if b == 0:          # stride 2, or layer1.0 whose inplanes (w) differ from 4 w
                out[p + ".downsample.0.weight"] = (4 * planes, ci, 1, 1)
                out.update(_bn_shapes(p + ".downsample.1", 4 * planes))
        cin = 4 * planes
    a = "visual.attnpool."
    out[a + "positional_embedding"] = (cfg["tokens"], E)
    for n in ("q", "k", "v"):
        out[f"{a}{n}_proj.weight"], out[f"{a}{n}_proj.bias"] = (E, E), (E,)
    out[a + "c_proj.weight"], out[a + "c_proj.bias"] = (cfg["out_dim"], E), (cfg["out_dim"],)
    return out


def _bn(sd, p, x, calib=None):
    if calib is not None:       # train-mode pass of the stand-in: running statistics = this batch's (momentum None)
        calib[p + ".running_mean"] = x.mean((0, 2, 3)).detach().clone()
        calib[p + ".running_var"] = x.var((0, 2, 3), unbiased=True).detach().clone()
        return F.batch_norm(x, None, None, sd[p + ".weight"], sd[p + ".bias"], True, 0.0, 1e-5)
    return F.batch_norm(x, sd[p + ".running_mean"], sd[p + ".running_var"], sd[p + ".weight"], sd[p + ".bias"],
                        False, 0.0, 1e-5)


def _block(sd, p, x, stride, calib=None):
    """One Bottleneck -> (output, branch = bn3's output before the add, shortcut = the downsample's output or x)."""
    y = F.relu(_bn(sd, p + ".bn1", F.conv2d(x, sd[p + ".conv1.weight"]), calib))
    y = F.relu(_bn(sd, p + ".bn2", F.conv2d(y, sd[p + ".conv2.weight"], padding=1), calib))
    if stride > 1:
        y = F.avg_pool2d(y, stride)
    y = _bn(sd, p + ".bn3", F.conv2d(y, sd[p + ".conv3.weight"]), calib)
    if p + ".downsample.0.weight" in sd:
        if stride > 1:
            x = F.avg_pool2d(x, stride)
        x = _bn(sd, p + ".downsample.1", F.conv2d(x, sd[p + ".downsample.0.weight"]), calib)
    return F.relu(x + y), y, x


def blocks(cfg):
    """Every Bottleneck in execution order: (key prefix, stride, layer index)."""
    return [(f"visual.layer{L + 1}.{b}", 2 if (b == 0 and L > 0) else 1, L)
            for L, nb in enumerate(cfg["layers"]) for b in range(nb)]


def _stem(sd, x, calib=None):
    x = F.relu(_bn(sd, "visual.bn1", F.conv2d(x, sd["visual.conv1.weight"], stride=2, padding=1), calib))
    x = F.relu(_bn(sd, "visual.bn2", F.conv2d(x, sd["visual.conv2.weight"], padding=1), calib))
    return F.relu(_bn(sd, "visual.bn3", F.conv2d(x, sd["visual.conv3.weight"], padding=1), calib))


def block(sd, cfg, i, x):
    """Bottleneck i (execution order) on its input as the engine takes it -- block 0 the UNPOOLED stem output, whose
    AvgPool2d(2) the engine fuses into layer1.0's convs -> (output, branch, shortcut)."""
    p, stride, _ = blocks(cfg)[i]
    return _block(sd, p, F.avg_pool2d(x, 2) if i == 0 else x, stride)


def block_inputs(sd, x, cfg):
    """The trunk's input to every block, in execution order, as ``block`` takes it (block 0: the stem output)."""
    y = _stem(sd, x)
    ins = []
    for i in range(len(blocks(cfg))):
        ins.append(y)
        y = block(sd, cfg, i, y)[0]
    return ins


def trunk(sd, x, cfg, calib=None):
    """stem .. layer4 -> (layer4, {stage: activation})."""
    st = {}
    x = _stem(sd, x, calib)
    st["stem"] = x
    x = F.avg_pool2d(x, 2)
    for L, nb in enumerate(cfg["layers"]):
        for b in range(nb):
            x = _block(sd, f"visual.layer{L + 1}.{b}", x, 2 if (b == 0 and L > 0) else 1, calib)[0]
        st[f"layer{L + 1}"] = x
    return x, st


def pool_tokens(sd, x):
    """AttentionPool2d's token sequence: (HW + 1, N, E), the mean first, positional embedding added."""
    x = x.flatten(start_dim=2).permute(2, 0, 1)
    x = torch.cat([x.mean(dim=0, keepdim=True), x], dim=0)
    return x + sd["visual.attnpool.positional_embedding"][:, None, :].to(x.dtype)


def attention_pool(sd, tokens, heads, out_proj=True):
    """F.multi_head_attention_forward as AttentionPool2d.forward calls it: query token 0, keys / values all tokens.
    out_proj=False returns the attention output before c_proj (the out-projection replaced by an identity)."""
    a = "visual.attnpool."
    E = tokens.shape[-1]
    if out_proj:
        ow, ob = sd[a + "c_proj.weight"], sd[a + "c_proj.bias"]
    else:
        ow, ob = torch.eye(E, dtype=tokens.dtype, device=tokens.device), torch.zeros(E, dtype=tokens.dtype, device=tokens.device)
    y, _ = F.multi_head_attention_forward(
        query=tokens[:1], key=tokens, value=tokens, embed_dim_to_check=E, num_heads=heads,
        q_proj_weight=sd[a + "q_proj.weight"], k_proj_weight=sd[a + "k_proj.weight"],
        v_proj_weight=sd[a + "v_proj.weight"], in_proj_weight=None,
        in_proj_bias=torch.cat([sd[a + "q_proj.bias"], sd[a + "k_proj.bias"], sd[a + "v_proj.bias"]]),
        bias_k=None, bias_v=None, add_zero_attn=False, dropout_p=0.0, out_proj_weight=ow, out_proj_bias=ob,
        use_separate_proj_weight=True, training=False, need_weights=False)
    return y.squeeze(0)


def forward(sd, x, taps: bool = False):
    """x: (n, 3, n_px, n_px) normalised -> (n, out_dim) (``model.encode_image``); with ``taps`` also {stage: tensor}:
    stem (conv3 + bn3 + relu), layer1..4 (NCHW), tokens (n, T, E), pre_cproj (n, E)."""
    cfg = config(sd)
    x4, st = trunk(sd, x, cfg)
    tok = pool_tokens(sd, x4)
    y = attention_pool(sd, tok, cfg["heads"])
    if not taps:
        return y
    st["tokens"] = tok.permute(1, 0, 2)
    st["pre_cproj"] = attention_pool(sd, tok, cfg["heads"], out_proj=False)
    return y, st


def preprocess_frame(frame, n_px: int) -> torch.Tensor:
    """clip.clip._transform(n_px) on one decoded frame (H x W x 3 uint8, channel order untouched as in the reference):
    Resize(n_px, BICUBIC) of the short side, CenterCrop(n_px), ToTensor, Normalize -> (3, n_px, n_px) fp32.  The same
    Pillow + torch fp32 steps as oracle/clip_preprocess.py (whose transform is fixed at 224), at the towers' own size:
    224 for RN50 / RN101, 288 for RN50x4, 384 for RN50x16."""
    import numpy as np
    from PIL import Image
    from oracle.clip_preprocess import MEAN, STD, center_crop_offset, resized_geometry
    img = Image.fromarray(frame)
    h, w = frame.shape[:2]
    oh, ow = resized_geometry(h, w, n_px)
    if (oh, ow) != (h, w):
        img = img.resize((ow, oh), Image.BICUBIC)
    top, left = center_crop_offset(oh, n_px), center_crop_offset(ow, n_px)
    img = img.crop((left, top, left + n_px, top + n_px)).convert("RGB")
    x = torch.from_numpy(np.asarray(img).copy()).permute(2, 0, 1).to(torch.float32).div(255)
    mean = torch.tensor(MEAN, dtype=torch.float32)[:, None, None]
    std = torch.tensor(STD, dtype=torch.float32)[:, None, None]
    return x.sub_(mean).div_(std)


def preprocess_batch(frames, n_px: int) -> torch.Tensor:
    return torch.stack([preprocess_frame(f, n_px) for f in frames])


def calibration_images(n_px: int, seed: int = 0, n: int = 8) -> torch.Tensor:
    """n seeded CLIP-normalised n_px x n_px images: smooth random fields plus pixel noise, quantised to uint8."""
    from oracle.clip_preprocess import MEAN, STD
    g = torch.Generator().manual_seed(3000 + seed)
    low = torch.rand(n, 3, 14, 14, generator=g)
    img = F.interpolate(low, size=(n_px, n_px), mode="bilinear", align_corners=False)
    img = (img * 0.8 + 0.2 * torch.rand(n, 3, n_px, n_px, generator=g)).mul(255).round().clamp(0, 255)
    return img.div(255).sub(torch.tensor(MEAN)[:, None, None]).div(torch.tensor(STD)[:, None, None])


@functools.lru_cache(maxsize=None)
def _stand_in(name: str, seed: int):
    layers, w, n_px, out_dim = TOWERS[name]
    E = 32 * w
    cfg = dict(layers=layers, width=w, n_px=n_px, embed=E, heads=E // 64, out_dim=out_dim, tokens=(n_px // 32) ** 2 + 1)
    g = torch.Generator().manual_seed(4000 + seed)
    sd = {}
    with torch.random.fork_rng(devices=[]):
        torch.manual_seed(seed)
        for k, shape in expected_shapes(cfg).items():
            if len(shape) == 4:                                  # torch's default conv init (kaiming_uniform, a=sqrt(5))
                conv = torch.nn.Conv2d(shape[1], shape[0], shape[2], bias=False)
                sd[k] = conv.weight.detach().clone()
    for k, shape in expected_shapes(cfg).items():
        if k.endswith(".weight") and len(shape) == 1:            # BatchNorm gain; openai zero-initialises every bn3
            gain = torch.rand(shape, generator=g) + 0.5
            sd[k] = gain * 0.25 if (k.endswith("bn3.weight") and ".layer" in k) else gain
        elif k.endswith(".bias") and "attnpool" not in k:
            sd[k] = torch.randn(shape, generator=g) * 0.1
    a = "visual.attnpool."
    for n in ("q", "k", "v", "c"):                                # openai: normal(std = E^-1/2); Linear's default bias
        sd[f"{a}{n}_proj.weight"] = torch.randn(expected_shapes(cfg)[f"{a}{n}_proj.weight"], generator=g) * E ** -0.5
        nb = expected_shapes(cfg)[f"{a}{n}_proj.bias"]
        sd[f"{a}{n}_proj.bias"] = (torch.rand(nb, generator=g) * 2 - 1) * E ** -0.5
    sd[a + "positional_embedding"] = torch.randn(cfg["tokens"], E, generator=g) / E ** 0.5
    calib = {}
    with torch.no_grad():
        trunk(sd, calibration_images(n_px, seed), cfg, calib)
    sd.update(calib)
    return {k: sd[k] for k in expected_shapes(cfg)}


def stand_in_state_dict(name: str, seed: int = 0):
    """Calibrated seeded stand-in for tower `name` (no trained CLIP RN weights exist offline; a random tower with eval
    BatchNorm at mean 0 / var 1 is too ill-conditioned to test against): torch's default conv init under
    torch.manual_seed(seed); BatchNorm gains ~ U(0.5, 1.5), times 0.25 on every block's bn3 (openai initialises bn3 to
    zero, which would make every residual branch vanish), biases ~ N(0, 0.1); running statistics from one train-mode
    pass over 8 seeded calibration images at n_px; attention-pool weights ~ N(0, E^-1/2) and the positional embedding
    randn / sqrt(E) as in openai's init.  openai's ``visual.*`` keys.  Returns a fresh copy."""
    return {k: v.clone() for k, v in _stand_in(name, seed).items()}

"""Plain-torch restatement of torchvision's S3D clip feature: ``torchvision.models.video.s3d()`` in eval mode,
``model.avgpool(model.features(x)).mean((2, 3, 4))``, the ``S3D_Weights.KINETICS400_V1`` clip transform, and a
calibrated seeded stand-in for the Kinetics weights (``s3d-d76dad2f.pth`` cannot be fetched offline).  Test
infrastructure (the checker), never imported by the product."""
import functools

import numpy as np
import torch
import torch.nn.functional as F

from oracle.r21d_net import form_slices, resize_restated  # noqa: F401  (form_slices: the same full-stack slicing)

KINETICS_MEAN = [0.43216, 0.394666, 0.37645]
KINETICS_STD = [0.22803, 0.22145, 0.216989]
RESIZE = (256, 256)
CROP = 224
EPS = 1e-3
MIN_T = 13
HEAD_KEYS = ("classifier.1.weight", "classifier.1.bias")
# SepInceptionBlock3D(cin, b0, b1 mid, b1, b2 mid, b2, b3) at features[i]
MIXED = {5: (192, 64, 96, 128, 16, 32, 32), 6: (256, 128, 128, 192, 32, 96, 64),
         8: (480, 192, 96, 208, 16, 48, 64), 9: (512, 160, 112, 224, 24, 64, 64),
         10: (512, 128, 128, 256, 24, 64, 64), 11: (512, 112, 144, 288, 32, 64, 64),
         12: (528, 256, 160, 320, 32, 128, 128), 14: (832, 256, 160, 320, 32, 128, 128),
         15: (832, 384, 192, 384, 48, 128, 128)}
STAGES = ("stem", "features3", "mixed_3c", "mixed_4f", "mixed_5c")     # vf_s3d_read_stage ids 0..4
STAGE_AFTER = {0: "stem", 3: "features3", 6: "mixed_3c", 12: "mixed_4f", 15: "mixed_5c"}


def _cna(sd, p, x, stride=1, padding=0):
    """Conv3dNormActivation p: conv p.0 (no bias) -> BatchNorm3d p.1 (eval, eps 1e-3) -> ReLU."""
    x = F.conv3d(x, sd[p + ".0.weight"], stride=stride, padding=padding)
    x = F.batch_norm(x, sd[p + ".1.running_mean"], sd[p + ".1.running_var"], sd[p + ".1.weight"], sd[p + ".1.bias"],
                     False, 0.0, EPS)
    return F.relu(x)


def _sep(sd, p, x, k, s, pad):
    """TemporalSeparableConv: (1,k,k)/(1,s,s) pad (0,p,p), then (k,1,1)/(s,1,1) pad (p,0,0)."""
    x = _cna(sd, p + ".0", x, (1, s, s), (0, pad, pad))
    return _cna(sd, p + ".1", x, (s, 1, 1), (pad, 0, 0))


def _mixed(sd, p, x):
    x0 = _cna(sd, p + ".branch0", x)
    x1 = _sep(sd, p + ".branch1.1", _cna(sd, p + ".branch1.0", x), 3, 1, 1)
    x2 = _sep(sd, p + ".branch2.1", _cna(sd, p + ".branch2.0", x), 3, 1, 1)
    x3 = _cna(sd, p + ".branch3.1", F.max_pool3d(x, 3, 1, 1))
    return torch.cat((x0, x1, x2, x3), 1)


def features(sd, x, taps: bool = False):
    """``model.features(x)``; with ``taps`` also {stage name: activation} (STAGES)."""
    sd = {k[7:] if k.startswith("module.") else k: v for k, v in sd.items()}
    st = {}
    for i in range(16):
        if i == 0:
            x = _sep(sd, "features.0", x, 7, 2, 3)
        elif i in (1, 4):
            x = F.max_pool3d(x, (1, 3, 3), (1, 2, 2), (0, 1, 1))
        elif i == 2:
            x = _cna(sd, "features.2", x)
        elif i == 3:
            x = _sep(sd, "features.3", x, 3, 1, 1)
        elif i == 7:
            x = F.max_pool3d(x, 3, 2, 1)
        elif i == 13:
            x = F.max_pool3d(x, 2, 2, 0)
        else:
            x = _mixed(sd, f"features.{i}", x)
        if taps and i in STAGE_AFTER:
            st[STAGE_AFTER[i]] = x
    return (x, st) if taps else x


def forward(sd, x, taps: bool = False):
    """x: (n, 3, T, 224, 224) normalised, T >= 13 -> (n, 1024) features ``avgpool(features(x)).mean((2, 3, 4))``;
    with ``taps`` also {stage name: activation}."""
    y = features(sd, x, taps)
    if taps:
        y, st = y
    y = F.avg_pool3d(y, (2, 7, 7), 1).mean(dim=(2, 3, 4))
    return (y, st) if taps else y


def logits(sd, feats):
    """classifier.1 (Conv3d 1024 -> 400 with bias) on the feature: ``model(x)`` in exact arithmetic (dropout is the
    identity in eval and the head is linear, so it commutes with the spatio-temporal mean)."""
    sd = {k[7:] if k.startswith("module.") else k: v for k, v in sd.items()}
    w, b = sd[HEAD_KEYS[0]], sd[HEAD_KEYS[1]]
    return feats @ w.reshape(w.shape[0], -1).to(feats.dtype).T + b.to(feats.dtype)


def temporal_sizes(T: int):
    """(T1, T2, T3): frames after the stem, after the (3,3,3)/2 pool and after the (2,2,2)/2 pool (floor mode)."""
    T1 = (T - 1) // 2 + 1
    T2 = (T1 - 1) // 2 + 1
    return T1, T2, T2 // 2


def crop_offset(d: int, crop: int = CROP) -> int:
    """torchvision center_crop's offset: int(round((d - crop) / 2))."""
    return int(round((d - crop) / 2.0))


def resize_u8(rgb_u8: np.ndarray) -> np.ndarray:
    """(..., H, W) uint8 -> (..., 256, 256) uint8: F.resize(bilinear, antialias=False) on uint8, restated as the CUDA
    kernel computes it: float bilinear (oracle.r21d_net.resize_restated), torch.round (half to even), uint8."""
    r = resize_restated(np.asarray(rgb_u8).astype(np.float32), *RESIZE)
    return np.rint(r).astype(np.uint8)


def transform(rgb_u8) -> torch.Tensor:
    """(T, H, W, 3) uint8 RGB frames -> (3, T, 224, 224) fp32, S3D_Weights.KINETICS400_V1.transforms() restated:
    Resize((256, 256)) on uint8, CenterCrop(224) at offset 16, /255, Normalize."""
    x = np.ascontiguousarray(np.asarray(rgb_u8).transpose(3, 0, 1, 2))          # (3, T, H, W)
    r = resize_u8(x)
    i, j = crop_offset(RESIZE[0]), crop_offset(RESIZE[1])
    vid = torch.from_numpy(r[..., i:i + CROP, j:j + CROP].copy()).to(torch.float32) / 255
    shape = (-1, 1, 1, 1)
    return (vid - torch.as_tensor(KINETICS_MEAN).reshape(shape)) / torch.as_tensor(KINETICS_STD).reshape(shape)


def transform_torchvision(rgb_u8) -> torch.Tensor:
    """The preset itself on (T, H, W, 3) uint8 RGB frames -> (3, T, 224, 224)."""
    import torchvision
    vid = torch.as_tensor(np.asarray(rgb_u8)).permute(0, 3, 1, 2).contiguous()       # (T, C, H, W)
    return torchvision.models.video.S3D_Weights.KINETICS400_V1.transforms()(vid)


def calibration_clips(seed: int = 0, n: int = 2, T: int = 16) -> torch.Tensor:
    """n seeded normalised (3, T, 224, 224) clips: smooth random space-time fields plus pixel noise, quantised to uint8
    like decoded frames."""
    g = torch.Generator().manual_seed(4000 + seed)
    low = torch.rand(n, 3, 3, 8, 8, generator=g)
    clip = F.interpolate(low, size=(T, CROP, CROP), mode="trilinear", align_corners=False)
    clip = (clip * 0.8 + 0.2 * torch.rand(n, 3, T, CROP, CROP, generator=g)).mul(255).round().clamp(0, 255)
    shape = (-1, 1, 1, 1)
    return (clip.div(255) - torch.as_tensor(KINETICS_MEAN).reshape(shape)) / torch.as_tensor(KINETICS_STD).reshape(shape)


@functools.lru_cache(maxsize=None)
def _stand_in(seed: int):
    import torchvision
    with torch.random.fork_rng(devices=[]):
        torch.manual_seed(seed)
        net = torchvision.models.video.s3d(weights=None)
    g = torch.Generator().manual_seed(2000 + seed)
    for m in net.modules():
        if isinstance(m, torch.nn.BatchNorm3d):
            with torch.no_grad():
                m.weight.copy_(torch.rand(m.num_features, generator=g, dtype=torch.float64) + 0.5)
                m.bias.copy_(torch.randn(m.num_features, generator=g, dtype=torch.float64) * 0.1)
            m.momentum = None
            m.reset_running_stats()
    with torch.no_grad():
        head = net.classifier[1]
        head.weight.normal_(0.0, 0.05, generator=g)
        head.bias.normal_(0.0, 0.1, generator=g)
    x = calibration_clips(seed)
    net.train()
    with torch.no_grad():
        net.features(x)
    net.eval()
    return {k: v.detach().clone() for k, v in net.state_dict().items()}


def stand_in_state_dict(seed: int = 0):
    """Calibrated seeded stand-in for torchvision's s3d-d76dad2f.pth: (1) torchvision's init under
    torch.manual_seed(seed); (2) BatchNorm gains ~ U(0.5, 1.5), biases ~ N(0, 0.1); classifier.1 weight ~ N(0, 0.05),
    bias ~ N(0, 0.1); (3) running statistics = the batch statistics of one train-mode pass (momentum None) over 2 seeded
    16-frame clips (calibration_clips).  Same keys and shapes as the torchvision state_dict.  Returns a fresh copy."""
    return {k: v.clone() for k, v in _stand_in(seed).items()}

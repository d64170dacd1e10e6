"""Plain-torch restatement of the reference's R(2+1)D clip-feature path (models/r21d/extract_r21d.py): torchvision
``r2plus1d_18`` with ``fc = Identity`` in eval mode, its clip transform (models/r21d/transforms/rgb_transforms.py), and a
calibrated seeded stand-in for the Kinetics weights.  Test infrastructure (the checker), never imported by the product."""
import functools
import hashlib

import numpy as np
import torch
import torch.nn.functional as F

KINETICS_MEAN = [0.43216, 0.394666, 0.37645]
KINETICS_STD = [0.22803, 0.22145, 0.216989]
PRE_CROP = (128, 171)
CROP = 112
COUT = (64, 128, 256, 512)
STAGES = ("stem", "layer1", "layer2", "layer3", "layer4")       # vf_r21d_read_stage ids 0..4


def _bn(sd, p, x):
    return F.batch_norm(x, sd[p + ".running_mean"], sd[p + ".running_var"], sd[p + ".weight"], sd[p + ".bias"],
                        False, 0.0, 1e-5)


def _conv2plus1d(sd, p, x, stride):
    """Conv2Plus1D: (1,3,3) spatial conv -> BN -> ReLU -> (3,1,1) temporal conv (torchvision video_resnet.py)."""
    x = F.relu(_bn(sd, p + ".1", F.conv3d(x, sd[p + ".0.weight"], stride=(1, stride, stride), padding=(0, 1, 1))))
    return F.conv3d(x, sd[p + ".3.weight"], stride=(stride, 1, 1), padding=(1, 0, 0))


def _block(sd, p, x, stride):
    y = F.relu(_bn(sd, p + ".conv1.1", _conv2plus1d(sd, p + ".conv1.0", x, stride)))
    y = _bn(sd, p + ".conv2.1", _conv2plus1d(sd, p + ".conv2.0", y, 1))
    if p + ".downsample.0.weight" in sd:
        x = _bn(sd, p + ".downsample.1", F.conv3d(x, sd[p + ".downsample.0.weight"], stride=stride))
    return F.relu(x + y)


def forward(sd, x, taps: bool = False):
    """x: (n, 3, T, 112, 112) normalised -> (n, 512) features; with ``taps`` also {stage name: activation}."""
    sd = {k[7:] if k.startswith("module.") else k: v for k, v in sd.items()}
    st = {}
    x = F.relu(_bn(sd, "stem.1", F.conv3d(x, sd["stem.0.weight"], stride=(1, 2, 2), padding=(0, 3, 3))))
    x = F.relu(_bn(sd, "stem.4", F.conv3d(x, sd["stem.3.weight"], padding=(1, 0, 0))))
    st["stem"] = x
    for L in range(4):
        for b in range(2):
            x = _block(sd, f"layer{L + 1}.{b}", x, 2 if (b == 0 and L > 0) else 1)
        st[f"layer{L + 1}"] = x
    y = torch.flatten(F.adaptive_avg_pool3d(x, 1), 1)
    return (y, st) if taps else y


def crop_offset(d: int, crop: int = CROP) -> int:
    return int(round((d - crop) / 2.0))


def transform(rgb_u8) -> torch.Tensor:
    """(T, H, W, 3) uint8 RGB frames (a tensor or array) -> (3, T, 112, 112) fp32, the reference's Compose in its order:
    ToFloatTensorInZeroOne, Resize((128, 171)) (F.interpolate bilinear, align_corners=False), Normalize,
    CenterCrop(112) at offsets (8, 30)."""
    vid = torch.as_tensor(np.asarray(rgb_u8))
    vid = vid.permute(3, 0, 1, 2).to(torch.float32) / 255
    vid = F.interpolate(vid, size=PRE_CROP, scale_factor=None, mode="bilinear", align_corners=False)
    shape = (-1,) + (1,) * (vid.dim() - 1)
    vid = (vid - torch.as_tensor(KINETICS_MEAN).reshape(shape)) / torch.as_tensor(KINETICS_STD).reshape(shape)
    i, j = crop_offset(PRE_CROP[0]), crop_offset(PRE_CROP[1])
    return vid[..., i:i + CROP, j:j + CROP]


def _fma(a, b, c):
    """fp32 fma: the float64 product of two floats is exact; one rounding of the sum to fp32 (the double rounding this
    risks does not occur on the tested geometries)."""
    return (a.astype(np.float64) * b.astype(np.float64) + c.astype(np.float64)).astype(np.float32)


def bilinear_taps(n_in: int, n_out: int):
    """torch's CPU upsample_bilinear2d source indices and weights, restated as the CUDA kernel computes them:
    scale = float(in) / out, src = max(fma(scale, d + 0.5, -0.5), 0), i0 = min(floor(src), in - 1),
    l1 = clamp(src - i0, 0, 1), i1 = i0 + (i0 < in - 1), l0 = 1 - l1."""
    f32 = np.float32
    scale = np.full(n_out, f32(n_in) / f32(n_out), f32)
    src = np.maximum(_fma(scale, np.arange(n_out, dtype=f32) + f32(0.5), np.full(n_out, -0.5, f32)), f32(0))
    i0 = np.minimum(np.floor(src).astype(np.int64), n_in - 1)
    l1 = np.clip(src - i0.astype(f32), f32(0), f32(1)).astype(f32)
    return i0, i0 + (i0 < n_in - 1), (f32(1) - l1).astype(f32), l1


def resize_restated(x: np.ndarray, out_h: int, out_w: int) -> np.ndarray:
    """(..., H, W) fp32 -> (..., out_h, out_w) with the kernel's arithmetic: t = fma(l0w, x_0, l1w * x_1) per source
    row, out = fma(l0h, t_0, l1h * t_1) (torch's `t0 * w0 + t1 * w1`, contracted by its compiler)."""
    h0, h1, a0, a1 = bilinear_taps(x.shape[-2], out_h)
    w0, w1, b0, b1 = bilinear_taps(x.shape[-1], out_w)

    def row(h):
        return _fma(b0, x[..., h[:, None], w0[None, :]], (b1 * x[..., h[:, None], w1[None, :]]).astype(np.float32))
    return _fma(a0[:, None], row(h0), (a1[:, None] * row(h1)).astype(np.float32))


def tensor_hash(t: torch.Tensor) -> str:
    """sha1 of the fp32 bytes of one transformed (3, T, 112, 112) stack (fixture key for bit-exact transform checks)."""
    return hashlib.sha1(t.contiguous().numpy().astype(np.float32).tobytes()).hexdigest()


def form_slices(size: int, stack_size: int, step_size: int):
    """The reference's utils.form_slices: full stacks only."""
    return [(i * step_size, i * step_size + stack_size) for i in range((size - stack_size) // step_size + 1)]


def calibration_clips(seed: int = 0, n: int = 3, T: int = 8) -> torch.Tensor:
    """n seeded normalised (3, T, 112, 112) clips: smooth random space-time fields plus pixel noise, quantised to uint8
    like decoded frames."""
    g = torch.Generator().manual_seed(3000 + seed)
    low = torch.rand(n, 3, 3, 8, 8, generator=g)
    clip = F.interpolate(low, size=(T, 112, 112), mode="trilinear", align_corners=False)
    clip = (clip * 0.8 + 0.2 * torch.rand(n, 3, T, 112, 112, generator=g)).mul(255).round().clamp(0, 255)
    shape = (-1, 1, 1, 1)
    return (clip.div(255) - torch.as_tensor(KINETICS_MEAN).reshape(shape)) / torch.as_tensor(KINETICS_STD).reshape(shape)


@functools.lru_cache(maxsize=None)
def _stand_in(seed: int):
    import torchvision
    with torch.random.fork_rng(devices=[]):
        torch.manual_seed(seed)
        net = torchvision.models.video.r2plus1d_18(weights=None)
    g = torch.Generator().manual_seed(1000 + seed)
    for name, m in net.named_modules():
        if isinstance(m, torch.nn.BatchNorm3d):
            with torch.no_grad():
                gain = torch.rand(m.num_features, generator=g, dtype=torch.float64) + 0.5
                if name.endswith("conv2.1"):
                    gain = gain * 0.25
                m.weight.copy_(gain)
                m.bias.copy_(torch.randn(m.num_features, generator=g, dtype=torch.float64) * 0.1)
            m.momentum = None
            m.reset_running_stats()
    x = calibration_clips(seed)
    net.train()
    with torch.no_grad():
        net(x)
    net.eval()
    return {k: v.detach().clone() for k, v in net.state_dict().items()}


def stand_in_state_dict(seed: int = 0):
    """Calibrated seeded stand-in for the Kinetics weights of torchvision r2plus1d_18 (no trained weights exist
    offline): (1) torchvision's init under torch.manual_seed(seed); (2) BatchNorm gains ~ U(0.5, 1.5), times 0.25 on
    the last BatchNorm of every residual branch (layerX.Y.conv2.1), biases ~ N(0, 0.1); (3) running statistics = the
    batch statistics of one train-mode pass (momentum None) over 3 seeded 8-frame clips (calibration_clips).  Same keys
    and shapes as the torchvision state_dict (fc included).  Returns a fresh copy."""
    return {k: v.clone() for k, v in _stand_in(seed).items()}

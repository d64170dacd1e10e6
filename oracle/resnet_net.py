"""Plain-torch restatement of the reference's ResNet feature path (models/resnet/extract_resnet.py): the torchvision
ResNet-18/34/50/101/152 trunk with ``fc = Identity`` in eval mode, its per-frame transform, and a calibrated seeded
stand-in for the ImageNet weights.  Test infrastructure (the checker), never imported by the product."""
import functools
import hashlib

import numpy as np
import torch
import torch.nn.functional as F

# torchvision resnet.py: block type and blocks per stage
LAYERS = {18: (False, (2, 2, 2, 2)), 34: (False, (3, 4, 6, 3)), 50: (True, (3, 4, 6, 3)),
          101: (True, (3, 4, 23, 3)), 152: (True, (3, 8, 36, 3))}
MEAN, STD = [0.485, 0.456, 0.406], [0.229, 0.224, 0.225]
STAGES = ("stem", "maxpool", "layer1", "layer2", "layer3", "layer4")     # vf_resnet_read_stage ids 0..5


def out_dim(depth: int) -> int:
    return 2048 if LAYERS[depth][0] else 512


def _bn(sd, p, x):
    return F.batch_norm(x, sd[p + ".running_mean"], sd[p + ".running_var"], sd[p + ".weight"], sd[p + ".bias"],
                        False, 0.0, 1e-5)


def _block(sd, p, x, bottleneck, stride):
    if bottleneck:      # v1.5: the stride sits on the 3x3
        y = F.relu(_bn(sd, p + ".bn1", F.conv2d(x, sd[p + ".conv1.weight"])))
        y = F.relu(_bn(sd, p + ".bn2", F.conv2d(y, sd[p + ".conv2.weight"], stride=stride, padding=1)))
        y = _bn(sd, p + ".bn3", F.conv2d(y, sd[p + ".conv3.weight"]))
    else:
        y = F.relu(_bn(sd, p + ".bn1", F.conv2d(x, sd[p + ".conv1.weight"], stride=stride, padding=1)))
        y = _bn(sd, p + ".bn2", F.conv2d(y, sd[p + ".conv2.weight"], padding=1))
    if p + ".downsample.0.weight" in sd:
        x = _bn(sd, p + ".downsample.1", F.conv2d(x, sd[p + ".downsample.0.weight"], stride=stride))
    return F.relu(x + y)


def forward(sd, x, depth: int, taps: bool = False):
    """x: (n, 3, 224, 224) normalised -> (n, D) features; with ``taps`` also {stage name: activation}."""
    sd = {k[7:] if k.startswith("module.") else k: v for k, v in sd.items()}
    bottleneck, layers = LAYERS[depth]
    st = {}
    x = F.relu(_bn(sd, "bn1", F.conv2d(x, sd["conv1.weight"], stride=2, padding=3)))
    st["stem"] = x
    x = F.max_pool2d(x, 3, 2, 1)
    st["maxpool"] = x
    for L, nb in enumerate(layers):
        for b in range(nb):
            x = _block(sd, f"layer{L + 1}.{b}", x, bottleneck, 2 if (b == 0 and L > 0) else 1)
        st[f"layer{L + 1}"] = x
    y = torch.flatten(F.adaptive_avg_pool2d(x, 1), 1)
    return (y, st) if taps else y


def resize_geometry(h: int, w: int, size: int = 256):
    """torchvision Resize(int) on a PIL image: short side -> size, long side int(size * long / short)."""
    if h <= w:
        return size, int(size * w / h)
    return int(size * h / w), size


def crop_offset(d: int, crop: int = 224) -> int:
    return int(round((d - crop) / 2.0))


def normalize(rgb_u8: np.ndarray) -> torch.Tensor:
    """(H, W, 3) uint8 RGB, already resized -> CenterCrop(224) -> ToTensor -> Normalize, torchvision's fp32 op order."""
    h, w = rgb_u8.shape[:2]
    cy, cx = crop_offset(h), crop_offset(w)
    t = torch.from_numpy(np.ascontiguousarray(rgb_u8[cy:cy + 224, cx:cx + 224])).permute(2, 0, 1).contiguous()
    t = t.to(torch.float32).div(255)
    mean = torch.as_tensor(MEAN, dtype=torch.float32)[:, None, None]
    std = torch.as_tensor(STD, dtype=torch.float32)[:, None, None]
    return t.sub(mean).div(std)


def transform(bgr_u8: np.ndarray) -> torch.Tensor:
    """One decoded (BGR) frame through the reference transform: BGR->RGB, ToPILImage, Resize(256) (Pillow bilinear),
    CenterCrop(224), ToTensor, Normalize -> (3, 224, 224) fp32."""
    from PIL import Image
    rgb = np.ascontiguousarray(bgr_u8[:, :, ::-1])
    oh, ow = resize_geometry(*rgb.shape[:2])
    return normalize(np.asarray(Image.fromarray(rgb).resize((ow, oh), Image.BILINEAR)))


def tensor_hash(t: torch.Tensor) -> str:
    """sha1 of the fp32 bytes of one transformed frame (fixture key for bit-exact transform checks)."""
    return hashlib.sha1(t.contiguous().numpy().astype(np.float32).tobytes()).hexdigest()


@functools.lru_cache(maxsize=None)
def _stand_in(depth: int, seed: int):
    import torchvision
    with torch.random.fork_rng(devices=[]):
        torch.manual_seed(seed)
        net = getattr(torchvision.models, f"resnet{depth}")(weights=None)
    g = torch.Generator().manual_seed(1000 + seed)
    last = "bn3" if LAYERS[depth][0] else "bn2"
    for name, m in net.named_modules():
        if isinstance(m, torch.nn.BatchNorm2d):
            with torch.no_grad():
                gain = torch.rand(m.num_features, generator=g, dtype=torch.float64) + 0.5
                if name.endswith(last):
                    gain = gain * 0.25
                m.weight.copy_(gain)
                m.bias.copy_(torch.randn(m.num_features, generator=g, dtype=torch.float64) * 0.1)
            m.momentum = None
            m.reset_running_stats()
    x = calibration_images(seed)
    net.train()
    with torch.no_grad():
        net(x)
    net.eval()
    return {k: v.detach().clone() for k, v in net.state_dict().items()}


def calibration_images(seed: int = 0, n: int = 16) -> torch.Tensor:
    """n seeded normalised 224x224 images: smooth random fields plus pixel noise, quantised to uint8 like a frame."""
    g = torch.Generator().manual_seed(2000 + seed)
    low = torch.rand(n, 3, 14, 14, generator=g)
    img = F.interpolate(low, size=(224, 224), mode="bilinear", align_corners=False)
    img = (img * 0.8 + 0.2 * torch.rand(n, 3, 224, 224, generator=g)).mul(255).round().clamp(0, 255)
    mean = torch.as_tensor(MEAN)[:, None, None]
    std = torch.as_tensor(STD)[:, None, None]
    return img.div(255).sub(mean).div(std)


def stand_in_state_dict(depth: int, seed: int = 0):
    """Calibrated seeded stand-in for the ImageNet weights of torchvision resnet{depth} (no trained weights exist
    offline; a random-init ResNet with eval BatchNorm at mean 0 / var 1 is far too ill-conditioned to test against):
    (1) torchvision's init under torch.manual_seed(seed); (2) BatchNorm gains ~ U(0.5, 1.5), times 0.25 on the last
    BatchNorm of every residual branch (bn3 of a bottleneck, bn2 of a basic block: trained ResNets damp their branches
    this way), biases ~ N(0, 0.1); (3) running statistics = the cumulative batch statistics of one train-mode pass
    (momentum None) over 16 seeded normalised images (calibration_images).  Same keys and shapes as the torchvision
    state_dict (fc included).  Returns a fresh copy."""
    return {k: v.clone() for k, v in _stand_in(depth, seed).items()}

"""Reference for the IG65M R(2+1)D-34 models (upstream video_features' `r2plus1d_34_{32,8}_ig65m_ft_kinetics`), beside
oracle/r21d_net.py, which restates r2plus1d_18 and is left as it is.  The network is torchvision's
``VideoResNet(BasicBlock, [Conv2Plus1D] * 4, [3, 4, 6, 3], R2Plus1dStem)`` with fc 512 -> 400 and the two changes of
the ig65m-pytorch definition as it is recalled (no copy exists here to check against): layerL.0.conv2[0] of layer2..4
is Conv2Plus1D(planes, planes, 288 / 576 / 1152) (torchvision's formula, which those blocks' conv1 keeps, gives 230 /
460 / 921), and every BatchNorm3d has eps 1e-3.

forward() takes the blocks per stage and the eps, so with LAYERS_18 and 1e-5 it is r21d_net.forward bit for bit
(test_r21d_34_cpu.py); the transform, the calibration clips and the slicing are r21d_net's.  Test infrastructure, never
imported by the product."""
import functools

import torch
import torch.nn.functional as F

from oracle import r21d_net

LAYERS_18 = (2, 2, 2, 2)
LAYERS_34 = (3, 4, 6, 3)
EPS_34 = 1e-3                                   # every BatchNorm3d of the IG65M R(2+1)D-34 models
MID2_34 = {2: 288, 3: 576, 4: 1152}             # layerL.0.conv2's mid width (torchvision's formula: 230, 460, 921)
NET_34 = dict(eps=EPS_34, layers=LAYERS_34)     # forward()'s network arguments for R(2+1)D-34


def _bn(sd, p, x, eps):
    return F.batch_norm(x, sd[p + ".running_mean"], sd[p + ".running_var"], sd[p + ".weight"], sd[p + ".bias"],
                        False, 0.0, eps)


def _conv2plus1d(sd, p, x, stride, eps):
    """Conv2Plus1D: (1,3,3) spatial conv -> BN -> ReLU -> (3,1,1) temporal conv (torchvision video_resnet.py)."""
    x = F.relu(_bn(sd, p + ".1", F.conv3d(x, sd[p + ".0.weight"], stride=(1, stride, stride), padding=(0, 1, 1)), eps))
    return F.conv3d(x, sd[p + ".3.weight"], stride=(stride, 1, 1), padding=(1, 0, 0))


def _block(sd, p, x, stride, eps):
    y = F.relu(_bn(sd, p + ".conv1.1", _conv2plus1d(sd, p + ".conv1.0", x, stride, eps), eps))
    y = _bn(sd, p + ".conv2.1", _conv2plus1d(sd, p + ".conv2.0", y, 1, eps), eps)
    if p + ".downsample.0.weight" in sd:
        x = _bn(sd, p + ".downsample.1", F.conv3d(x, sd[p + ".downsample.0.weight"], stride=stride), eps)
    return F.relu(x + y)


def forward(sd, x, taps: bool = False, eps: float = EPS_34, layers=LAYERS_34):
    """x: (n, 3, T, 112, 112) normalised -> (n, 512) features; with ``taps`` also {stage name: activation} under
    r21d_net.STAGES (a stage's last block).  ``eps``: every BatchNorm's; ``layers``: blocks per stage."""
    sd = {k[7:] if k.startswith("module.") else k: v for k, v in sd.items()}
    st = {}
    x = F.relu(_bn(sd, "stem.1", F.conv3d(x, sd["stem.0.weight"], stride=(1, 2, 2), padding=(0, 3, 3)), eps))
    x = F.relu(_bn(sd, "stem.4", F.conv3d(x, sd["stem.3.weight"], padding=(1, 0, 0)), eps))
    st["stem"] = x
    for L in range(4):
        for b in range(layers[L]):
            x = _block(sd, f"layer{L + 1}.{b}", x, 2 if (b == 0 and L > 0) else 1, eps)
        st[f"layer{L + 1}"] = x
    y = torch.flatten(F.adaptive_avg_pool3d(x, 1), 1)
    return (y, st) if taps else y


def r2plus1d_34():
    """The R(2+1)D-34 module above (fc 512 -> 400), its convs initialised as VideoResNet initialises them."""
    from torchvision.models.video.resnet import BasicBlock, Conv2Plus1D, R2Plus1dStem, VideoResNet
    net = VideoResNet(BasicBlock, [Conv2Plus1D] * 4, list(LAYERS_34), R2Plus1dStem, num_classes=400)
    for L, mid in MID2_34.items():
        planes = r21d_net.COUT[L - 1]
        conv = Conv2Plus1D(planes, planes, mid)
        for m in conv.modules():
            if isinstance(m, torch.nn.Conv3d):
                torch.nn.init.kaiming_normal_(m.weight, mode="fan_out", nonlinearity="relu")
        getattr(net, f"layer{L}")[0].conv2[0] = conv
    for m in net.modules():
        if isinstance(m, torch.nn.BatchNorm3d):
            m.eps = EPS_34
    return net


@functools.lru_cache(maxsize=None)
def _stand_in(seed: int):
    with torch.random.fork_rng(devices=[]):
        torch.manual_seed(seed)
        net = r2plus1d_34()
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
    x = r21d_net.calibration_clips(seed)
    net.train()
    with torch.no_grad():
        net(x)
    net.eval()
    return {k: v.detach().clone() for k, v in net.state_dict().items()}


def stand_in_state_dict_34(seed: int = 0):
    """Calibrated seeded stand-in for the IG65M R(2+1)D-34 weights, built as r21d_net.stand_in_state_dict builds
    r2plus1d_18's: (1) r2plus1d_34()'s init under torch.manual_seed(seed); (2) BatchNorm gains ~ U(0.5, 1.5), times 0.25
    on layerX.Y.conv2.1, biases ~ N(0, 0.1); (3) running statistics = the batch statistics of one train-mode pass over
    r21d_net.calibration_clips(seed).  torchvision keys, fc at 400.  Returns a fresh copy."""
    return {k: v.clone() for k, v in _stand_in(seed).items()}

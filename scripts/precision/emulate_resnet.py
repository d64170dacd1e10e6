"""CPU emulation of the ResNet trunk's operand precision (decides DESIGN.md §4.6's split scheme).

    python scripts/precision/emulate_resnet.py [--depths 18 34 50 101 152] [--frames 4]

The reference (float64 forward of oracle/resnet_net.py's stand-in, BatchNorm in full precision) is compared with the
same forward whose conv operands are rounded per tensor class: 'fp16' rounds the class to one fp16 value, 'split'
to fp32 (a split-fp16 pair hi + lo carries ~22 mantissa bits, fp32 has 24).  Classes:
  stem   the stem conv's input          w      every conv weight
  c1x1   inputs of the 1x1 convs (bottleneck conv1 / conv3)
  c3x3   inputs of the 3x3 convs        down   the downsample conv's input
  resid  the block input on the identity path of x + branch(x) (the residual stream)
Printed per depth and scheme: the worst per-row rel-L2 and max-abs / max|ref| over the frames, against the project's
bar (rel-L2 <= 1e-3 and max-abs <= 1e-3 max per row).
"""
import argparse
import os
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import resnet_net  # noqa: E402

CLASSES = ("stem", "c1x1", "c3x3", "down", "resid", "w")


def _q(x, mode):
    if mode == "fp16":
        return x.half().double()
    return x.float().double()


def forward(sd, x, depth, scheme):
    """scheme: class -> 'fp16' | 'split'.  Float64 arithmetic with operands rounded per class."""
    bottleneck, layers = resnet_net.LAYERS[depth]
    W = {k: (_q(v, scheme["w"]) if k.endswith("conv1.weight") or ".conv" in k or "downsample.0" in k else v)
         for k, v in sd.items()}

    def bn(p, y):
        return F.batch_norm(y, sd[p + ".running_mean"], sd[p + ".running_var"], sd[p + ".weight"], sd[p + ".bias"],
                            False, 0.0, 1e-5)

    def conv(y, key, cls, **kw):
        return F.conv2d(_q(y, scheme[cls]), W[key], **kw)

    y = F.relu(bn("bn1", conv(x, "conv1.weight", "stem", stride=2, padding=3)))
    y = F.max_pool2d(y, 3, 2, 1)
    for L, nb in enumerate(layers):
        for b in range(nb):
            p, s = f"layer{L + 1}.{b}", (2 if (b == 0 and L > 0) else 1)
            if bottleneck:
                t = F.relu(bn(p + ".bn1", conv(y, p + ".conv1.weight", "c1x1")))
                t = F.relu(bn(p + ".bn2", conv(t, p + ".conv2.weight", "c3x3", stride=s, padding=1)))
                t = bn(p + ".bn3", conv(t, p + ".conv3.weight", "c1x1"))
            else:
                t = F.relu(bn(p + ".bn1", conv(y, p + ".conv1.weight", "c3x3", stride=s, padding=1)))
                t = bn(p + ".bn2", conv(t, p + ".conv2.weight", "c3x3", padding=1))
            if p + ".downsample.0.weight" in sd:
                r = bn(p + ".downsample.1", conv(y, p + ".downsample.0.weight", "down", stride=s))
            else:
                r = _q(y, scheme["resid"])
            y = F.relu(r + t)
    return torch.flatten(F.adaptive_avg_pool2d(y, 1), 1)


def errors(y, ref):
    rel = ((y - ref).norm(dim=1) / ref.norm(dim=1)).max().item()
    mx = ((y - ref).abs().amax(dim=1) / ref.abs().amax(dim=1)).max().item()
    return rel, mx


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--depths", type=int, nargs="+", default=[18, 34, 50, 101, 152])
    ap.add_argument("--frames", type=int, default=4)
    a = ap.parse_args()
    torch.set_grad_enabled(False)
    x = resnet_net.calibration_images(seed=5, n=a.frames).double()
    schemes = {"all split (engine)": {c: "split" for c in CLASSES}, "all fp16": {c: "fp16" for c in CLASSES}}
    for c in CLASSES:
        schemes[f"fp16 {c} only"] = dict({k: "split" for k in CLASSES}, **{c: "fp16"})
    for depth in a.depths:
        sd = {k: v.double() if v.is_floating_point() else v for k, v in resnet_net.stand_in_state_dict(depth).items()}
        ref = resnet_net.forward(sd, x, depth)
        for name, sc in schemes.items():
            rel, mx = errors(forward(sd, x, depth, sc), ref)
            ok = "ok  " if rel <= 1e-3 and mx <= 1e-3 else "MISS"
            print(f"resnet{depth:<3d} {name:<20s} rel-L2 {rel:.1e}  max-abs/max {mx:.1e}  {ok}", flush=True)


if __name__ == "__main__":
    main()

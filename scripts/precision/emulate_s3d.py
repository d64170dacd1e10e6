"""CPU emulation of the S3D trunk's operand precision (decides DESIGN.md §4.12's split scheme).

    python scripts/precision/emulate_s3d.py [--clips 1] [--T 16]

The reference (float64 forward of oracle/s3d_net.py's stand-in, BatchNorm in full precision) is compared with the
same forward whose conv operands are rounded per tensor class: 'fp16' rounds the class to one fp16 value, 'split'
to fp32 (a split-fp16 pair hi + lo carries ~22 mantissa bits, fp32 has 24).  A max pool picks one of its inputs, so
rounding a pool's output is rounding the tensor it reads.  Classes:
  stem    the stem's (1,7,7) conv input (the transformed clip)
  stemt   the stem's (7,1,1) temporal conv input
  f2in    the first pool's output, read by features.2 (1x1x1)
  spat    inputs of the (1,3,3) spatial convs (features.2's output, every Mixed 1x1x1 reducer's output)
  temp    inputs of the (3,1,1) temporal convs (features.3's and every Mixed branch's spatial conv output)
  concat  the Mixed blocks' inputs: the second pool's output and every Mixed output (and pool3 / pool4 outputs), read
          by the 1x1x1 convs of the next block
  pool3   the Mixed blocks' branch-3 (3,3,3) pool outputs, read by branch3's 1x1x1 conv
  w       every conv weight
Printed per scheme: the worst per-clip rel-L2 and max-abs / max|ref| of the features, against the project's bar
(rel-L2 <= 1e-3 and max-abs <= 1e-3 max per row).
"""
import argparse
import os
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import s3d_net  # noqa: E402

CLASSES = ("stem", "stemt", "f2in", "spat", "temp", "concat", "pool3", "w")


def _q(x, mode):
    if mode == "fp16":
        return x.half().double()
    return x.float().double()


def forward(sd, x, scheme, taps=False):
    """scheme: class -> 'fp16' | 'split'.  Float64 arithmetic with operands rounded per class.  With ``taps`` also
    {stage name: activation} under oracle/s3d_net.py's STAGES names."""
    W = {k: (_q(v, scheme["w"]) if k.endswith("weight") and v.dim() == 5 else v) for k, v in sd.items()}

    def cna(y, p, cls, stride=1, padding=0):
        y = F.conv3d(_q(y, scheme[cls]), W[p + ".0.weight"], stride=stride, padding=padding)
        y = F.batch_norm(y, sd[p + ".1.running_mean"], sd[p + ".1.running_var"], sd[p + ".1.weight"],
                         sd[p + ".1.bias"], False, 0.0, s3d_net.EPS)
        return F.relu(y)

    def sep(y, p, in_cls):
        return cna(cna(y, p + ".0", in_cls, 1, (0, 1, 1)), p + ".1", "temp", 1, (1, 0, 0))

    def mixed(y, p):
        x0 = cna(y, p + ".branch0", "concat")
        x1 = sep(cna(y, p + ".branch1.0", "concat"), p + ".branch1.1", "spat")
        x2 = sep(cna(y, p + ".branch2.0", "concat"), p + ".branch2.1", "spat")
        x3 = cna(F.max_pool3d(y, 3, 1, 1), p + ".branch3.1", "pool3")
        return torch.cat((x0, x1, x2, x3), 1)

    st = {}
    y = cna(x, "features.0.0", "stem", (1, 2, 2), (0, 3, 3))
    y = cna(y, "features.0.1", "stemt", (2, 1, 1), (3, 0, 0))
    st["stem"] = y
    y = cna(F.max_pool3d(y, (1, 3, 3), (1, 2, 2), (0, 1, 1)), "features.2", "f2in")
    y = sep(y, "features.3", "spat")
    st["features3"] = y
    y = F.max_pool3d(y, (1, 3, 3), (1, 2, 2), (0, 1, 1))
    for i in (5, 6):
        y = mixed(y, f"features.{i}")
    st["mixed_3c"] = y
    y = F.max_pool3d(y, 3, 2, 1)
    for i in (8, 9, 10, 11, 12):
        y = mixed(y, f"features.{i}")
    st["mixed_4f"] = y
    y = F.max_pool3d(y, 2, 2, 0)
    for i in (14, 15):
        y = mixed(y, f"features.{i}")
    st["mixed_5c"] = y
    out = F.avg_pool3d(y, (2, 7, 7), 1).mean(dim=(2, 3, 4))
    return (out, st) if taps else out


def errors(y, ref):
    rel = ((y - ref).norm(dim=1) / ref.norm(dim=1)).max().item()
    mx = ((y - ref).abs().amax(dim=1) / ref.abs().amax(dim=1)).max().item()
    return rel, mx


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--clips", type=int, default=1)
    ap.add_argument("--T", type=int, default=16)
    a = ap.parse_args()
    torch.set_grad_enabled(False)
    x = s3d_net.calibration_clips(seed=5, n=a.clips, T=a.T).double()
    sd = {k: v.double() if v.is_floating_point() else v for k, v in s3d_net.stand_in_state_dict().items()}
    ref, rtaps = s3d_net.forward(sd, x, taps=True)
    schemes = {"all split (engine)": {c: "split" for c in CLASSES}, "all fp16": {c: "fp16" for c in CLASSES}}
    for c in CLASSES:
        schemes[f"fp16 {c} only"] = dict({k: "split" for k in CLASSES}, **{c: "fp16"})
    for name, sc in schemes.items():
        y, taps = forward(sd, x, sc, taps=True)
        rel, mx = errors(y, ref)
        ok = "ok  " if rel <= 1e-3 and mx <= 1e-3 else "MISS"
        stages = "  ".join(f"{s} {errors(taps[s].flatten(1), rtaps[s].flatten(1))[0]:.1e}" for s in s3d_net.STAGES)
        print(f"s3d {name:<20s} features rel-L2 {rel:.1e}  max-abs/max {mx:.1e}  {ok} | {stages}", flush=True)


if __name__ == "__main__":
    main()

"""CPU emulation of the R(2+1)D trunk's operand precision (decides DESIGN.md §4.7's split scheme).

    python scripts/precision/emulate_r21d.py [--clips 2] [--T 16] [--depth 18 | 34]

--depth 34 runs the IG65M R(2+1)D-34 stand-in (tests/r21d_34_ref.py stand_in_state_dict_34: blocks 3, 4, 6, 3,
BatchNorm eps 1e-3) against that module's float64 forward.

The reference (float64 forward of oracle/r21d_net.py's stand-in, BatchNorm in full precision) is compared with the
same forward whose conv operands are rounded per tensor class: 'fp16' rounds the class to one fp16 value, 'split'
to fp32 (a split-fp16 pair hi + lo carries ~22 mantissa bits, fp32 has 24).  Classes:
  stem   the stem's (1,7,7) conv input     spat   inputs of the (1,3,3) spatial convs (block inputs, conv2 inputs)
  temp   inputs of the (3,1,1) temporal convs (the stem's too)
  down   the downsample conv's input       resid  the block input on the identity path (the residual stream)
  w      every conv weight
Printed per scheme: the worst per-row rel-L2 and max-abs / max|ref| over the clips, against the project's bar
(rel-L2 <= 1e-3 and max-abs <= 1e-3 max per row).  The 'lo-skip' scheme is the engine's arithmetic more closely: every
operand is the fp16 pair hi + lo of its fp32 value, and every conv drops the a_lo . w_lo products (the W_lo pass the
engine skips on K blocks that meet only lo halves), computing conv(a_hi, w_hi + w_lo) + conv(a_lo, w_hi).
"""
import argparse
import os
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import r21d_34_ref as ref34  # noqa: E402
from oracle import r21d_net  # noqa: E402

CLASSES = ("stem", "spat", "temp", "down", "resid", "w")


def _q(x, mode):
    if mode == "fp16":
        return x.half().double()
    if mode == "pair":
        return sum(_pair(x))
    return x.float().double()


def _pair(x):
    """The split-fp16 pair (hi, lo) of x's fp32 value, as the GEMM epilogue and the weight upload make it."""
    v = x.float().double()
    hi = v.half().double()
    return hi, (v - hi).half().double()


def forward(sd, x, scheme, taps=False, eps=1e-5, layers=ref34.LAYERS_18, lo_skip=False):
    """scheme: class -> 'fp16' | 'split' | 'pair'.  Float64 arithmetic with operands rounded per class.  With ``taps``
    also {stage name: activation} under oracle/r21d_net.py's STAGES names.  ``lo_skip``: every conv drops a_lo . w_lo
    (operands as pairs)."""
    W = {k: (_q(v, scheme["w"]) if k.endswith("weight") and v.dim() == 5 else v) for k, v in sd.items()}
    W_hi = {k: _pair(v)[0] for k, v in sd.items() if k.endswith("weight") and v.dim() == 5} if lo_skip else {}

    def bn(p, y):
        return F.batch_norm(y, sd[p + ".running_mean"], sd[p + ".running_var"], sd[p + ".weight"], sd[p + ".bias"],
                            False, 0.0, eps)

    def conv(y, key, cls, **kw):
        if lo_skip:
            hi, lo = _pair(y)
            return F.conv3d(hi, W[key], **kw) + F.conv3d(lo, W_hi[key], **kw)
        return F.conv3d(_q(y, scheme[cls]), W[key], **kw)

    def c2p1(y, p, s):
        y = F.relu(bn(p + ".1", conv(y, p + ".0.weight", "spat", stride=(1, s, s), padding=(0, 1, 1))))
        return conv(y, p + ".3.weight", "temp", stride=(s, 1, 1), padding=(1, 0, 0))

    y = F.relu(bn("stem.1", conv(x, "stem.0.weight", "stem", stride=(1, 2, 2), padding=(0, 3, 3))))
    y = F.relu(bn("stem.4", conv(y, "stem.3.weight", "temp", padding=(1, 0, 0))))
    st = {"stem": y}
    for L in range(4):
        for b in range(layers[L]):
            p, s = f"layer{L + 1}.{b}", (2 if (b == 0 and L > 0) else 1)
            t = F.relu(bn(p + ".conv1.1", c2p1(y, p + ".conv1.0", s)))
            t = bn(p + ".conv2.1", c2p1(t, p + ".conv2.0", 1))
            if p + ".downsample.0.weight" in sd:
                r = bn(p + ".downsample.1", conv(y, p + ".downsample.0.weight", "down", stride=s))
            else:
                r = _q(y, scheme["resid"])
            y = F.relu(r + t)
        st[f"layer{L + 1}"] = y
    out = torch.flatten(F.adaptive_avg_pool3d(y, 1), 1)
    return (out, st) if taps else out


def errors(y, ref):
    rel = ((y - ref).norm(dim=1) / ref.norm(dim=1)).max().item()
    mx = ((y - ref).abs().amax(dim=1) / ref.abs().amax(dim=1)).max().item()
    return rel, mx


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--clips", type=int, default=2)
    ap.add_argument("--T", type=int, default=16)
    ap.add_argument("--depth", type=int, choices=[18, 34], default=18)
    a = ap.parse_args()
    torch.set_grad_enabled(False)
    x = r21d_net.calibration_clips(seed=5, n=a.clips, T=a.T).double()
    if a.depth == 18:
        sd, net = r21d_net.stand_in_state_dict(), dict(eps=1e-5, layers=ref34.LAYERS_18)
    else:
        sd, net = ref34.stand_in_state_dict_34(), ref34.NET_34
    sd = {k: v.double() if v.is_floating_point() else v for k, v in sd.items()}
    ref = ref34.forward(sd, x, **net)      # at depth 18 this is r21d_net.forward bit for bit
    schemes = {"all split (engine)": ({c: "split" for c in CLASSES}, False),
               "lo-skip (engine)": ({c: "pair" for c in CLASSES}, True),
               "all fp16": ({c: "fp16" for c in CLASSES}, False)}
    for c in CLASSES:
        schemes[f"fp16 {c} only"] = (dict({k: "split" for k in CLASSES}, **{c: "fp16"}), False)
    tag = f"r21d-{a.depth} T={a.T}"
    for name, (sc, skip) in schemes.items():
        rel, mx = errors(forward(sd, x, sc, lo_skip=skip, **net), ref)
        ok = "ok  " if rel <= 1e-3 and mx <= 1e-3 else "MISS"
        print(f"{tag} {name:<20s} rel-L2 {rel:.1e}  max-abs/max {mx:.1e} ({max(rel, mx) / 1e-3:.4f} of the bar) {ok}",
              flush=True)


if __name__ == "__main__":
    main()

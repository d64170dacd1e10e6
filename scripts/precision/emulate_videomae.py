"""Float64 emulation of the VideoMAE engine's rounding (DESIGN.md §4.18), to decide whether the GEMM weights can be
plain fp16 (the ping-pong GEMM) or must be split-fp16 pairs (split_linear).

    python scripts/precision/emulate_videomae.py [--models videomae_vits16 ...] [--clips 2] [--device cuda]

The stand-in network (oracle/videomae_net.py) runs in float64 with the operands of each tensor class either exact (a
split-fp16 pair carries ~22 bits, far below the bar) or rounded to one fp16 value:
  w       every GEMM weight (tubelet embedding, qkv, proj, fc1, fc2)
  tube    the tubelet rows (the transformed clip)
  ln      the layernorm_before / layernorm_after outputs
  qkv     q, k and v
  p       P = exp(s - running max) per 64-key block, multiplied into v (the sum stays exact)
  att     the attention output (proj's input)
  hidden  the MLP hidden layer (fc2's input)
For each model it prints, per scheme, the worst per-clip rel-L2 and max-abs / max at the feature against the exact
float64 forward: every class alone in fp16, the activations in fp16 with weights exact (the split-weight engine,
oracle ENGINE_FP16), and the same with plain fp16 weights.  The project bar is 1e-3 / 1e-3 at the features.
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle import videomae_net as V  # noqa: E402

ENGINE = V.ENGINE_FP16
PLAIN_FP16_WEIGHTS = ENGINE + ("w",)


def errors(y, ref):
    """(worst per-clip rel-L2, worst per-clip max-abs / max)."""
    d = y - ref
    return (d.norm(dim=1) / ref.norm(dim=1)).max().item(), (d.abs().amax(dim=1) / ref.abs().amax(dim=1)).max().item()


def table(name, n, device, schemes, depth=None):
    """{scheme label: (rel-L2, max-abs / max) at the feature} for the stand-in of `name` (``depth`` blocks, default
    all) on n calibration clips."""
    p = V.prepare(V.stand_in_state_dict(name, depth=depth), torch.float64, device)
    x = V.calibration_clips(0, n).double().to(device)
    with torch.no_grad():
        ref = V.forward(p, x)
        return {label: errors(V.forward(p, x, fp16=fp16), ref) for label, fp16 in schemes.items()}


def schemes():
    s = {c: (c,) for c in V.CLASSES}
    s["engine (split weights)"] = ENGINE
    s["plain fp16 weights"] = PLAIN_FP16_WEIGHTS
    return s


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--models", nargs="+", default=list(V.SHAPES))
    ap.add_argument("--clips", type=int, default=2)
    ap.add_argument("--device", default="cuda" if torch.cuda.is_available() else "cpu")
    ap.add_argument("--depth", type=int, default=None)
    a = ap.parse_args()
    for name in a.models:
        tab = table(name, a.clips, a.device, schemes(), a.depth)
        for label, (rel, mx) in tab.items():
            print(f"{name:16s} {label:24s} rel-L2 {rel:.2e}  max-abs/max {mx:.2e}", flush=True)
        print(json.dumps({"model": name, "table": tab}), flush=True)


if __name__ == "__main__":
    main()

"""Float64 emulation of the DINOv2 engine's declared rounding (DESIGN.md §4.17), to decide which tensor classes must be
carried as split-fp16 pairs (or fp32).

    python scripts/precision/emulate_dinov2.py [--models dinov2_vits14 ...] [--frames 2] [--device cpu]

The stand-in network (oracle/dinov2_net.py) runs in float64 with LayerScale folded as the engine folds it and the
operands of each tensor class either kept exact ("split": a split-fp16 pair carries ~22 bits, far below the bar; fp32
for the SwiGLU inputs) or rounded to one fp16 value:
  w       every GEMM weight (patch embedding, qkv, proj, fc1 / fc2 or w12 / w3)
  patch   the patch rows (the transformed frame)
  ln      the norm1 / norm2 outputs
  qkv     q, k and v
  p       P = exp(s - running max) per 64-key block, multiplied into v (the sum stays fp32)
  att     the attention output (proj's input)
  hidden  the FFN hidden layer (fc2 / w3's input)
  swiglu  g only: the w12 output (a, b) the SwiGLU kernel reads
For each model it prints, per scheme, the worst per-frame rel-L2 and max-abs / max at the feature against the exact
float64 forward -- all fp16, each class alone in fp16, and the engine's scheme (oracle ENGINE_FP16) -- and the largest
magnitude every fp16 class reaches (fp16 overflows at 65504).  The project bar is 1e-3 / 1e-3 at the features.
"""
import argparse
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle import dinov2_net as D  # noqa: E402

CLASSES = D.CLASSES
ENGINE = D.ENGINE_FP16
# the classes the engine does not round to one fp16 value
SPLIT = tuple(c for c in CLASSES if c not in ENGINE)


def classes_of(name):
    """The classes a model has (swiglu only for g)."""
    return tuple(c for c in CLASSES if c != "swiglu" or D.shape_of(name)[2] == "swiglu")


def errors(y, ref):
    """(worst per-frame rel-L2, worst per-frame max-abs / max)."""
    d = y - ref
    return (d.norm(dim=1) / ref.norm(dim=1)).max().item(), (d.abs().amax(dim=1) / ref.abs().amax(dim=1)).max().item()


def table(name, n, device, schemes, depth=None):
    """{scheme label: (rel-L2, max-abs / max) at the feature} for the stand-in of `name` (``depth`` blocks, default
    all) on n calibration frames."""
    sd = D.prepare(D.stand_in_state_dict(name, depth=depth), torch.float64, device)
    x = D.calibration_frames(0, n).double().to(device)
    with torch.no_grad():
        ref = D.forward(sd, x, (), True)
        return {label: errors(D.forward(sd, x, fp16, True), ref) for label, fp16 in schemes.items()}


def magnitudes(name, n, device, depth=None):
    """{class: largest |value|} of the tensors the engine rounds to fp16, on the exact forward."""
    sd = D.prepare(D.stand_in_state_dict(name, depth=depth), torch.float64, device)
    x = D.calibration_frames(0, n).double().to(device)
    peak = {}
    real_q = D._q

    def spy(t, cls, fp16):
        peak[cls] = max(peak.get(cls, 0.0), t.abs().max().item())
        return real_q(t, cls, fp16)
    D._q = spy
    try:
        with torch.no_grad():
            D.forward(sd, x, (), True)
    finally:
        D._q = real_q
    return peak


def schemes(name):
    cl = classes_of(name)
    s = {"all fp16": cl}
    s.update({f"{c} alone fp16": (c,) for c in cl})
    s[f"engine ({'+'.join(c for c in SPLIT if c in cl)} not fp16)"] = ENGINE
    return s


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--models", nargs="+", default=list(D.MODELS))
    ap.add_argument("--frames", type=int, default=2)
    ap.add_argument("--device", default="cpu")
    a = ap.parse_args()
    for name in a.models:
        tab = table(name, a.frames, a.device, schemes(name))
        print(f"{name}, {a.frames} calibration frames (feature rel-L2 / max-abs÷max):", flush=True)
        for label, (rel, mx) in tab.items():
            print(f"  {label:28s} {rel:.2e} / {mx:.2e}", flush=True)
        peak = magnitudes(name, a.frames, a.device)
        print("  largest |value| per class: " + ", ".join(f"{c} {v:.3g}" for c, v in sorted(peak.items())), flush=True)


if __name__ == "__main__":
    main()

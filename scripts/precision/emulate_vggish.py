"""CPU emulation of the VGGish trunk's operand precision (decides DESIGN.md §4.10's split scheme).

    python scripts/precision/emulate_vggish.py [--seconds 8]

The reference is the float64 forward of oracle/vggish_net.py's stand-in on the fp32 log-mel examples of seeded audio
(44.1 kHz stereo, resampled by the oracle).  Each variant rounds ONE tensor class to single fp16 and keeps the rest in
float64; 'all split' rounds every class to fp32 (a split-fp16 pair hi + lo carries ~22 mantissa bits, fp32 has 24).
Classes: input (conv1's log-mel input), conv_w, conv_act (inputs of conv2..6), fc_w, fc_act (inputs of fc1..3).
Printed: the worst per-example rel-L2 and max-abs / max|ref| of the features and of pool1, against the project's
feature bar (rel-L2 <= 1e-3 and max-abs <= 1e-3 max per row).
"""
import argparse
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import vggish_net  # noqa: E402

CLASSES = ("input", "conv_w", "conv_act", "fc_w", "fc_act")


def errs(y, ref):
    d = (y - ref).flatten(1)
    r = ref.flatten(1)
    return (d.norm(dim=1) / r.norm(dim=1)).max().item(), (d.abs().amax(1) / r.abs().amax(1)).max().item()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=8.0)
    a = ap.parse_args()
    x = vggish_net.synthetic_audio(a.seconds, 44100, 2, seed=21)
    ex = torch.from_numpy(vggish_net.examples(x, 44100)).double()
    sd = {k: v.double() for k, v in vggish_net.stand_in_state_dict().items()}
    with torch.no_grad():
        ref, st = vggish_net.forward(sd, ex, taps=True)
        variants = [(f"{c} fp16", {c: torch.float16}) for c in CLASSES]
        variants.append(("all split (fp32)", {c: torch.float32 for c in CLASSES}))
        print(f"{ex.shape[0]} examples; worst row rel-L2 / max-abs÷max")
        print(f"{'variant':<20} {'pool1':>22} {'features':>22}  within 1e-3")
        for name, rounding in variants:
            y, s = vggish_net.forward(sd, ex, taps=True, rounding=rounding)
            p, f = errs(s[0], st[0]), errs(y, ref)
            print(f"{name:<20} {p[0]:>10.2e} / {p[1]:.2e} {f[0]:>10.2e} / {f[1]:.2e}  {f[0] <= 1e-3 and f[1] <= 1e-3}")


if __name__ == "__main__":
    main()

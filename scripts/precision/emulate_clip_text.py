"""Float64 emulation of the CLIP text tower's declared rounding (DESIGN.md §4.16), to decide per GEMM whether its
weights are single fp16 values or split-fp16 pairs.

    python scripts/precision/emulate_clip_text.py [--prompts 64] [--seed 0]

The synthetic towers (synthetic_weights.clip_text_state_dict) at the three released geometries run in float64
(oracle/clip_text.py) on seeded prompts of 6..20 ids whose EOT is the vocabulary's largest id.  The activations the
engine stores in fp16 (LayerNorm outputs, q / k / v, the attention output, fc1 after QuickGELU) are rounded in every
scheme; the schemes differ in the GEMM weights: all split (the engine), all fp16, and each GEMM alone in fp16.  Printed
per scheme: the worst row error of the normalised text features against the exact float64 tower, as max |dt| and
max ||dt||_2.  A zero-shot logit is 100 t.i with unit vectors, so its error is at most 100 ||dt||_2.
"""
import argparse
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle import clip_text as T  # noqa: E402
from video_features_b200 import synthetic_weights  # noqa: E402

GEOMETRIES = {"512/8": (512, 512), "640/10": (640, 640), "768/12": (768, 768)}
VOCAB = 1000


def prompts(n: int, seed: int):
    g = torch.Generator().manual_seed(seed)
    tokens = torch.zeros(n, 77, dtype=torch.int32)
    for b in range(n):
        k = int(torch.randint(6, 21, (1,), generator=g))
        tokens[b, 0] = VOCAB - 2
        tokens[b, 1:k - 1] = torch.randint(0, VOCAB - 2, (k - 2,), generator=g)
        tokens[b, k - 1] = VOCAB - 1
    return tokens


def errors(sd, tokens, exact, rounding):
    t = T.encode_text_declared(sd, tokens, rounding=rounding)
    d = t - exact
    return d.abs().max().item(), d.norm(dim=1).max().item()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--prompts", type=int, default=64)
    ap.add_argument("--seed", type=int, default=0)
    a = ap.parse_args()
    tokens = prompts(a.prompts, a.seed)
    for name, (width, embed) in GEOMETRIES.items():
        sd = synthetic_weights.clip_text_state_dict(a.seed, width, embed, VOCAB)
        exact = T.encode_text_declared(sd, tokens, rounding=T.Rounding(act=False))
        schemes = [("engine: weights split", T.Rounding()), ("all weights fp16", T.Rounding(fp16_weights=T.GEMMS))]
        schemes += [(f"{g} weights fp16", T.Rounding(fp16_weights=(g,))) for g in T.GEMMS]
        for label, r in schemes:
            mx, l2 = errors(sd, tokens, exact, r)
            print(f"{name:7s} {label:24s} max|dt| {mx:.2e}  max||dt|| {l2:.2e}  logit <= {100 * l2:.2e}", flush=True)


if __name__ == "__main__":
    main()

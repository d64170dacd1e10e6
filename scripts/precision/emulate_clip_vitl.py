"""Does the single-fp16 operand scheme of the ViT towers hold at the ViT-L/14 shape (DESIGN.md §4.13)?

    python scripts/precision/emulate_clip_vitl.py [--frames 2] [--seed 0] [--tiny]

For the synthetic weights (plain and outlier variants, video_features_b200/synthetic_weights.py) of ViT-B/32 (the
calibration row), ViT-L/14 at 224 px (257 tokens) and at 336 px (577 tokens), the tower in float64 with the engine's
declared fp16 rounding -- weights, patches, LayerNorm outputs, q / k / v, P, attention output, MLP hidden -- against the
same float64 tower with nothing rounded.  At L/14, P is the streamed attention kernel's: fp16(exp(s - running max)) per
block of 64 keys (tests/clip_vitl_ref.py).  Reports the worst row's rel-L2 / max-abs÷max of the features; the project's
bar is 1e-3 against the fp32 oracle.  --tiny runs a two-block tower of width 128 at 56 px (a smoke run).
"""
import argparse
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import clip_vitl_ref  # noqa: E402
from oracle import clip_resnet, clip_tower  # noqa: E402
from video_features_b200 import synthetic_weights  # noqa: E402


def row_err(y, ref):
    rel = ((y - ref).norm(dim=1) / ref.norm(dim=1)).max().item()
    mx = ((y - ref).abs().amax(dim=1) / ref.abs().amax(dim=1)).max().item()
    return rel, mx


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=2)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--tiny", action="store_true")
    a = ap.parse_args()
    if a.tiny:
        shapes = [("tiny", lambda s, o: synthetic_weights._vit_state_dict(s, o, 128, 2, 14, 56, 64), 56)]
        a.frames = 1
    else:
        shapes = [("B/32 (calibration)", lambda s, o: synthetic_weights.clip_vit_b32_state_dict(s, o), 224),
                  ("L/14 224 px, 257 tokens", lambda s, o: synthetic_weights.clip_vit_l14_state_dict(s, o, 224), 224),
                  ("L/14@336px, 577 tokens", lambda s, o: synthetic_weights.clip_vit_l14_state_dict(s, o, 336), 336)]
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    print(f"{'shape':26s} {'weights':9s} rel-L2     max-abs/max")
    for name, make, n_px in shapes:
        x = clip_resnet.calibration_images(n_px, a.seed, a.frames).double()
        for outliers in (False, True):
            sd = {k: v.double() for k, v in make(a.seed, outliers).items()}
            if name.startswith("B/32"):
                ref = clip_tower.encode_image_declared(sd, x, dtype=torch.float64, declared_rounding=False)
                y = clip_tower.encode_image_declared(sd, x, dtype=torch.float64, declared_rounding=True)
            else:
                ref = clip_vitl_ref.encode_image(sd, x, dtype=torch.float64)
                y = clip_vitl_ref.encode_image(sd, x, dtype=torch.float64, declared_rounding=True)
            rel, mx = row_err(y, ref)
            print(f"{name:26s} {'outliers' if outliers else 'plain':9s} {rel:.2e}   {mx:.2e}", flush=True)


if __name__ == "__main__":
    main()

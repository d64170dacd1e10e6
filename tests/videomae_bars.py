"""Bars of the VideoMAE engine (tests/test_videomae_gpu.py, tests/test_extract_videomae_gpu.py).  Each is (worst
per-row rel-L2, worst per-row max-abs / max).

FEATURES holds the engine against the exact float64 forward: the project's 1e-3 feature bar with 2x headroom.  "embed"
holds the tubelet embedding against float64 of the same fp16 tubelet rows (only the engine's fp32 arithmetic and its
split weights show).  "block" holds the residual update of one block run alone on the float64 chain's stream.  The
attention bars hold the wgmma kernel against the float64 reference of its declared rounding (tests/attention_ref.py,
64-key blocks): the max-abs part is about one fp16 ulp of the output, so its bar is two."""
FEATURES = {384: (7e-5, 8e-5), 768: (7e-5, 8e-5), 1024: (7e-5, 8e-5)}
BARS = {"embed": (6e-6, 8e-6), "block": (6e-4, 7.5e-4), "head": (3.5e-7, 6e-7),
        "attention": (1e-4, 1e-3), "attention hard": (6e-5, 1e-3)}
# About 2x the worst an H100 80GB HBM3 (700 W power limit) measured on the seeded stand-ins of S, B and L: features
# 3.0e-5 / 3.5e-5, embedding 2.7e-6 / 3.9e-6, one block's update 2.9e-4 / 3.6e-4, head 1.7e-7 / 2.8e-7; the attention
# at S in {1, 63, 64, 65, 1000, 1568, 2048} with 6 / 12 / 16 heads 4.8e-5 / 4.9e-4 (random) and 2.7e-5 / 4.7e-4 (hard).
PROJECT = (1e-3, 1e-3)
SEPARATION = 3.0          # a lost lo half must exceed the feature and embedding bars by this factor
SCHEME_FRACTION = 0.5     # the emulated split-weight scheme may cost this fraction of the feature bar
WEIGHT_DOMINANCE = 5.0    # fp16 weights cost at least this many times all the fp16 activations together

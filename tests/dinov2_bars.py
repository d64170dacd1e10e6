"""Bars of the DINOv2 engine (tests/test_dinov2_gpu.py), shared with their CPU companion (tests/test_dinov2_bars_cpu.py).
Each is (worst per-frame rel-L2, worst per-frame max-abs / max), about 2x the worst an H100 80GB HBM3 (700 W power
limit) measured over the eight stand-ins (DESIGN.md §4.17).

FEATURES holds the engine against the exact float64 forward, per width (g/14's 40 blocks and SwiGLU cost more; its bar
is the project's 1e-3).  The embedding and the head are checked against the float64 oracle of the declared rounding:
each is one step with no fp16 rounding after it, so only the engine's own arithmetic shows.  "blocks" holds the stream
after every 4th block of the engine's own chain against the same oracle; there the fp16 roundings that fall the other
way from fp32 vs float64 inputs add up like fresh rounding noise, so that bar is as wide as the feature's.  "block"
holds the residual update of one block run alone on the oracle's stream: those flips stay within one block, so it is
tight enough that weights rounded to fp16 exceed it (BLOCK_SEPARATION, rel-L2).  A lost lo half must exceed the
embedding bar by SEPARATION."""
FEATURES = {384: (7e-4, 9e-4), 768: (7e-4, 9e-4), 1024: (7e-4, 9e-4), 1536: (1e-3, 1e-3)}
BARS = {"embed": (3e-6, 4e-6), "blocks": (1.1e-3, 1.3e-3), "block": (2.6e-4, 5e-4), "head": (3e-7, 4e-7)}
PROJECT = (1e-3, 1e-3)
SEPARATION = 3.0
# "block" is 1.14-1.6x the engine's measured worst (1.7-2.3e-4 rel-L2), not 2x, so that it works as a control: fp16
# weights move one block's update by 4.6e-4 (S/14) and 5.1e-4 (g/14_reg), 1.8-2.0x the bar.  The activations' own
# fp16 flips are within about 2x of the weights' rounding, so the one-block control cannot separate by 3x
BLOCK_SEPARATION = 1.5
# The fraction of its FEATURES bar that the emulated scheme, and each single-fp16 class alone, may cost
# (scripts/precision/emulate_dinov2.py, tests/test_dinov2_bars_cpu.py).  Half for S, B and L.  g/14 is an explicit
# exception: its scheme costs 6.1e-4 / 7.8e-4 (78 % of the 1e-3 bar) and its norm outputs alone 4.2e-4 / 5.3e-4.  Only
# split-fp16 activations (LayerNorm outputs, FFN hidden layer) would lower that, at up to 1.5x the GEMM work of the
# model that already loses to torch's fp16 autocast; that is not built (DESIGN.md §4.17).
SCHEME_FRACTION = {384: 0.5, 768: 0.5, 1024: 0.5, 1536: 0.8}

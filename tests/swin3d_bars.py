"""Bars of the Swin3D engine against float64 (tests/test_swin3d_gpu.py), shared with their CPU companion
(tests/test_swin3d_bars_cpu.py).  Each is (worst per-clip rel-L2, worst per-clip max-abs / max), about 1.5-2x the worst
value an H100 80GB HBM3 (700 W power limit) measured over the t / s / b stand-ins at T = 32, 17 and 10 with every GEMM
weight a split-fp16 pair (DESIGN.md §4.14)."""
BARS = {"embed": (4.5e-4, 6e-4), "stage1": (6e-4, 9e-4), "stage2": (8e-4, 9e-4), "stage3": (8e-4, 1e-3),
        "stage4": (8e-4, 1.1e-3), "norm": (8e-4, 1.3e-3), "features": (1.2e-4, 1.5e-4),
        "attention hard": (3.5e-5, 1e-3)}
# "attention hard": the window-attention kernel alone on hard inputs (tests/test_attention_hard_gpu.py) against the
# float64 reference of its declared rounding (tests/attention_ref.py), every stage's C at T' = 16 / 9 / 5, shifted and
# not: measured 1.7e-5 / 4.8e-4 on the same H100 (the max-abs part one fp16 ulp of the output).  The kernel built
# with the -100 mask added in log2 units measured 0.11 / 0.92 or more where shift regions meet, without the rescale of
# its output 1.1 / 1.6.
# a lost lo half must exceed the feature bar by at least this factor, in both measures
SEPARATION = 3.0

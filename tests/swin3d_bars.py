"""Bars of the Swin3D engine against float64 (tests/test_swin3d_gpu.py), shared with their CPU companion
(tests/test_swin3d_bars_cpu.py).  Each is (worst per-clip rel-L2, worst per-clip max-abs / max), about 1.5-2x the worst
value an H100 80GB HBM3 (700 W power limit) measured over the t / s / b stand-ins at T = 32, 17 and 10 with every GEMM
weight a split-fp16 pair (DESIGN.md §4.14)."""
BARS = {"embed": (4.5e-4, 6e-4), "stage1": (6e-4, 9e-4), "stage2": (8e-4, 9e-4), "stage3": (8e-4, 1e-3),
        "stage4": (8e-4, 1.1e-3), "norm": (8e-4, 1.3e-3), "features": (1.2e-4, 1.5e-4)}
# a lost lo half must exceed the feature bar by at least this factor, in both measures
SEPARATION = 3.0

"""Bars of the S3D engine against a float64 forward of the same network (worst row: clip; rel-L2, max-abs / max|ref|),
shared by the GPU test (test_s3d_gpu.py) and the CPU check that they separate the engine's split scheme from every
single-fp16 tensor class of scripts/precision/emulate_s3d.py (test_s3d_bars_cpu.py).

Each bar sits 1.5x .. 2.3x above the worst value measured on one H100 80GB HBM3 (700 W power limit) over T = 64, 17, 16
and 13 with one and three clips (beside each bar).  The stand-in amplifies rounding errors from Mixed 3c on: fp32 torch
on the CPU goes 2.6e-6 (3c) -> 3.0e-5 (4f) -> 8.2e-5 (5c) against float64, the engine 3.7e-5 -> 4.9e-4 -> 1.3e-3 (its
fp32 tensor-core accumulation per conv is 1e-6 .. 1.5e-5, as for R(2+1)D).  The (2,7,7) average pool cancels most of it
again at the features."""

STAGES = ("stem", "features3", "mixed_3c", "mixed_4f", "mixed_5c", "features")
BARS = {"stem": (7e-6, 7e-6),               # 3.1e-6 / 3.4e-6
        "features3": (2.5e-5, 2.5e-5),      # 1.0e-5 / 1.1e-5
        "mixed_3c": (8e-5, 8e-5),           # 3.7e-5 / 3.8e-5
        "mixed_4f": (8e-4, 8.5e-4),         # 4.9e-4 / 5.4e-4
        "mixed_5c": (2e-3, 2.1e-3),         # 1.27e-3 / 1.39e-3
        "features": (6.5e-4, 1.3e-3)}       # 4.2e-4 / 8.1e-4 (T = 13 and 17: one or two pool positions)

# The first stage each emulated class (emulate_s3d.CLASSES) reaches, and how far above the bar (rel-L2 and max-abs)
# leaving that one class in single fp16 lies at every stage from there on, in the CPU float64 emulation of 1 clip x 16
# frames.  Measured minimum over the classes in parentheses; the Mixed blocks' branch-3 pool outputs are the closest
# class past Mixed 3c.
FIRST_STAGE = {"stem": "stem", "stemt": "stem", "w": "stem", "f2in": "features3", "spat": "features3",
               "temp": "features3", "concat": "mixed_3c", "pool3": "mixed_3c"}
SEPARATION = {"stem": 20,          # (37.8 / 49.3: fp16 stem temporal input)
              "features3": 8,      # (10.1 / 12.5: fp16 temporal-conv inputs)
              "mixed_3c": 4,       # (4.9 / 6.1: fp16 branch-3 pool outputs)
              "mixed_4f": 4,       # (5.2 / 4.1)
              "mixed_5c": 3.5,     # (4.7 / 3.8)
              "features": 3.5}     # (3.7 / 5.1)

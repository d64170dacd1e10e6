"""Bars of the MViT engine against float64 (tests/test_mvit_gpu.py; the stand-in ablations of
tests/test_mvit_oracle_cpu.py).  Each is (worst per-clip rel-L2, worst per-clip max-abs / max), about 2x the worst
value an H100 80GB HBM3 (700 W power limit) measured over the mvit_v1_b and mvit_v2_s stand-ins at 1 and 3 clips per
call with every GEMM weight a split-fp16 pair (DESIGN.md §4.15)."""
BARS = {"embed": (4.5e-4, 5e-4), "stage1": (9e-4, 1.2e-3), "stage2": (1.2e-3, 1.4e-3), "stage3": (1.5e-3, 1.8e-3),
        "stage4": (1.4e-3, 1.5e-3), "norm": (1.5e-3, 1.9e-3), "features": (9e-4, 1e-3),
        "attention hard": (5e-5, 1.2e-3)}
# "attention hard": the pooling-attention kernel alone on hard inputs (tests/test_attention_hard_gpu.py) against the
# float64 reference of its declared rounding (tests/attention_ref.py), every block geometry of v1 and v2: measured
# 2.4e-5 / 5.7e-4 on the same H100 (the max-abs part one fp16 ulp of the output).  The kernel built with the rel-pos
# term taken from the scaled q measured 0.34 / 0.42 or more (v2), without the rescale of its output 0.48 / 0.75.
# fp16-rounded GEMM weights (a lost lo half) must raise the feature rel-L2 error by at least this factor; the float64
# emulation (scripts/precision/emulate_mvit.py) predicts 2.1x for v1_b and 2.0x for v2_s
SEPARATION = 1.5

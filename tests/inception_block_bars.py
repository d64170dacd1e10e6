"""Bars of the I3D and S3D Mixed blocks, branch by branch, against float64 of the same block on the same split-fp16
input (test_inception_blocks_gpu.py), and of the shared (2,7,7) head kernel; test_inception_block_bars_cpu.py checks in
a CPU float64 emulation how far above them a lo half lost inside one branch lies.

BARS[engine][block]: per branch 0 .. 3, (rel-L2, max-abs / max|ref|) of that branch's channel slice, worst clip, over
the real input of the float64 trunk (S3D T = 13, I3D rgb T = 16, flow T = 12) and synthetic inputs at T = 1, 2, 3, 8
with one and three clips.  Each bar sits 1.5x above the worst value measured on one H100 80GB HBM3 (700 W power
limit), written under it; the engines are deterministic, so a rerun gives the same values.  A change to the conv GEMM
that reorders its fp32 sums moves them by as much with no loss of precision, and re-measures them.

S3D: 1.5e-6 .. 1.6e-5, the fp32 tensor-core accumulation of up to three convs in a row (branches 1 and 2).
I3D: branches 0 and 3 (one 1x1x1 conv on the pair input) 4e-7 .. 7e-6; branches 1 and 2 2e-5 .. 1.7e-4 rel-L2 with
max-abs up to 4e-4, because their 3x3x3 conv reads the 1x1x1 reducer's output as single fp16 (declared): the engine
rounds its fp32 value and the reference its float64 value, and an element near a rounding boundary flips by one ulp.
A lost lo half in those two branches is told apart by split_engine_bars.defect_share instead (SHARE below)."""
from oracle import s3d_net

# (cin, branch 0, 1, 2, 3 widths) and the side S of Mixed block 0 .. 8: the same for I3D and S3D
WIDTHS = tuple((c[0], c[1], c[3], c[5], c[6]) for c in s3d_net.MIXED.values())
SIDE = (28, 28, 14, 14, 14, 14, 14, 7, 7)
ENGINES = ("s3d", "i3d-rgb", "i3d-flow")

BARS = {
    "s3d": {
        0: [(2.2e-06, 2.7e-06), (1.1e-05, 1.3e-05), (4.3e-06, 3.9e-06), (3.9e-06, 2.7e-06)],
        #    1.46e-06 / 1.75e-06, 7.22e-06 / 8.11e-06, 2.86e-06 / 2.55e-06, 2.54e-06 / 1.79e-06
        1: [(2.4e-06, 3e-06), (1.4e-05, 1.7e-05), (7.2e-06, 8.2e-06), (4.1e-06, 4.5e-06)],
        #    1.54e-06 / 2.00e-06, 9.08e-06 / 1.11e-05, 4.77e-06 / 5.42e-06, 2.71e-06 / 2.94e-06
        2: [(8.5e-06, 7.3e-06), (1.6e-05, 1.7e-05), (1.8e-05, 1.9e-05), (1.6e-05, 1.3e-05)],
        #    5.65e-06 / 4.86e-06, 1.04e-05 / 1.09e-05, 1.14e-05 / 1.21e-05, 1.02e-05 / 8.50e-06
        3: [(4.3e-06, 5.1e-06), (1.6e-05, 1.9e-05), (7.1e-06, 7.6e-06), (8.3e-06, 7.2e-06)],
        #    2.86e-06 / 3.37e-06, 1.02e-05 / 1.24e-05, 4.70e-06 / 5.02e-06, 5.49e-06 / 4.80e-06
        4: [(4.6e-06, 7e-06), (1.7e-05, 1.9e-05), (8.5e-06, 9e-06), (9e-06, 1.1e-05)],
        #    3.04e-06 / 4.66e-06, 1.11e-05 / 1.25e-05, 5.64e-06 / 5.97e-06, 5.98e-06 / 6.99e-06
        5: [(4.2e-06, 5.4e-06), (1.9e-05, 2.3e-05), (9.7e-06, 1.4e-05), (9.3e-06, 8.9e-06)],
        #    2.76e-06 / 3.55e-06, 1.25e-05 / 1.53e-05, 6.41e-06 / 9.01e-06, 6.20e-06 / 5.90e-06
        6: [(4.5e-06, 5.2e-06), (2e-05, 2e-05), (9e-06, 1.1e-05), (9.8e-06, 1.2e-05)],
        #    2.97e-06 / 3.46e-06, 1.28e-05 / 1.33e-05, 5.96e-06 / 7.21e-06, 6.48e-06 / 7.95e-06
        7: [(1.2e-05, 1.4e-05), (2.4e-05, 2.5e-05), (1.9e-05, 1.9e-05), (2.1e-05, 1.5e-05)],
        #    7.38e-06 / 9.31e-06, 1.55e-05 / 1.62e-05, 1.23e-05 / 1.24e-05, 1.38e-05 / 9.55e-06
        8: [(6.4e-06, 7.3e-06), (2.3e-05, 3e-05), (1.4e-05, 1.7e-05), (1.2e-05, 1.3e-05)],
        #    4.25e-06 / 4.84e-06, 1.52e-05 / 1.97e-05, 9.07e-06 / 1.13e-05, 7.97e-06 / 8.28e-06
    },
    "i3d-rgb": {
        0: [(8.4e-07, 1.3e-06), (2.7e-05, 0.00012), (2.1e-05, 0.00019), (5.6e-07, 1.1e-06)],
        #    5.60e-07 / 8.09e-07, 1.80e-05 / 7.73e-05, 1.36e-05 / 1.21e-04, 3.72e-07 / 7.00e-07
        1: [(1.5e-06, 2.4e-06), (6.8e-05, 0.00021), (3.7e-05, 0.00018), (1.2e-06, 1.8e-06)],
        #    9.77e-07 / 1.54e-06, 4.47e-05 / 1.40e-04, 2.44e-05 / 1.18e-04, 7.53e-07 / 1.15e-06
        2: [(2.3e-06, 3.8e-06), (4e-05, 0.00014), (1.9e-05, 8.4e-05), (2.7e-06, 4.4e-06)],
        #    1.53e-06 / 2.48e-06, 2.65e-05 / 9.21e-05, 1.22e-05 / 5.57e-05, 1.77e-06 / 2.92e-06
        3: [(3.5e-06, 4.8e-06), (6.1e-05, 0.00013), (2.5e-05, 9.1e-05), (2.7e-06, 4.3e-06)],
        #    2.30e-06 / 3.16e-06, 4.05e-05 / 8.63e-05, 1.61e-05 / 6.03e-05, 1.74e-06 / 2.81e-06
        4: [(2.6e-06, 3.7e-06), (4.7e-05, 0.00012), (0.00013, 0.00045), (2.8e-06, 4.2e-06)],
        #    1.67e-06 / 2.44e-06, 3.07e-05 / 7.69e-05, 8.21e-05 / 2.96e-04, 1.85e-06 / 2.76e-06
        5: [(2.6e-06, 3.8e-06), (6.5e-05, 0.00014), (5.3e-05, 0.00019), (2.7e-06, 3.8e-06)],
        #    1.72e-06 / 2.48e-06, 4.33e-05 / 8.67e-05, 3.47e-05 / 1.25e-04, 1.76e-06 / 2.52e-06
        6: [(4e-06, 4.8e-06), (7.6e-05, 0.00015), (5.5e-05, 0.00023), (3.3e-06, 3.6e-06)],
        #    2.63e-06 / 3.19e-06, 5.01e-05 / 9.45e-05, 3.64e-05 / 1.53e-04, 2.16e-06 / 2.39e-06
        7: [(6.9e-06, 7e-06), (8.8e-05, 0.00016), (0.00013, 0.00026), (8.1e-06, 8.3e-06)],
        #    4.54e-06 / 4.63e-06, 5.86e-05 / 1.06e-04, 8.40e-05 / 1.69e-04, 5.40e-06 / 5.49e-06
        8: [(6.5e-06, 7.7e-06), (0.00011, 0.00017), (0.00026, 0.0006), (9.1e-06, 8.3e-06)],
        #    4.28e-06 / 5.07e-06, 6.92e-05 / 1.13e-04, 1.68e-04 / 3.96e-04, 6.05e-06 / 5.48e-06
    },
    "i3d-flow": {
        0: [(1.2e-06, 1.8e-06), (4.5e-05, 0.00014), (2.9e-05, 0.00027), (1e-06, 1.6e-06)],
        #    7.49e-07 / 1.17e-06, 2.96e-05 / 9.31e-05, 1.88e-05 / 1.79e-04, 6.63e-07 / 1.01e-06
        1: [(1.5e-06, 1.6e-06), (7.7e-05, 0.00025), (4e-05, 0.00018), (1.2e-06, 1.8e-06)],
        #    9.94e-07 / 1.04e-06, 5.07e-05 / 1.64e-04, 2.62e-05 / 1.20e-04, 7.93e-07 / 1.15e-06
        2: [(2.7e-06, 3.4e-06), (6.5e-05, 0.00018), (2.3e-05, 0.00015), (2.8e-06, 4.4e-06)],
        #    1.75e-06 / 2.21e-06, 4.27e-05 / 1.16e-04, 1.47e-05 / 9.84e-05, 1.86e-06 / 2.93e-06
        3: [(2.9e-06, 4.2e-06), (4.6e-05, 0.00015), (3.2e-05, 0.00014), (1.7e-06, 2.1e-06)],
        #    1.92e-06 / 2.78e-06, 3.05e-05 / 1.00e-04, 2.10e-05 / 8.82e-05, 1.11e-06 / 1.37e-06
        4: [(2.3e-06, 3.6e-06), (5.3e-05, 0.00014), (6.3e-05, 0.00021), (3.5e-06, 4.9e-06)],
        #    1.50e-06 / 2.40e-06, 3.48e-05 / 8.75e-05, 4.19e-05 / 1.37e-04, 2.27e-06 / 3.21e-06
        5: [(2.4e-06, 4.1e-06), (4.6e-05, 0.00011), (3.9e-05, 0.00016), (2.3e-06, 3.2e-06)],
        #    1.59e-06 / 2.67e-06, 3.03e-05 / 7.28e-05, 2.55e-05 / 1.02e-04, 1.53e-06 / 2.09e-06
        6: [(3.8e-06, 4.8e-06), (5.9e-05, 0.00018), (3.9e-05, 0.00013), (3e-06, 5e-06)],
        #    2.49e-06 / 3.14e-06, 3.88e-05 / 1.17e-04, 2.54e-05 / 8.48e-05, 1.97e-06 / 3.32e-06
        7: [(6.5e-06, 6.9e-06), (0.00013, 0.00018), (9.8e-05, 0.00018), (7.2e-06, 7.6e-06)],
        #    4.33e-06 / 4.55e-06, 8.06e-05 / 1.18e-04, 6.49e-05 / 1.15e-04, 4.78e-06 / 5.06e-06
        8: [(6.6e-06, 7.4e-06), (0.00016, 0.00027), (0.00014, 0.00024), (1.1e-05, 9.1e-06)],
        #    4.36e-06 / 4.88e-06, 1.04e-04 / 1.74e-04, 9.17e-05 / 1.60e-04, 6.72e-06 / 6.03e-06
    },
}

# GPU controls: (block, branch, the conv whose weights are pre-rounded to fp16), and the factor by which that branch
# must fail its bar (bars.beyond; measured: S3D 11.0x / 11.0x, I3D 80x / 62x)
S3D_CONTROL = (6, 1, "features.12.branch1.1.1.0.weight")     # Mixed 4f, branch 1's temporal conv
I3D_CONTROL = (6, 0, 39)                                      # mixed_4f.branch_0 (a split unit)
# split units of I3D branches 1 / 2 whose fp16 weights the bars do not separate: told apart by defect_share
I3D_SHARE_CONTROLS = ((6, 1, 41),                             # mixed_4f.branch_1.1
                      (8, 2, 55))                             # mixed_5c.branch_2.1 (0.9x / 0.3x its bar on the CPU)
CONTROL_FACTOR = {"s3d": 10, "i3d": 30}

# the (2,7,7) average pool + temporal mean, T3 = 2 .. 32, C = 832 / 1024: 9.4e-8 / 3.0e-7 (fp32 sums of <= 98 T3
# non-negative terms)
HEAD_BAR = (2e-7, 6e-7)

# least factor by which a defect inside one branch exceeds that branch's bar in the CPU emulation (bars.beyond)
# (measured: S3D 3b 20.5x, 4f 11.1x, 5c 9.2x; I3D rgb branches 0 and 3: 3b 149x, 4f 57x, 5c 28x).  At S3D Mixed 5c
# tenfold is NOT reached: branch 1's store lies 9.2x and its temporal conv's fp16 weights 9.5x / 8.4x above the bars,
# which already sit at 1.5x the engine's measured error, so 9x is what the bars can hold there.
SEPARATION = {"s3d": {0: 15, 6: 10, 8: 9}, "i3d": {0: 100, 6: 40, 8: 20}}
# I3D branches 1 and 2: defect_share of the branch slice along each defect the bars do not separate (fp16 weights of
# a split unit, the fp16 pair input of the 1x1x1 reducer, a lost store lo half), (most the intact engine may carry,
# least a defect shows).  In the CPU emulation with the flips modelled: all split |share| <= 0.002, every defect
# >= 0.97.  On the H100, over every block and input of both stand-ins: |share| <= 0.016 (store), 0.044 (weights),
# 0.058 (reducer input); the controls with fp16 weights carry +1.00 (mixed_5c.branch_2.1 at 0.9x / 0.4x its bar).
SHARE = (0.3, 0.7)

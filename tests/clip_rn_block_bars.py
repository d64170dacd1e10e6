"""Bars of the CLIP ResNet towers piece by piece against float64 (test_clip_resnet_blocks_gpu.py), the exact-pair
emulation of one Bottleneck both test files use, and the factors by which a lo half lost inside one Bottleneck lies
above the bars in a CPU float64 emulation (test_clip_rn_block_bars_cpu.py).

BLOCK[tower][layer][part]: (rel-L2, max-abs / max|ref|) of a block's output, branch (bn3's output before the residual
add) or shortcut (the downsample's output), worst frame, over every block of that layer on the float64 trunk's real
input to it (two frames) and on synthetic half-zero inputs (n = 1; 3 with one frame scaled 50x; 5 = max_frames) for the
first and last block of the layer, against a float64 block with the ORIGINAL weights on the same split-pair input.  Each
bar sits 1.5x above the worst value measured on one H100 80GB HBM3 (700 W power limit), written under it; the engine is
deterministic, so a rerun gives the same values.  A change to the conv GEMM that reorders its fp32 sums moves them by as
much with no loss of precision, and re-measures them.

What the bars consist of: the tensor cores' fp32 accumulation over K (up to 2 x 9 x 2048 for a layer4 3x3), which
grows with depth -- 2e-6 at a layer1 shortcut, 6e-5 at a layer4 branch.  The weights' subnormal lo halves (a hi + lo
pair of a weight under 0.125 keeps about 19 bits) are a small part of it: against float64 with the uploaded hi + lo
weights the engine measures the same values to within 7 % (the printed "uploaded weights" column), and the exact-pair
CPU emulation, which has no accumulation error, sits at most PAIR_SHARE of any bar.  Scaling the weights into fp16's
normal range at upload would therefore not move the bars; the split scheme is left as it is."""
import torch
import torch.nn.functional as F

BLOCK = {
    "RN50": {
        0: {"branch": (7.1e-06, 9e-06), "shortcut": (2.2e-06, 2.9e-06), "out": (3.1e-06, 3.6e-06)},
        #  4.67e-06 / 5.94e-06,  1.46e-06 / 1.87e-06,  2.02e-06 / 2.34e-06
        1: {"branch": (1.6e-05, 1.9e-05), "shortcut": (8.2e-06, 9.2e-06), "out": (8.7e-06, 8.9e-06)},
        #  1.05e-05 / 1.26e-05,  5.41e-06 / 6.11e-06,  5.76e-06 / 5.89e-06
        2: {"branch": (3e-05, 3.2e-05), "shortcut": (1.7e-05, 1.6e-05), "out": (1.9e-05, 2e-05)},
        #  1.97e-05 / 2.11e-05,  1.12e-05 / 1.02e-05,  1.21e-05 / 1.33e-05
        3: {"branch": (5.8e-05, 5.9e-05), "shortcut": (4.1e-05, 4.6e-05), "out": (4.3e-05, 5.2e-05)},
        #  3.82e-05 / 3.93e-05,  2.73e-05 / 3.06e-05,  2.83e-05 / 3.44e-05
    },
    # layers 1 .. 3 measure as RN50's: the stand-ins share their seeds and the worst block of each is one both have
    "RN101": {
        0: {"branch": (7.1e-06, 9e-06), "shortcut": (2.2e-06, 2.9e-06), "out": (3.1e-06, 3.6e-06)},
        #  4.67e-06 / 5.94e-06,  1.46e-06 / 1.87e-06,  2.02e-06 / 2.34e-06
        1: {"branch": (1.6e-05, 1.9e-05), "shortcut": (8.2e-06, 9.2e-06), "out": (8.7e-06, 8.9e-06)},
        #  1.05e-05 / 1.26e-05,  5.41e-06 / 6.11e-06,  5.76e-06 / 5.89e-06
        2: {"branch": (3e-05, 3.2e-05), "shortcut": (1.7e-05, 1.6e-05), "out": (1.9e-05, 2e-05)},
        #  1.97e-05 / 2.11e-05,  1.12e-05 / 1.02e-05,  1.21e-05 / 1.33e-05
        3: {"branch": (5.5e-05, 6.5e-05), "shortcut": (4.7e-05, 4.1e-05), "out": (4.8e-05, 4.3e-05)},
        #  3.64e-05 / 4.33e-05,  3.09e-05 / 2.72e-05,  3.16e-05 / 2.83e-05
    },
    "RN50x4": {
        0: {"branch": (9e-06, 9.9e-06), "shortcut": (2.8e-06, 3.6e-06), "out": (3.7e-06, 3.9e-06)},
        #  5.95e-06 / 6.60e-06,  1.83e-06 / 2.35e-06,  2.46e-06 / 2.58e-06
        1: {"branch": (1.9e-05, 2e-05), "shortcut": (1.1e-05, 1.1e-05), "out": (1.2e-05, 1.3e-05)},
        #  1.21e-05 / 1.33e-05,  6.90e-06 / 6.87e-06,  7.53e-06 / 8.10e-06
        2: {"branch": (3.8e-05, 4.4e-05), "shortcut": (2.3e-05, 1.8e-05), "out": (2.4e-05, 1.8e-05)},
        #  2.48e-05 / 2.88e-05,  1.47e-05 / 1.20e-05,  1.54e-05 / 1.18e-05
        3: {"branch": (7.3e-05, 8.8e-05), "shortcut": (5.3e-05, 4.7e-05), "out": (5.4e-05, 4.8e-05)},
        #  4.81e-05 / 5.82e-05,  3.48e-05 / 3.07e-05,  3.57e-05 / 3.15e-05
    },
    "RN50x16": {
        0: {"branch": (1.2e-05, 1.2e-05), "shortcut": (3.3e-06, 3.9e-06), "out": (3.9e-06, 4.2e-06)},
        #  7.39e-06 / 7.35e-06,  2.14e-06 / 2.54e-06,  2.57e-06 / 2.77e-06
        1: {"branch": (2.2e-05, 2.4e-05), "shortcut": (1.3e-05, 1.3e-05), "out": (1.4e-05, 1.3e-05)},
        #  1.44e-05 / 1.57e-05,  8.44e-06 / 8.48e-06,  9.13e-06 / 8.28e-06
        2: {"branch": (4.2e-05, 5.3e-05), "shortcut": (2.6e-05, 2.2e-05), "out": (2.7e-05, 2.1e-05)},
        #  2.75e-05 / 3.49e-05,  1.71e-05 / 1.44e-05,  1.79e-05 / 1.38e-05
        3: {"branch": (8.6e-05, 9.9e-05), "shortcut": (6.5e-05, 5.6e-05), "out": (6.6e-05, 5.9e-05)},
        #  5.71e-05 / 6.54e-05,  4.30e-05 / 3.71e-05,  4.40e-05 / 3.91e-05
    },
}

# The attention pool, each piece against float64 of the engine's own input to it, worst frame (all four towers, n = 1,
# 3, 5; the core also through the stateless entry at T = 1 .. 257).  Measured in the comments.
ATTN = {"kv": (2e-05, 2.6e-05),            # 1.31e-05 / 1.70e-05   split-weight GEMM, K = 2E up to 6144
        "q": (2e-05, 2.3e-05),             # 1.32e-05 / 1.49e-05
        "cproj": (2e-05, 2.7e-05),         # 1.29e-05 / 1.76e-05
        "core": (6.9e-07, 1.1e-06),        # 4.58e-07 / 7.19e-07   fp32 scores, softmax and sum, then the split
        # scores of +-30 .. +-100 and a tied maximum: the two tied keys carry almost all the weight, so the output is
        # nearly their mean and its error smaller than at a flat softmax
        "core hard": (2.1e-07, 3.4e-07)}   # 1.39e-07 / 2.26e-07
# K|V rounded to fp16 must fail the attention-core bar by this factor (measured at least 340x flat, 940x hard)
KV_FP16_FACTOR = 10

# CPU premise (test_clip_rn_block_bars_cpu.py: layer1.0, layer2.0, layer3.1, layer4.1 of each stand-in, one frame):
# SEPARATION[tower][layer] is the least factor (bars.beyond) by which every single-fp16 defect of that layer's emulated
# block exceeds the bar of the part it is checked against; the least measured in the comment, with the defect that
# sets it.  Tenfold is reached at layer1 only.  Past it the engine's own fp32 accumulation, which the bars hold, comes
# within 3 .. 10x of a lost lo half (2e-4 .. 4e-4 rel-L2 in any block), down to 2.7x at RN50x16 layer4.1, whose
# conv3 input has its lo half dropped.  Where tenfold is not reached the GPU test also asserts defect_share (SHARE).
SEPARATION = {
    "RN50": {0: 28, 1: 9, 2: 7.5, 3: 4.5},        # 31.0 (conv3 weights), 10.1 (conv3 input), 8.6 (conv3 w), 5.1 (conv3 w)
    "RN101": {0: 28, 1: 9, 2: 7.5, 3: 3.8},       # 31.0, 10.1, 8.6, 4.3 (conv3 input)
    "RN50x4": {0: 25, 1: 8, 2: 5, 3: 2.8},        # 27.5 (conv1 input), 8.9 (conv3 input), 5.7 (conv3 w), 3.2 (conv3 input)
    "RN50x16": {0: 20, 1: 6.8, 2: 5, 3: 2.4},     # 22.8 (conv1 input), 7.6, 5.5, 2.7 (conv3 input)
}
# The exact-pair emulation's own distance from float64 with the original weights, as a share of the bar: measured at
# most 0.18 (RN50x16 layer1.0's shortcut; 0.175 at RN50 layer1.0's branch).  Under a third, so the weights' subnormal
# lo halves are left as they are.
PAIR_SHARE = 1 / 3

# defect_share of a part along a single-fp16 defect's direction (split_engine_bars.defect_share, against the exact-pair
# emulation): (the most the intact engine may carry, the least an engine with the defect shows).  Asserted for every
# DEFECTS direction of every block of layers 2 .. 4 on its real input, where the bars do not separate tenfold.
SHARE = (0.3, 0.7)

# GPU controls: (tower, block index, the defect: a conv's weights pre-rounded to fp16, the part whose bar it must fail
# by SEPARATION of its layer).  Measured on the H100: RN50 layer4.1.conv3 4.3x / 5.1x its branch bar, RN50x16
# layer4.0.downsample.0 6.7x / 7.8x its shortcut bar.
CONTROLS = (("RN50", 14, ("w", "conv3"), "branch"),
            ("RN50x16", 32, ("w", "downsample.0"), "shortcut"))

PARTS = ("out", "branch", "shortcut")
DEFECTS = (("w", "conv1"), ("w", "conv2"), ("w", "conv3"), ("w", "downsample.0"), ("x", "conv1"), ("x", "conv2"),
           ("x", "conv3"), ("x", "downsample.0"), ("store", "branch"), ("store", "out"))
# the part a defect is checked against: the convs of the residual branch and the branch store by the branch, the
# downsample by the shortcut, the output store by the output
PART = {"conv1": "branch", "conv2": "branch", "conv3": "branch", "downsample.0": "shortcut", "branch": "branch",
        "out": "out"}


def pair(t: torch.Tensor) -> torch.Tensor:
    """The value of the split pair the engine stores for t: fp16(t) + fp16(t - fp16(t)), subnormal lo included."""
    hi = t.half()
    return hi.double() + (t - hi.double()).half().double()


def emulated_block(sd, cfg, i, x, defect=None):
    """Bottleneck i (execution order) on the pair value x (block 0: the unpooled stem output), in float64 with every
    split pair modelled exactly -- the weights and every stored activation (conv1's and conv2's outputs, the branch, the
    shortcut, the block output) -- and `defect` (one of DEFECTS, or None) in single fp16 -> dict(out, branch, shortcut).
    The convolutions are exact: what is left is the pair representation alone."""
    from oracle import clip_resnet
    p, stride, _ = clip_resnet.blocks(cfg)[i]

    def w(name):
        t = sd[f"{p}.{name}.weight"]
        return t.half().double() if defect == ("w", name) else pair(t)

    def inp(t, name):
        return t.half().double() if defect == ("x", name) else t

    def bn(t, name):
        return F.batch_norm(t, sd[f"{p}.{name}.running_mean"], sd[f"{p}.{name}.running_var"], sd[f"{p}.{name}.weight"],
                            sd[f"{p}.{name}.bias"], False, 0.0, 1e-5)

    def store(t, name):
        return t.half().double() if defect == ("store", name) else pair(t)

    pooled_in = i == 0
    a = inp(x, "conv1")
    t1 = pair(F.relu(bn(F.conv2d(F.avg_pool2d(a, 2) if pooled_in else a, w("conv1")), "bn1")))
    t2 = pair(F.relu(bn(F.conv2d(inp(t1, "conv2"), w("conv2"), padding=1), "bn2")))
    b = inp(t2, "conv3")
    branch = store(bn(F.conv2d(F.avg_pool2d(b, 2) if stride > 1 else b, w("conv3")), "bn3"), "branch")
    short = x
    if f"{p}.downsample.0.weight" in sd:
        d = inp(x, "downsample.0")
        d = F.avg_pool2d(d, 2) if (stride > 1 or pooled_in) else d
        short = pair(bn(F.conv2d(d, w("downsample.0")), "downsample.1"))
    return dict(out=store(F.relu(short + branch), "out"), branch=branch, shortcut=short)


def has_downsample(sd, cfg, i) -> bool:
    from oracle import clip_resnet
    return f"{clip_resnet.blocks(cfg)[i][0]}.downsample.0.weight" in sd

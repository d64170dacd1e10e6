"""Bars of the split-fp16 engines against a float64 forward of the same network (worst row: per frame or clip for a
stage, per feature row), shared by the float64 GPU tests (test_split_engines_float64_gpu.py: ResNet, R(2+1)D;
test_i3d_raft_float64_gpu.py: I3D, RAFT, against a reference with each engine's declared fp16 rounding), and
test_split_engine_bars_cpu.py, which checks in a CPU float64 emulation how far above each bar every variant that leaves
one tensor class in single fp16 lies.  SEPARATION (ResNet, R(2+1)D) and SEPARATION_I3D / SEPARATION_RAFT state that
factor per stage; a stage a class does not appear under is one where it is not told apart from the engine's own error.

Each entry is (rel-L2, max-abs / max|ref|).  A bar sits 1.5x to 3x above the worst value the engine measured on an
H100 (the GPU tests' docstrings and the comments below have the numbers; the engines are deterministic, so a rerun gives
the same values).  The margin is narrow because the engine's error is its fp32 accumulation (and, for I3D, 1-ulp
differences in its single-fp16 tensors): a change to the conv GEMM's K order, pipeline staging or tile widths that
reorders the fp32 sums can move these values by that much with no loss of precision; such a change re-measures them.
That the engines upload every lo half, W_lo row and lo_mask bit is checked exactly, conv by conv, by
test_conv_gemm_resnet_r21d_gpu.py and test_i3d_raft_uploads_gpu.py.  That read-back sees weights only; a loss too small
to show at a stage (most I3D classes past mixed_3c, or one branch's store, conv input or pool) is guarded by the
per-branch block tests of test_inception_blocks_gpu.py (bars in inception_block_bars.py)."""
import torch

RESNET_STAGES = ("stem", "maxpool", "layer1", "layer2", "layer3", "layer4", "features")
R21D_STAGES = ("stem", "layer1", "layer2", "layer3", "layer4", "features")

RESNET_BARS = {
    18: {"stem": (4e-6, 5e-6), "maxpool": (4e-6, 5e-6), "layer1": (8e-6, 8e-6), "layer2": (2e-5, 2e-5),
         "layer3": (3.5e-5, 3.5e-5), "layer4": (5e-5, 5e-5), "features": (4e-5, 8e-5)},
    50: {"stem": (4e-6, 6e-6), "maxpool": (4e-6, 6e-6), "layer1": (1.2e-5, 1.2e-5), "layer2": (3e-5, 3e-5),
         "layer3": (9e-5, 9e-5), "layer4": (1.6e-4, 1.6e-4), "features": (1e-4, 2e-4)},
    152: {"stem": (4e-6, 6e-6), "maxpool": (4e-6, 6e-6), "layer1": (1.2e-5, 1.5e-5), "layer2": (4.5e-5, 4.5e-5),
          "layer3": (5e-4, 5.5e-4), "layer4": (9e-4, 1e-3), "features": (2.5e-4, 5e-4)},
}
R21D_BARS = {"stem": (7e-6, 8e-6), "layer1": (1.7e-5, 1.5e-5), "layer2": (2.5e-5, 2.5e-5), "layer3": (4e-5, 4e-5),
             "layer4": (1.3e-4, 1.6e-4), "features": (1e-4, 1.5e-4)}

# How far (both halves) every single-fp16 class must lie above the bar, per stage, in the CPU emulation of ResNet-18 (2
# frames) and R(2+1)D (1 clip x 8 frames).  Tenfold up to layer4; less at the deep end, where the engine's own error
# (the fp32 accumulation of the tensor-core MMAs over K up to 16k, about 1e-6 .. 1.5e-5 per conv) comes within reach
# of a lost lo half, and at the features, where the average pool cancels most of a rounding error but not the
# accumulation's.  A lost lo half is therefore caught at the stages, and most sharply at the stem.
SEPARATION = {
    "resnet18": {"stem": 10, "maxpool": 10, "layer1": 10, "layer2": 10, "layer3": 10, "layer4": 10, "features": 3},
    "r21d": {"stem": 10, "layer1": 10, "layer2": 10, "layer3": 10, "layer4": 4, "features": 1.5},
}


def row_errors(y: torch.Tensor, ref: torch.Tensor):
    """Worst row (dim 0: frame, clip or feature row) of rel-L2 and max-abs / max|ref|, in float64."""
    y = y.double().flatten(1)
    ref = ref.double().flatten(1).to(y.device)
    d = y - ref
    rel = (d.norm(dim=1) / ref.norm(dim=1)).max().item()
    mx = (d.abs().amax(dim=1) / ref.abs().amax(dim=1)).max().item()
    return rel, mx


def within(err, bar, factor: float = 1.0) -> bool:
    """Both halves of err at or under factor x bar."""
    return err[0] <= factor * bar[0] and err[1] <= factor * bar[1]


def beyond(err, bar, factor: float = 1.0) -> bool:
    """rel-L2 or max-abs above factor x its bar: the check fails by at least that factor."""
    return err[0] > factor * bar[0] or err[1] > factor * bar[1]



# ---- I3D and RAFT, against a float64 forward with the engine's declared rounding (oracle/i3d_net.py,
# oracle/raft_net.py declared_rounding=True: the operands the engine keeps as single fp16 are rounded, nothing else),
# held by test_i3d_raft_float64_gpu.py.  Worst rows measured on one H100 80GB HBM3 (400 W power limit), rel-L2 /
# max-abs÷max; the bars sit 1.5x .. 3x above them (I3D rgb 1a: 2.9x / 2.4x, the rest 1.5x .. 2x):
#   I3D rgb (T = 16, 11, two stacks; controls T = 12)      I3D flow (T = 12)
#   1a  6.8e-7 / 2.1e-6                                    1.0e-6 / 2.1e-6
#   2c  1.6e-5 / 1.2e-4                                    2.9e-5 / 1.5e-4
#   3c  4.4e-5 / 1.1e-4                                    6.4e-5 / 1.1e-4
#   4f  1.1e-4 / 2.3e-4                                    1.3e-4 / 2.4e-4
#   5c  2.5e-4 / 3.9e-4                                    2.8e-4 / 4.8e-4
#   features 3.8e-5 / 4.8e-5                               4.8e-5 / 4.4e-5
# Past the stem I3D's error jumps (1a 6.8e-7, 2c 1.6e-5 with a max-abs 7x its rel-L2).  That is what 1-ulp flips of
# the single-fp16 tensors (conv3d_2b's and every 1x1x1 reducer's output) would give: the engine rounds its fp32 value,
# the reference its float64 value, an element near a rounding boundary lands on the other side, and each flip is a
# 2^-11 error in that element that the Mixed blocks carry on (an estimate; the flips were not counted).  The bars therefore separate a lost lo class most sharply at 1a
# (fp16 stem input or weights: 1.1e-4 against 2e-6) and 2c (fp16 weights: 2.8e-4, 11x the rgb bar).
#   RAFT (128x160, 200x200, 270x480, 96x128, 64x120; 1 and 3 iterations): fnet 5.1e-6 / 5.0e-6, cnet 2.0e-6 / 2.4e-6,
#   pyramid 3.6e-6 / 6.0e-6, lookup 3.4e-6 / 6.3e-6, GRU state 1.4e-5 / 2.5e-5, low-res flow 9.9e-5 / 1.1e-4,
#   flow_up 4.6e-5 / 1.3e-4; flow_up after 20 iterations 2.7e-5 / 1.2e-4.
# fp16 RAFT weights cost fnet 9.9e-4 (120x its bar).  The low-res flow's relative error is large because the flow after
# one to three steps is small: the flow head's fp32 accumulation over K = 2 x 2304 is most of it.
I3D_STAGES = ("1a", "2c", "3c", "4f", "5c", "features")       # read_stage 0 .. 4, then the features
I3D_BARS = {
    "rgb": {"1a": (2e-6, 5e-6), "2c": (2.5e-5, 2e-4), "3c": (7e-5, 2e-4), "4f": (1.8e-4, 3.5e-4),
            "5c": (3.7e-4, 6e-4), "features": (6e-5, 8e-5)},
    "flow": {"1a": (2e-6, 4e-6), "2c": (4.5e-5, 2.5e-4), "3c": (1e-4, 2e-4), "4f": (2e-4, 3.7e-4),
             "5c": (4.3e-4, 7.5e-4), "features": (7.5e-5, 7e-5)},
}
RAFT_STAGES = ("fnet", "cnet", "pyramid", "lookup", "net", "lowres", "flow_up")
RAFT_BARS = {"fnet": (8e-6, 8e-6), "cnet": (3.5e-6, 4e-6), "pyramid": (6e-6, 9e-6), "lookup": (6e-6, 1e-5),
             "net": (2.2e-5, 4e-5), "lowres": (1.5e-4, 1.7e-4), "flow_up": (7e-5, 2e-4)}
RAFT_BAR_20_ITERS = (4.5e-5, 2e-4)      # flow_up after 20 iterations

# How far above the bar (bars.beyond: rel-L2 or max-abs, whichever is further) each variant that leaves one class in
# single fp16 lies, in the CPU float64 emulation of test_split_engine_bars_cpu.py, at the stages where it is asserted.
# I3D (rgb stand-in, 1 x 3 x 10 x 224 x 224, against the declared-rounding reference; measured in parentheses).  Every
# class is separated at the first stage it reaches (2c: 9.7 .. 11x, 3c: 2.5 .. 4.3x); past 3c most are within 2x of
# the bar or under it, where only the conv read-back sees them.  The 1x1x1 weights show again at the features (6.8x).
SEPARATION_I3D = {
    "stem output": {"2c": 8, "3c": 2},                        # (9.7, 2.5)   the stem output = conv3d_2b's input
    "pool outputs": {"3c": 2.4},                              # (2.9)        every branch_3 pool, pool3a / 4a / 5a
    "concat buffers": {"3c": 2.2, "4f": 1.5},                 # (2.7, 1.8)   the Mixed outputs read by the next block
    "1x1x1 inputs": {"2c": 8, "3c": 3.5, "4f": 1.7},          # (9.7, 4.3, 2.1)
    "2b / 2c weights": {"2c": 9, "3c": 2.3},                  # (11.0, 2.8)
    "1x1x1 weights": {"3c": 3.3, "4f": 1.8, "features": 5},   # (4.1, 2.2, 6.8)
    "4x / 5x 3x3x3 weights": {"features": 2.3},               # (3.2)
}
# RAFT (stand-in, 2 frames of 128 x 160, 3 iterations, the operand groups of scripts/precision/emulate_raft.py).
# Strongly separated at the first stage each reaches; at the low-res flow and flow_up every class lies 1.3 .. 9x above
# the bars and is not asserted.  The flow head's conv2 input is separated nowhere (1.3x at the low-res flow).
SEPARATION_RAFT = {
    "fnet weights": {"fnet": 100, "pyramid": 35, "lookup": 20, "net": 18},   # (124, 47, 44, 27)
    "cnet weights": {"cnet": 45, "net": 9},                                    # (60, 12)
    "motion encoder weights": {"net": 18},                                     # (23)
    "GRU weights": {"net": 7.5},                                               # (9.5)
    "flow head weights": {"flow_up": 7.5},                                     # (9.4)
    "fnet inner inputs": {"fnet": 100, "pyramid": 35, "lookup": 20, "net": 15},  # (131, 50, 46, 20)
    "cnet inner inputs": {"cnet": 50, "net": 10},                              # (77, 12.5)
    "motion encoder intermediates": {"net": 11},                               # (14)
    "flow head conv2 input": {},                                               # (1.3 at the low-res flow)
    "GRU motion slice": {"net": 4.5},                                          # (5.8)
}


# ---- CLIP ViT towers, piece by piece against a float64 reference with the tower's declared rounding
# (oracle/clip_tower.py DECLARED: embed / block / head / attention_core), each piece fed the ENGINE's own input, held by
# test_clip_float64_gpu.py.  Worst row = worst TOKEN row (768 values) for embed / block / attention, worst feature row
# for head / features; (rel-L2, max-abs / max|ref|).  Measured values: the comment beside each bar.
#
# What the bars consist of.  Every fp16 rounding point sits behind fp32 arithmetic in the engine and float64 in the
# reference; a relative difference e between the two flips the rounding of a fraction ~e / 2^-11 of the elements, each by
# one ulp, so the rounded tensor differs by ~sqrt(e * 2^-11) rms: 7e-6 for e = 1e-7, against the 1e-7 itself.  A block has
# six such points in a row (ln_1, q/k/v, P, attention output, ln_2, MLP hidden), which is where its 2e-5 .. 6e-5 comes
# from, and any fp16 tensor compared directly (the attention output) has a max-abs floor of one ulp, 4.9e-4, whenever its
# largest element flips.  Perturbations smaller than the flips they cause (unrounded P, fp16 scores, eps 1e-6 on rows
# of unit variance, a QuickGELU constant of 1.7) therefore cannot be told apart by any rel-L2 bar; for those the tests use
# defect_share() below, which can.
# Measured on one H100 80GB HBM3 (700 W power limit); the engine is deterministic, a rerun gives the same values.
CLIP_VIT = {
    "embed": (4e-6, 7e-6),                        # 2.1e-6 / 3.9e-6   B/32 and B/16, 1 / 3 / 13 frames, both entries
    "block": {"plain": (1e-4, 1.2e-4),            # 5.7e-5 / 6.6e-5   12 blocks x 1 / 2 / 5 / 23 frames, block 5 at 250, split path
              "outlier": (6e-5, 6e-5),            # 3.1e-5 / 3.1e-5   residual peaks above 50 (relative to larger rows)
              "plain16": (1e-4, 1.1e-4)},         # 5.5e-5 / 5.7e-5   B/16, 3 frames
    # VF_CLIP_RESID=y / mix: one flip of an fp16 increment is 2^-11 of that element, straight into the stream
    "block y": {"plain": (1.4e-4, 3.5e-4),        # 7.6e-5 / 2.0e-4   (mix: 5.9e-5 / 1.0e-4)
                "outlier": (1e-4, 9e-5)},         # 5.3e-5 / 4.5e-5
    "head": (7e-6, 8e-6),                         # 3.5e-6 / 4.0e-6   the row of variance 1e-6; engine stream rows 1.0e-6 / 1.3e-6
    # A row of 768 equal values: the kernel's mean is sum * fl(1 / 768), not sum / 768, so x - mean is 2^-25 x instead of
    # 0; times rstd = 1 / sqrt(eps) = 316 that is 1e-5 absolute in an output that consists of the bias alone (|b| ~ 0.05).
    "head constant row": (5e-4, 5.5e-4),          # 2.5e-4 / 2.8e-4
    "attention": (5e-4, 1.6e-3),                  # 2.7e-4 / 8.7e-4   block 5 on its own ln_1 output; an fp16 output: 1 ulp = 4.9e-4
    # scores of 20 .. 100 (several hundred at most): one flipped q or k element moves a score by ~1e-2 and P with it
    "attention hard": (7e-3, 1.5e-2),             # 3.6e-3 / 7.6e-3   B/32 1 / 2 / 5 / 23 frames, B/16 1 / 3 / 7
    # The flips of 12 blocks compound, and the tower amplifies them: 6.5x a block's error, 2.7x under the 1e-3 product
    # gate.  The declared-rounding tower in fp32 on the CPU lies as far from the float64 one (3.3e-4 / 3.7e-4).
    "features": (6e-4, 8e-4),                     # 3.7e-4 / 5.1e-4   8 and 270 frames
}
# Controls: (bar the control is asserted against, factor by which it must fail it; measured on the GPU in the comment).
CLIP_VIT_CONTROLS = {
    "bf16 weights": ("block", 4),                 # 5.1x / 5.6x
    "in_proj bias group zeroed": ("attention", 10),   # 19x / 36x  (6.1x / 5.3x the block bar)
    "eps 1e-6": ("head", 1000),                   # on the row of variance 1e-6
}
# defect_share: the most the engine's error may carry of a defect's direction, and the least an engine with the defect
# shows.  Measured on the GPU at block 5: P unrounded +0.28, eps 1e-6 +0.22, QuickGELU 1.7 +0.06, bias group zeroed
# +0.001.  The first two are not 0: a perturbation far under one ulp acts only through the elements that sit on a
# rounding boundary, and those are the elements the engine's own fp32 error flips too, in the same direction half the time.
CLIP_VIT_SHARE = (0.5, 0.65)


def defect_share(got: torch.Tensor, ref: torch.Tensor, ref_defect: torch.Tensor) -> float:
    """Least-squares coefficient of (ref_defect - ref) in (got - ref): 1 when `got` was computed the way `ref_defect` was,
    0 when the way `ref` was.  Rounding flips are uncorrelated with the direction, so over the ~1e5 elements of a block
    output they move the coefficient by ~1e-2 even where they exceed the defect in norm."""
    ref = ref.double().flatten()
    d = ref_defect.double().flatten().to(ref.device) - ref
    e = got.double().flatten().to(ref.device) - ref
    return float((e @ d) / (d @ d))


# ---- PWC-Net and RAFT under motion (test_flow_motion_gpu.py; premise: test_flow_steering_cpu.py)
# The seeded stand-ins warp PWC's second frame by ~1 px and move RAFT's lookup centre by under half a cell; the steered
# state dicts of tests/flow_steering.py reach 8 px and 3 .. 45 cells.  SEPARATION_FLOW_MOTION: how far above the bar a
# defective sampler lies in the float64 oracle (PWC: worst rel-L2 of the cost volume, decoder flow and final flow over
# its bar; RAFT: bars.beyond at lookup / GRU state / flow_up), on the stand-in's small motion (128 x 160, the inputs
# and bars of test_pwc_gpu.py / test_i3d_raft_float64_gpu.py) and on the steered inputs (PWC_MOTION_BARS /
# RAFT_MOTION_BARS below).  Measured in parentheses; 0 = stated as NOT separated (under the bar).
# What it shows: the gross sampler defects -- truncation for floor, border clamp for zero padding, a dropped mask,
# align_corners=False, an untransposed window, the level scaling misplaced -- were already far above the bars on the
# small-motion inputs, through the border pixels alone (a border sample with negative flow has a negative coordinate
# and an outside tap).  What small motion does NOT separate is a lost lo half of PWC's upsampled-flow pair: 2^-11 of
# the flow is under the bars while the flow is about a pixel (0.34x), and above them once it is eight (5.6x, 7.7x).
# RAFT's flow pair is separated by neither.  `mask >= 0.999` is
# separated by no input (a raw mask of exactly 0.999 does not occur); the GPU test brackets the threshold instead, with
# border raw masks of 0.9995 and 0.9985.
SEPARATION_FLOW_MOTION = {
    "pwc": {
        "truncation for floor": {"small motion": 5000, "uniform level 2": 800, "varying level 2": 2500},   # (7950, 1300, 3820)
        "border clamp for zeros": {"small motion": 5500, "uniform level 2": 7000, "varying level 2": 5000},  # (8410, 10600, 8120)
        "mask >= 0.999": {"small motion": 0, "uniform level 2": 0, "varying level 2": 0},                 # (1e-11)
        "mask dropped": {"small motion": 5500, "uniform level 2": 2000, "varying level 2": 2300},         # (8380, 3210, 3540)
        "align_corners=False": {"small motion": 3000, "uniform level 2": 3000, "varying level 2": 4000},  # (4590, 4620, 6570)
        "upflow pair's lo half lost": {"small motion": 0, "uniform level 2": 3.5, "varying level 2": 5},  # (0.34, 5.6, 7.7)
    },
    "raft": {
        "truncation for floor": {"small motion": 9e4, "uniform step": 6e4, "varying flow": 1e4},          # (1.4e5, 9.1e4, 1.6e4)
        "border clamp for zeros": {"small motion": 1.7e5, "uniform step": 2e5, "varying flow": 2.5e4},    # (2.5e5, 3.2e5, 4.0e4)
        "window not transposed": {"small motion": 9e4, "uniform step": 9e4, "varying flow": 1.3e4},       # (1.4e5, 1.3e5, 2.0e4)
        "level scaling after the floor": {"small motion": 6e4, "uniform step": 7.5e4, "varying flow": 6e3},  # (9.3e4, 1.2e5, 9.1e3)
        # Not separated by any input: 2^-11 of a 3.5-cell flow is 0.65x the 20-iteration bars (the refinement's own
        # error has grown as much).  (A uniform step's flow is a multiple of 2^-3: its pair has no lo half to lose.)
        "flow pair's lo half lost": {"small motion": 0, "uniform step": 0, "varying flow": 0},            # (0.07, 2e-10, 0.65)
    },
}

# Bars of test_flow_motion_gpu.py, 1.5x .. 3x above the worst value measured on one H100 80GB HBM3 (700 W power limit;
# the engines are deterministic).  PWC: rel-L2 of the cost volume against the oracle's warp of the engine's own features
# and upflow, of each decoder flow and of the final flow (rel-L2, max-abs / max) against the oracle's forward, over
# uniform warps at levels 5 .. 2 (128x160, 200x333), the threshold warps, the varying warps and the 40x50 frames.
PWC_MOTION_BARS = {"volume": 3.5e-5,              # 1.70e-5 (level 5; 3.4e-6 and under below it)
                   "flow": 1.5e-4,                # 7.2e-5
                   "final": (1.8e-4, 2.5e-4)}     # 9.1e-5 / 1.24e-4 (the level-4 varying warp; 7.4e-5 / 7.4e-5 at level 2)
# RAFT, per steered input, the stages of RAFT_STAGES; a stage not listed keeps its RAFT_BARS entry (fnet, cnet and the
# pyramid do not depend on the flow: 4.95e-6 / 4.4e-6, 1.93e-6 / 2.35e-6, 3.5e-6 / 5.2e-6 as in RAFT_BARS' own runs).
RAFT_MOTION_BARS = {
    # lookup 3.5e-6 / 5.7e-6 (centres up to 45 cells from the query: no worse than in the query's own cell)
    "uniform": dict(RAFT_BARS, net=(2.2e-5, 6e-5),            # 1.17e-5 / 3.0e-5
                    lowres=(0.0, 0.0),                        # exact: dyadic steps
                    flow_up=(1.2e-5, 2.6e-4)),                # 5.7e-6 / 1.30e-4
    "varying 3": dict(RAFT_BARS, lowres=(5e-5, 6e-5),         # 2.34e-5 / 2.89e-5 (net 1.41e-5 / 2.19e-5)
                      flow_up=(5e-5, 3.5e-4)),                # 2.33e-5 / 1.78e-4
    # after 20 iterations of a 3.5-cell flow the lookup is taken at coordinates that carry the flow's own error
    "varying 20": dict(RAFT_BARS, lookup=(4e-5, 1.5e-4),      # 1.85e-5 / 7.11e-5
                       net=(7e-5, 2.2e-4),                    # 3.35e-5 / 1.08e-4
                       lowres=(6e-5, 9e-5),                   # 2.90e-5 / 4.20e-5
                       flow_up=(6.5e-5, 2.5e-4)),             # 3.13e-5 / 1.22e-4
    # logits of +-60: where two of the nine are tied a logit error of 1e-5 x 60 moves the weights by as much, times
    # the difference between the two neighbours' flows
    "sharp": dict(RAFT_BARS, flow_up=(2.7e-4, 3.4e-3)),       # 1.33e-4 / 1.68e-3 (low-res flow 4.7e-5 / 5.6e-5)
}

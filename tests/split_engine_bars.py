"""Bars of the ResNet and R(2+1)D engines against a float64 forward of the same network (worst row: per frame or clip
for a stage, per feature row), shared by test_split_engines_float64_gpu.py, which holds the engines to them, and
test_split_engine_bars_cpu.py, which checks on the CPU that they tell the designed split-fp16 scheme apart from every
variant that leaves one tensor class in single fp16.

Each entry is (rel-L2, max-abs / max|ref|).  A bar sits 1.5x to 3x above the worst value the engine measured on an
H100 (test_split_engines_float64_gpu.py's docstring has the numbers; the engine is deterministic, so a rerun gives the
same values), and SEPARATION below says how far under the smallest error of any single-fp16 class it lies (the CPU test
asserts it for ResNet-18 and R(2+1)D).  The margin is narrow because the engine's error is its fp32 accumulation:
a change to the conv GEMM's K order, pipeline staging or tile widths that reorders the fp32 sums can move these values
by that much with no loss of precision; such a change re-measures them.  That the engines upload every lo half, W_lo
row and lo_mask bit is checked exactly, conv by conv and at every depth, by test_conv_gemm_resnet_r21d_gpu.py."""
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

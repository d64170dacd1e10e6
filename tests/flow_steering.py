"""State dicts that steer PWC-Net and RAFT into the motion regimes the seeded stand-ins never reach, shared by
test_flow_steering_cpu.py (which asserts in the float64 oracles that each regime is reached) and
test_flow_motion_gpu.py (which runs the engines there).  Pure functions: each returns a modified copy.

The stand-in weights move a PWC warp by ~1 px and a RAFT lookup centre by under half a cell, so the sampling kernels
only ever see their own pixel's neighbourhood.  The flow can be set through the weights alone:

- PWC: level l's warp is given DBL_BACKWARD[l] * moduleUpflow(flow of level l + 1).  A transposed conv with zero
  weights returns its bias, so bias (u, v) displaces every pixel by exactly DBL_BACKWARD[l] * (u, v).
- RAFT: every iteration adds flow_head.conv2's output to coords1; with zero weights that is its bias (du, dv), and the
  lookup of iteration k is centred at (x, y) + (k - 1) (du, dv).
"""
import torch

from oracle import pwc_net

RAFT_FLOW_CONV2 = "module.update_block.flow_head.conv2"
RAFT_MASK2 = "module.update_block.mask.2"


def fp16_pair_exact(v: float) -> float:
    """v rounded to a multiple of 2^-20 (|v| < 1) or 2^-10 (|v| < 2^11): at most 21 significant bits, none below 2^-24,
    so v is exact in fp32 and as the hi + lo of a split-fp16 pair (11 bits each): the engine and the float64 oracle are
    given the same number."""
    q = 2.0 ** 20 if abs(v) < 1 else 2.0 ** 10
    return round(v * q) / q


def pwc_uniform_warp(sd, level: int, dx: float, dy: float):
    """Level `level`'s backward warp displaces every pixel by (dx, dy) px of that level (each rounded so that the
    bias dx / DBL_BACKWARD is exact in a split-fp16 pair, fp16_pair_exact).  Returns (state dict, the exact displacement)."""
    dbl = pwc_net.DBL_BACKWARD[level]
    u, v = fp16_pair_exact(dx / dbl), fp16_pair_exact(dy / dbl)
    p = f"module{pwc_net.LEVEL_NAMES[level]}.moduleUpflow."
    out = dict(sd)
    out[p + "weight"] = torch.zeros_like(sd[p + "weight"])
    out[p + "bias"] = torch.tensor([u, v], dtype=sd[p + "bias"].dtype)
    return out, (u * dbl, v * dbl)


def pwc_varying_warp(sd, gains: dict):
    """gains: level -> factor on that level's moduleUpflow weight and bias: the stand-in's own, spatially varying
    upsampled flow, that many times larger."""
    out = dict(sd)
    for level, g in gains.items():
        p = f"module{pwc_net.LEVEL_NAMES[level]}.moduleUpflow."
        out[p + "weight"], out[p + "bias"] = sd[p + "weight"] * g, sd[p + "bias"] * g
    return out


def raft_uniform_step(sd, du: float, dv: float):
    """Every refinement iteration adds exactly (du, dv) cells (1/8-resolution pixels) to every coordinate."""
    out = dict(sd)
    out[RAFT_FLOW_CONV2 + ".weight"] = torch.zeros_like(sd[RAFT_FLOW_CONV2 + ".weight"])
    out[RAFT_FLOW_CONV2 + ".bias"] = torch.tensor([du, dv], dtype=sd[RAFT_FLOW_CONV2 + ".bias"].dtype)
    return out


def raft_varying_flow(sd, gain: float):
    """The flow head's last conv `gain` times larger (the stand-in attenuates it by 0.1, oracle/stand_in.py): the
    low-res flow varies over the image and reaches several cells."""
    out = dict(sd)
    for k in (".weight", ".bias"):
        out[RAFT_FLOW_CONV2 + k] = sd[RAFT_FLOW_CONV2 + k] * gain
    return out


def raft_sharp_mask(sd, gain: float):
    """The convex-upsampling mask head's last conv `gain` times larger: saturated 9-way softmaxes."""
    out = dict(sd)
    for k in (".weight", ".bias"):
        out[RAFT_MASK2 + k] = sd[RAFT_MASK2 + k] * gain
    return out


def warp_regime(raw: torch.Tensor, disp: torch.Tensor) -> dict:
    """What a backward warp with displacement `disp` (n, 2, h, w) px and raw mask `raw` (n, 1, h, w) exercised."""
    n, _, h, w = disp.shape
    ys, xs = torch.meshgrid(torch.arange(h), torch.arange(w), indexing="ij")
    cells = torch.floor(disp + torch.stack([xs, ys]).to(disp)) - torch.stack([xs, ys]).to(disp)
    masked = raw <= 0.999
    return {"max displacement": float(disp.abs().max()),
            "all taps outside": int((raw == 0).sum()),
            "masked": int(masked.sum()),
            "masked interior": int(masked[..., 1:-1, 1:-1].sum()),
            "cell offsets": len(torch.unique(cells.permute(0, 2, 3, 1).reshape(-1, 2), dim=0))}


def lookup_regime(coords: torch.Tensor) -> dict:
    """What a RAFT lookup centred at coords (n, 2, H8, W8) exercised at pyramid level 0."""
    n, _, h, w = coords.shape
    ys, xs = torch.meshgrid(torch.arange(h), torch.arange(w), indexing="ij")
    grid = torch.stack([xs, ys]).to(coords)
    off = coords - grid
    x, y = coords[:, 0], coords[:, 1]
    outside = (x < 0) | (x > w - 1) | (y < 0) | (y > h - 1)
    window_outside = (x < -5) | (x > w + 4) | (y < -5) | (y > h + 4)       # all 10 x 10 taps off the map
    return {"max offset": float(off.abs().max()),
            "centres outside": int(outside.sum()),
            "windows outside": int(window_outside.sum()),
            "cell offsets": len(torch.unique((torch.floor(coords) - grid).permute(0, 2, 3, 1).reshape(-1, 2), dim=0))}


# ---- the cases, shared by the CPU premise test and the GPU test
PWC_FRAMES = {(128, 160): dict(seed=3, shift=(1.3, -0.7)), (200, 333): dict(seed=5, shift=(1.3, -0.7)),
              (40, 50): dict(seed=3, shift=(1.3, -0.7))}
# level -> displacements (px of that level) of the uniform warps: fractional both ways, mostly negative, whole pixels
# (5 = DBL_BACKWARD x a power of two at every level: exact), and at level 5 one larger than the map
PWC_UNIFORM = {5: ((3.25, -2.5), (-7.75, 0.5), (5.0, -5.0), (-20.0, 15.0)),
               4: ((3.25, -2.5), (-7.75, 0.5), (5.0, -5.0)),
               3: ((3.25, -2.5), (-7.75, 0.5), (5.0, -5.0)),
               2: ((3.25, -2.5), (-7.75, 0.5), (5.0, -5.0), (-7.75, 3.25))}
PWC_VARYING = {"level 2 x9": {2: 9.0}, "level 4 x75": {4: 75.0}}
# level 2 displacements whose border raw mask 1 - f sits either side of the 0.999 threshold: (dx, dy) -> border mask
PWC_THRESHOLD = {(0.0005, 0.0): 1.0, (0.0015, 0.0): 0.0, (0.0, -0.0005): 1.0, (0.0, -0.0015): 0.0}

RAFT_UNIFORM = (((0.625, -0.375), 6), ((2.25, 1.75), 3), ((-3.5, 0.25), 6), ((9.0, 7.0), 2), ((9.0, 7.0), 6))
RAFT_VARYING_GAIN = 10.0
RAFT_SHARP_GAIN = 20.0

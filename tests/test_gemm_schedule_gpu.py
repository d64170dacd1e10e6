"""Edge cases of the wgmma GEMM's persistent ping-pong schedule (csrc/gemm.cu): 64-row tiles walked row-major over a
grid of min(tiles, SMs) CTAs, the CTA's even tiles on one consumer warpgroup and its odd ones on the other, the two main
loops taking turns.  Tile counts around one and two waves of 132 SMs (an H100 SXM), an odd number of tiles per CTA, a
CTA whose second warpgroup has no tile, N tails and `accumulate`.  The conv mode, which keeps the cooperative schedule
on the same kernel template, is run with split weights, lo_mask and a split output.

Each plain case is compared bitwise against the same product computed as several launches on row slices of A (other
tile counts, other tile-to-CTA assignments: an output element's sum runs over the same K steps in the same order
whatever its tile), and against the fp32 reference within the bars of test_gemm_gpu.py."""
import pytest
import torch

import conv_layout as cl
from conftest import rel_l2
from test_conv_gemm_gpu import run_and_check

import video_features_b200  # noqa: F401  (registers torch.ops.vfeat)

pytestmark = pytest.mark.gpu


def _operands(M, N, K, dev, seed):
    g = torch.Generator(device="cpu").manual_seed(seed)
    a = (torch.randn(M, K, generator=g) * 0.5).half().to(dev)
    b = (torch.randn(N, K, generator=g) * K ** -0.5).half().to(dev)
    bias = torch.randn(N, generator=g).to(dev)
    return a, b, bias


def _ref(a, b, bias, act):
    y = a.float() @ b.float().t() + bias
    return y * torch.sigmoid(1.702 * y) if act == 1 else y


def _slices(M):
    """Row slices of A that start on 64-row tile boundaries and split the tiles unevenly."""
    cuts = sorted({0, M} | {64 * ((M // 64) * f // 7) for f in (1, 3, 4)})
    return [(r0, r1) for r0, r1 in zip(cuts, cuts[1:]) if r1 > r0]


# M, N, K, act, out_f32.  N = 64 runs 64-wide tiles, so the tile count is ceil(M / 64); one CTA per SM on 132 SMs.
CASES = [
    (64, 64, 192, 0, True),           # 1 tile: the second warpgroup has none
    (128, 64, 192, 1, False),         # 2 tiles on 2 CTAs: one tile each
    (131 * 64 - 24, 64, 320, 0, True),    # 131 tiles, M tail
    (132 * 64, 64, 64, 1, False),     # 132 tiles: one full wave, one K block
    (133 * 64, 64, 448, 0, True),     # 133: CTA 0 has 2 tiles, the rest 1 (odd)
    (263 * 64 - 8, 64, 192, 1, False),    # 263: one CTA with 1 tile
    (264 * 64, 64, 576, 0, True),     # 264: two tiles everywhere, 9 K blocks over an 8-stage ring
    (265 * 64, 64, 128, 1, False),    # 265: CTA 0 has 3 tiles (odd)
    (396 * 64 - 40, 64, 64, 0, True),     # 396: three tiles per CTA (odd), M tail
    (97 * 64 + 10, 768, 3072, 0, True),   # 98 row blocks x 4 column tiles (192 wide): the tower's fc2 / patch-embed
    (6000, 3072, 768, 1, False),      # fc1 shape at a smaller M: 256-wide tiles, 12 per row block
    (1000, 200, 320, 0, True),        # N tail inside a 256-wide tile
    (2500, 328, 136, 1, False),       # N tail over two tiles, K tail
    (5000, 40, 256, 0, False),        # narrow N
]


@pytest.mark.parametrize("M,N,K,act,out_f32", CASES)
def test_schedule_matches_row_sliced_launches(cuda_device, M, N, K, act, out_f32):
    a, b, bias = _operands(M, N, K, cuda_device, M + 3 * N + K)
    whole = torch.ops.vfeat.gemm_f16(a, b, bias, None, act, out_f32)
    parts = torch.cat([torch.ops.vfeat.gemm_f16(a[r0:r1].contiguous(), b, bias, None, act, out_f32)
                       for r0, r1 in _slices(M)])
    torch.cuda.synchronize()
    assert torch.equal(whole, parts), "the schedule changed the bits of an output"
    ref = _ref(a, b, bias, act)
    err = rel_l2(whole.float(), ref)
    mx = float((whole.float() - ref).abs().max() / ref.abs().max())
    assert err < (2e-5 if out_f32 else 1.5e-3), err
    assert mx < (1e-4 if out_f32 else 2e-3), mx


@pytest.mark.parametrize("M,N,K", [(133 * 64, 768, 768), (265 * 64 - 8, 64, 3072), (64, 768, 3072)])
def test_schedule_accumulate_matches_row_sliced_launches(cuda_device, M, N, K):
    """out-proj / fc2 style: the fp32 TMA reduce-add into a residual stream, whole against row-sliced launches."""
    a, b, bias = _operands(M, N, K, cuda_device, M + N + K)
    x0 = (torch.randn(M, N, generator=torch.Generator().manual_seed(1)) * 3).to(cuda_device)
    whole, parts = x0.clone(), x0.clone()
    torch.ops.vfeat.gemm_f16_accumulate(whole, a, b, bias, 0)
    for r0, r1 in _slices(M):
        view = parts[r0:r1]
        torch.ops.vfeat.gemm_f16_accumulate(view, a[r0:r1].contiguous(), b, bias, 0)
    torch.cuda.synchronize()
    assert torch.equal(whole, parts)
    assert rel_l2(whole, x0 + _ref(a, b, bias, 0)) < 2e-6


CONV = {c["id"]: c for c in cl.I3D_CASES}


@pytest.mark.parametrize("cid", ["i3d3x3x3-c144-n320-1x11x14", "i3d1x1x1-pair-c480-n192-2x4x14",
                                 "i3d1x1x1-pair-c40-n24-2x4x7"])
def test_schedule_conv_split_weights_and_split_output(cuda_device, cid):
    """Conv mode with nsplit = 2 (W_hi + W_lo, the lo_mask skip of the pair cases) and the split-fp16 output against
    F.conv3d in float64: fp32, fp16 and split outputs, masked rows exactly zero."""
    case = CONV[cid]
    assert case["out"] == "split"
    run_and_check(case, 2, cuda_device, seed=5)

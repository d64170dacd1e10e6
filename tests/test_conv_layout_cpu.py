"""The shifted-row layout of tests/conv_layout.py against F.conv3d / F.conv2d in float64, for every geometry
test_conv_gemm_gpu.py runs: the GPU test's own layout arithmetic is right before the kernel is compared with it."""
import pytest
import torch

import conv_layout as cl

N_CPU = 8     # output channels kept here: the layout does not depend on them


def _check(case, nsplit, mask=True, n_out=N_CPU):
    d = cl.build_case(case, nsplit, seed=3, n_out=n_out)
    vol, f = d["vol"], d["f"]
    y = cl.emulate(d["X"], d["pitch"], vol, f, d["bias"], d["scale"], d["act"], mask=mask, lo_mask=False)
    ref = cl.reference_conv(d["x_eff"], d["w_eff"], d["bias"], d["scale"], d["act"], **d.get("conv", {}))
    if ref.dim() == 4:
        ref = ref.unsqueeze(2)
    got = vol.valid_rows(y)
    assert got.shape == ref.shape
    assert torch.allclose(got, ref, rtol=1e-12, atol=1e-12 * float(ref.abs().max())), float((got - ref).abs().max())
    # skipping W_lo on the lo_mask blocks, as the kernel does, moves the valid rows by a_lo . w_lo only
    y_skip = cl.emulate(d["X"], d["pitch"], vol, f, d["bias"], d["scale"], d["act"], mask=mask)
    assert float((vol.valid_rows(y_skip) - ref).abs().max()) <= 2.0 ** -22 * float(ref.abs().max())
    assert f["lo_mask"] == 0 or nsplit == 2
    return y, vol, f


@pytest.mark.parametrize("case", cl.ALL_CASES, ids=[c["id"] for c in cl.ALL_CASES])
@pytest.mark.parametrize("nsplit", [1, 2])
def test_emulator_equals_float64_convolution(case, nsplit):
    y, vol, f = _check(case, nsplit)
    keep = vol.keep()
    assert bool((y[~keep] == 0).all()) and int(keep.sum()) == vol.n * (vol.t1 - vol.t0) * (vol.h1 - vol.h0) * (vol.w1 - vol.w0)
    assert f["ntaps"] <= 64 and f["k_per_tap"] % 8 == 0 and case["pitch"] % 8 == 0
    assert f["Wt"].shape == (N_CPU, nsplit * f["ntaps"] * f["k_per_tap"])


@pytest.mark.parametrize("case", cl.ENGINE_CASES, ids=[c["id"] for c in cl.ENGINE_CASES])
def test_engine_layouts_equal_strided_float64_convolution(case):
    """The ResNet / R(2+1)D repacks and filters (phase, temporal phase, subsample, stems, padded widths) against
    F.conv2d / F.conv3d with the real strides and padding, at every output channel: pad channels come out exactly 0."""
    y, vol, f = _check(case, 2, n_out=None)
    N, co = case["N"], case.get("co", case["N"])
    assert f["Wt"].shape == (N, 2 * f["ntaps"] * f["k_per_tap"]) and f["ntaps"] <= 64 and f["k_per_tap"] % 8 == 0
    assert bool((y[:, co:] == 0).all()) and bool((y[~vol.keep()] == 0).all())


def test_engine_lo_masks():
    """The restated lo_mask builder against masks derived by hand from the layouts, including bit 63 of the 64-block
    taps.  (The engines' own upload_conv masks are compared with this builder, conv by conv, on the GPU:
    test_conv_gemm_resnet_r21d_gpu.py.)"""
    m = {c["id"]: cl.build_case(c, 2, seed=0, n_out=8)["f"]["lo_mask"] for c in cl.ENGINE_CASES}
    # layer4 1x1 at cin 2048: [hi 2048 | lo 2048], blocks 32 .. 63 lo only
    assert m["resnet-1x1-c2048-9"] == ((1 << 64) - 1) ^ ((1 << 32) - 1)
    # stride-2 3x3 at width 512: 4 phases of [hi 512 | lo 512], the lo blocks 16p + 8 .. 16p + 15
    assert m["resnet-3x3s2-c512-9"] == sum(((1 << 8) - 1) << (16 * p + 8) for p in range(4))
    assert m["resnet-3x3s2-c512-9"] >> 63 == 1
    # the stems: every K block holds hi columns
    assert m["resnet-stem-115"] == 0 and m["r21d-stem-59-T5"] == 0
    # 48-wide pair rows of 45 channels: block 0 holds hi 0..44 and lo 48..63, block 1 only lo
    assert m["r21d-temporal-c45-59-T5"] == 0b10
    # temporal phase rows [even | odd] of 232-wide pairs: hi at 0..229 and 464..693 (tap 1), 464..693 (tap 0)
    assert m["r21d-temporal2-c230-30-T5"] == sum(1 << b for b in (4, 5, 6, 11, 12, 13, 14))
    # the downsample reads 2C columns of an 8C phase row: hi blocks 0..15, lo 16..31
    assert m["resnet-down-c1024-9"] == ((1 << 32) - 1) ^ ((1 << 16) - 1)


def test_lo_mask_matches_the_engines():
    """lo_mask as i3d.cu prepare_unit (1x1x1 over [hi C | lo C]: K blocks at or past column C) and raft.cu upload_conv
    (HX rows: blocks alternately hi / lo) build it."""
    for case in cl.I3D_CASES:
        if case["k"] != (1, 1, 1):
            continue
        C = case["x"][1]
        f = cl.build_case(case, 2, seed=0, n_out=8)["f"]
        kb = (2 * C + 63) // 64
        assert f["lo_mask"] == sum(1 << kk for kk in range(kb) if kk * 64 >= C), case["id"]
    zr = next(c for c in cl.RAFT_CASES if c["id"].startswith("raft1x5"))
    f = cl.build_case(zr, 2, seed=0, n_out=8)["f"]
    assert f["k_per_tap"] == 5 * 768 and f["ntaps"] == 1
    assert f["lo_mask"] == sum(1 << (12 * d + b) for d in range(5) for b in (2, 3, 6, 7, 10, 11))
    q = next(c for c in cl.RAFT_CASES if c["id"].startswith("raft5x1"))
    f = cl.build_case(q, 2, seed=0, n_out=8)["f"]
    assert f["ntaps"] == 5 and f["lo_mask"] == sum(1 << b for b in (2, 3, 6, 7, 10, 11))
    assert cl.build_case(q, 1, seed=0, n_out=8)["f"]["lo_mask"] == 0


def test_tap_offsets_match_the_engines():
    """i3d.cu run_unit: (dt-1)*Hp*Wp + (dh-1)*Wp - 1; raft.cu run_conv: dh*Wp + dw0."""
    c = cl.I3D_CASES[1]
    d = cl.build_case(c, 1, seed=0, n_out=8)
    v = d["vol"]
    assert d["f"]["tap_off"] == [(j // 3 - 1) * v.Hp * v.Wp + (j % 3 - 1) * v.Wp - 1 for j in range(9)]
    c = next(c for c in cl.RAFT_CASES if "8x8" in c["id"])
    d = cl.build_case(c, 1, seed=0, n_out=8)
    v = d["vol"]
    assert d["f"]["tap_off"] == [(a - 4) * v.Wp + (b - 4) for a in range(8) for b in range(8)]


def test_unmasked_emulation_reads_the_real_rows():
    """Without the mask the border rows read across sample boundaries, the guard rows and the rows past P; the
    emulator follows the buffer (the GPU test compares the kernel with it there)."""
    case = next(c for c in cl.RAFT_CASES if c["id"] == "raft3x3-pair-c64")
    d = cl.build_case(case, 2, seed=1, n_out=8)
    y = cl.emulate(d["X"], d["pitch"], d["vol"], d["f"], mask=False)
    assert float(y[~d["vol"].keep()].abs().max()) > 0
    # shifting the junk past P changes the last border row and nothing inside the valid region
    X2 = d["X"].clone()
    X2[d["vol"].P:] = 0
    y2 = cl.emulate(X2, d["pitch"], d["vol"], d["f"], mask=False)
    assert torch.equal(y2[d["vol"].keep()], y[d["vol"].keep()])
    assert not torch.equal(y2, y)

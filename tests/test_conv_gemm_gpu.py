"""The shifted-row convolution mode of the wgmma GEMM (vf_conv_gemm_f16 -> conv_gemm_f16), which runs every I3D and RAFT
convolution, against F.conv3d / F.conv2d in float64 on the operands as the kernel sees them (fp16 activations or hi + lo
pair rows, fp16 weights or W_hi + W_lo).  The layouts come from tests/conv_layout.py, which test_conv_layout_cpu.py
checks against the same float64 convolutions without a GPU.

Bars (rel-L2 / max-abs relative to max|ref|):
  fp32 out      rel-L2 <= 2e-5, max-abs <= 1e-4 (fp16 products are exact in fp32: only the summation order differs,
                and the a_lo . w_lo terms of lo_mask blocks are below fp32 resolution; a dropped W_lo pass costs ~2^-12
                per weight and fails it)
  fp16 out      bit-equal to fp16 of the fp32 result of the same operands, and within 1 fp16 ulp of fp16(ref) plus
                the fp32 bar's max-abs.  The fp32 sum's error is absolute (it grows with K: 1.3e-5 max|ref| at
                K = 2 x 27 x 192 measured), so outputs near zero, whose ulp is finer than that, cannot be held to
                1 ulp: 5.25 ulp was measured at 2^-20 max|ref| with the accumulator inside the fp32 bar
  split out     hi + lo at the fp32 bar; hi bit-equal to the plain fp16 output
  masked rows   exactly 0.0 (with bias and sigmoid a missed row would read 0.5); rows past P keep their sentinel
Measured worst cases, one H100 80GB HBM3 (400 W power limit), every case below:
  fp32 out      rel-L2 1.10e-5, max-abs 1.28e-5 (i3d 3x3x3 C = 192, N = 384, nsplit = 2: the longest K)
  fp16 out      0.83 of (1 ulp + 1e-4 max|ref|) (raft 7x7 merged); bit-equal to fp16 of the fp32 result everywhere
  split out     hi + lo rel-L2 8.0e-6, max-abs 9.6e-6
  unmasked      rel-L2 2.9e-6, max-abs 5.4e-6 against the emulation
  W_lo dropped  rel-L2 2.0e-4 (fails the fp32 bar tenfold)
test_zz_report_measured prints the same figures for a run (pytest -s).
"""
import ctypes as C

import pytest
import torch

import conv_layout as cl
from conftest import rel_l2

import video_features_b200  # noqa: F401

pytestmark = pytest.mark.gpu

# worst case per bar over the tests of one session (test_zz_report_measured)
MEASURED = {}

SENT16 = 7.0
SENT32 = -3.5


def _lib():
    from video_features_b200 import _lib
    return _lib


def _stream():
    return torch.cuda.current_stream().cuda_stream


def launch(d, dev, out, N, ldd, c_off=0, split_off=0, region=True, lo_mask=None, nsplit=None, ntaps=None, extra_rows=8):
    """One vf_conv_gemm_f16 call on the case operands d (conv_layout.build_case); returns the whole output buffer
    (P + extra_rows rows of pitch ldd, sentinel-filled before the call)."""
    lib = _lib()
    vol, f = d["vol"], d["f"]
    P = vol.P
    X = d["X"].to(dev)
    Wt = f["Wt"].to(dev)
    bias, scale = d["bias"].float().to(dev), d["scale"].float().to(dev)
    f32 = out == "f32"
    D = torch.full((P + extra_rows, ldd), SENT32 if f32 else SENT16, dtype=torch.float32 if f32 else torch.float16,
                   device=dev)
    nt = f["ntaps"] if ntaps is None else ntaps
    taps = (C.c_int * max(nt, 1))(*(list(f["tap_off"]) + [0] * nt)[:nt])
    reg = (C.c_int * 9)(*(vol.region() if region is True else region)) if region else None
    with torch.cuda.device(dev):
        lib.check(lib.lib().vf_conv_gemm_f16(
            X.data_ptr(), d["pitch"], P, Wt.data_ptr(), N, nt, f["k_per_tap"], taps,
            f["nsplit"] if nsplit is None else nsplit, f["lo_mask"] if lo_mask is None else lo_mask, vol.row0, reg,
            D.data_ptr() + c_off * D.element_size(), ldd, int(f32), split_off, bias.data_ptr(), scale.data_ptr(),
            d["act"], _stream()))
    torch.cuda.synchronize()
    return D


def reference(d, dev):
    """float64 [P, N]: the valid rows from F.conv3d / F.conv2d (on the GPU, in float64), zeros elsewhere."""
    vol = d["vol"]
    ref = cl.reference_conv(d["x_eff"].to(dev), d["w_eff"].to(dev), d["bias"].to(dev), d["scale"].to(dev), d["act"],
                            **d.get("conv", {}))
    if ref.dim() == 4:
        ref = ref.unsqueeze(2)
    full = torch.zeros(vol.P, ref.shape[1], dtype=torch.float64, device=dev)
    keep = vol.keep().to(dev)
    full[keep] = ref.permute(0, 2, 3, 4, 1).reshape(-1, ref.shape[1])
    return full, keep


def _record(name, value):
    MEASURED[name] = max(MEASURED.get(name, 0.0), value)


def check_f32(y, ref, what):
    err = rel_l2(y, ref)
    mx = float((y.double() - ref).abs().max() / ref.abs().max())
    _record("fp32 rel-L2", err)
    _record("fp32 max-abs", mx)
    print(f"{what}: rel-L2 {err:.2e}, max-abs {mx:.2e}")
    assert err <= 2e-5 and mx <= 1e-4, (what, err, mx)


def fp16_ulp(r16):
    a = r16.float().abs().clamp_min(2.0 ** -14)
    return torch.exp2(torch.floor(torch.log2(a)) - 10).double()


def check_f16(y16, ref, what):
    r16 = ref.half()
    tol = fp16_ulp(r16) + 1e-4 * float(ref.abs().max())
    excess = float(((y16.double() - r16.double()).abs() / tol).max())
    _record("fp16 |out - fp16(ref)| over (ulp + 1e-4 max|ref|)", excess)
    print(f"{what}: max |out - fp16(ref)| = {excess:.2f} x (ulp + 1e-4 max|ref|)")
    assert excess <= 1.0, (what, excess)


def _output_of(case):
    if case["out"] == "split":
        ctot = case["ctot"]
        return dict(ldd=2 * ctot, c_off=case["c_off"], split_off=ctot)
    return dict(ldd=case["N"] + 8, c_off=0, split_off=0)


def run_and_check(case, nsplit, dev, seed=11):
    """Returns the output buffers of the launches: fp32 always, fp16 and split when the case's output has them."""
    d = cl.build_case(case, nsplit, seed=seed)
    N, P = case["N"], d["vol"].P
    ref, keep = reference(d, dev)
    o = _output_of(case)
    c0 = o["c_off"]
    # fp32 out: the numeric bar, the mask and the rows past P
    D32 = launch(d, dev, "f32", N, N + 8)
    y32 = D32[:P, :N]
    check_f32(y32, ref, f"{case['id']} nsplit={nsplit} fp32")
    assert bool((y32[~keep] == 0).all()), "rows outside the valid region must be written as 0.0"
    assert bool((D32[P:] == SENT32).all()) and bool((D32[:, N:] == SENT32).all())
    if case["out"] == "f32":
        return dict(f32=D32)
    # fp16 out: the rounding of the fp32 result above
    D16 = launch(d, dev, "f16", N, N + 8)
    y16 = D16[:P, :N]
    assert torch.equal(y16, y32.half()), "fp16 output must be the fp16 rounding of the same accumulator"
    check_f16(y16, ref, f"{case['id']} nsplit={nsplit} fp16")
    assert bool((D16[P:] == SENT16).all()) and bool((D16[:, N:] == SENT16).all())
    if case["out"] != "split":
        return dict(f32=D32, f16=D16)
    # split out into a channel slice of a wider concat row: columns outside both halves stay untouched
    ctot, so = o["split_off"], o["split_off"]
    Ds = launch(d, dev, "split", N, o["ldd"], c_off=c0, split_off=so)
    hi, lo = Ds[:P, c0:c0 + N], Ds[:P, so + c0:so + c0 + N]
    assert torch.equal(hi, y16), "hi half must equal the plain fp16 output"
    check_f32(hi.double() + lo.double(), ref, f"{case['id']} nsplit={nsplit} split hi+lo")
    assert torch.equal(lo, (y32 - y16.float()).half())
    untouched = torch.ones(Ds.shape[1], dtype=torch.bool)
    untouched[c0:c0 + N] = False
    untouched[so + c0:so + c0 + N] = False
    assert bool((Ds[:P, untouched.to(dev)] == SENT16).all()) and bool((Ds[P:] == SENT16).all())
    return dict(f32=D32, f16=D16, split=Ds)


@pytest.mark.parametrize("nsplit", [1, 2])
@pytest.mark.parametrize("case", cl.I3D_CASES, ids=[c["id"] for c in cl.I3D_CASES])
def test_i3d_conv_matches_float64(cuda_device, case, nsplit):
    run_and_check(case, nsplit, cuda_device)


@pytest.mark.parametrize("case", cl.RAFT_CASES, ids=[c["id"] for c in cl.RAFT_CASES])
def test_raft_conv_matches_float64(cuda_device, case):
    nsplit = 1 if "8x8" in case["id"] else 2
    run_and_check(case, nsplit, cuda_device)


@pytest.mark.parametrize("cid", ["i3d3x3x3-c24-n16-2x4x14", "raft3x3-pair-c64", "raft7x7-unmerged-49taps"])
def test_conv_without_mask_matches_emulator(cuda_device, cid):
    """No mask: every row, including the border rows whose taps cross sample boundaries, read the guard rows or run
    past the last row, against the float64 emulation of the same buffer."""
    case = next(c for c in cl.ALL_CASES if c["id"] == cid)
    d = cl.build_case(case, 2, seed=5)
    N, P = case["N"], d["vol"].P
    D = launch(d, cuda_device, "f32", N, N, region=False)
    # guard rows and rows past P hold arbitrary data, also in lo-half columns: emulate the skipped W_lo passes exactly
    ref = cl.emulate(d["X"].to(cuda_device), d["pitch"], d["vol"], d["f"], d["bias"].to(cuda_device),
                     d["scale"].to(cuda_device), d["act"], mask=False, lo_mask=True)
    check_f32(D[:P], ref, f"{cid} unmasked")


def test_conv_dropped_w_lo_pass_fails_the_bar(cuda_device):
    """The fp32 bar is tight enough to see the W_lo pass go missing: the same operands with every W_lo pass skipped."""
    case = next(c for c in cl.I3D_CASES if c["id"].startswith("i3d3x3x3-c96"))
    d = cl.build_case(case, 2, seed=11)
    ref, _ = reference(d, cuda_device)
    kpt = (d["f"]["k_per_tap"] + 63) // 64
    D = launch(d, cuda_device, "f32", case["N"], case["N"], lo_mask=(1 << kpt) - 1)
    err = rel_l2(D[:d["vol"].P], ref)
    print(f"W_lo skipped: rel-L2 {err:.2e}")
    assert err > 4 * 2e-5


def test_activations_saturate_cleanly_through_the_conv_epilogue(cuda_device):
    """fp32 sigmoid / tanh with pre-activations pushed to +-100 by the bias: no NaN, exact 0 / +-1 at saturation."""
    case = next(c for c in cl.RAFT_CASES if c["id"].startswith("raft1x5"))
    for act, lo_v, hi_v in ((cl.ACT_SIGMOID, 0.0, 1.0), (cl.ACT_TANH, -1.0, 1.0)):
        d = cl.build_case(case, 2, seed=2)
        d["act"] = act
        N = case["N"]
        d["bias"] = torch.where(torch.arange(N) % 2 == 0, 100.0, -100.0)
        D = launch(d, cuda_device, "f32", N, N)
        y = D[:d["vol"].P][d["vol"].keep().to(cuda_device)]
        assert torch.isfinite(y).all()
        assert bool((y[:, 0::2] == hi_v).all()) and bool((y[:, 1::2] == lo_v).all())


def test_conv_rejects_bad_geometry(cuda_device):
    """Argument checks of conv_gemm_f16, each a VfError before anything is launched."""
    VfError = _lib().VfError
    pair = next(c for c in cl.I3D_CASES if c["id"].startswith("i3d1x1x1-pair-c40"))
    d = cl.build_case(pair, 2, seed=0)                         # k_per_tap 80: 2 K blocks
    N = pair["N"]
    assert d["f"]["lo_mask"] == 0b10
    launch(d, cuda_device, "f32", N, N)                        # the valid call
    with pytest.raises(VfError, match="lo_mask"):
        launch(d, cuda_device, "f32", N, N, lo_mask=0b110)     # bit 2 >= kpt
    with pytest.raises(VfError, match="lo_mask"):
        launch(d, cuda_device, "f32", N, N, lo_mask=1 << 63)
    with pytest.raises(VfError, match="nsplit"):
        launch(d, cuda_device, "f32", N, N, nsplit=3)
    with pytest.raises(VfError, match="nsplit"):
        launch(d, cuda_device, "f32", N, N, nsplit=0)
    # a tap of more than 64 K blocks cannot carry a mask (lo_mask >> kk with kk >= 64)
    gru = next(c for c in cl.RAFT_CASES if c["id"].startswith("raft1x5"))
    big = dict(gru, pitch=1024, chan=list(range(384)), chan_lo=[512 + c for c in range(384)], row0=0)
    d2 = cl.build_case(big, 2, seed=0, n_out=8)
    assert d2["f"]["k_per_tap"] == 5 * 1024 and d2["f"]["lo_mask"] == 0
    launch(d2, cuda_device, "f32", 8, 8)
    with pytest.raises(VfError, match="lo_mask"):
        launch(d2, cuda_device, "f32", 8, 8, lo_mask=1)
    # 64 taps is the limit (raft8x8-unmerged-64taps runs it); 65 are rejected
    eight = next(c for c in cl.RAFT_CASES if "8x8" in c["id"])
    d3 = cl.build_case(eight, 1, seed=0)
    assert d3["f"]["ntaps"] == 64
    with pytest.raises(VfError, match="taps"):
        launch(d3, cuda_device, "f32", eight["N"], eight["N"], ntaps=65)
    with pytest.raises(VfError):
        launch(d3, cuda_device, "f32", eight["N"], eight["N"], ntaps=0)
    # a mask volume with an empty extent (the row -> position arithmetic divides by it)
    bad = d3["vol"].region()
    bad[2] = 0
    with pytest.raises(VfError, match="mask volume"):
        launch(d3, cuda_device, "f32", eight["N"], eight["N"], region=bad)


def test_zz_report_measured(cuda_device):
    """Prints the worst case per bar over the tests above (run in the same session)."""
    for k, v in sorted(MEASURED.items()):
        print(f"measured worst case {k}: {v:.3e}")

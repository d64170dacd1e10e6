"""The conv-GEMM geometries of the ResNet and R(2+1)D engines (csrc/resnet.cu, csrc/r21d.cu) through vf_conv_gemm_f16 at
the real stage volumes, against F.conv2d / F.conv3d in float64 with the real strides and padding: stride-2 3x3 over
the 2-D phase repack, the stride-2 1x1 downsample reading phase (0, 0) of an 8C row, the stems' phase volumes, the
temporal convs (stride 1 over masked border frames, stride 2 over the temporal phase repack), the (2,2,2) subsample,
widths padded to a multiple of 8, and the taps of exactly 64 K blocks whose lo_mask has bit 63 set.  Layouts and
filters come from tests/conv_layout.py (ENGINE_CASES), pinned against the same float64 convolutions on the CPU by
test_conv_layout_cpu.py.

Every case runs with split weights (nsplit = 2) and the engines' split output (ldo = 2 n_out, split_off = n_out), and
with fp32 and fp16 outputs, under test_conv_gemm_gpu.py's bars (run_and_check): fp32 rel-L2 <= 2e-5 and max-abs <=
1e-4 of max|ref|, masked rows exactly 0, rows past P untouched.  Pad output channels must be exactly 0 in both halves.

Measured, one H100 80GB HBM3 (700 W power limit), fp32 out against float64 (split hi + lo the same to two digits):
  stems (K 512)                    8.6e-7 / 1.2e-6      temporal c45 (K 3 x 96)          5.7e-7 / 8.7e-7
  3x3 c64 at 58^2                  2.1e-6 / 2.7e-6      stride-2 3x3 c64 at 30^2         2.1e-6 / 2.5e-6
  stride-2 3x3 c256 at 16^2        7.9e-6 / 8.3e-6      stride-2 3x3 c512 at 9^2 (bit 63) 1.5e-5 / 1.6e-5
  downsample c64                   3.4e-7 / 5.7e-7      downsample c1024 (8192 pitch)    4.3e-6 / 5.2e-6
  1x1 c2048 (bit 63)               8.6e-6 / 1.1e-5
  temporal2 c230 (K 2 x 928)       2.3e-6 / 2.6e-6      subsample + 1x1x1 c64            3.5e-7 / 6.4e-7
  spatial c256 -> 460 at 16^2      7.7e-6 / 9.1e-6      temporal c921 at 9^2, T' = 1     3.8e-6 / 4.3e-6
  (rel-L2 / max-abs÷max|ref|.)  The error grows with K: it is the fp32 accumulation, the operands are exact.  The bit-63
  control matches the lo_mask emulation at 7.1e-7, which sits 4.8e-4 from the emulation without lo_mask.  Layer4's
  stride-2 conv as one launch 1.58e-5, as four one-tap launches summed in float64 6.03e-6
  (test_long_k_error_is_the_accumulation).

The filters the engines actually upload are read back for every conv of ResNet-18/34/50/101/152 and R(2+1)D-18 and
must equal the restated ones bit for bit (test_*_uploads_match_the_restated_filters).
"""
import pytest
import torch

import conv_layout as cl
from conftest import rel_l2
from test_conv_gemm_gpu import check_f32, launch, run_and_check

import video_features_b200  # noqa: F401

pytestmark = pytest.mark.gpu

CASES = {c["id"]: c for c in cl.ENGINE_CASES}


@pytest.mark.parametrize("case", cl.ENGINE_CASES, ids=[c["id"] for c in cl.ENGINE_CASES])
def test_engine_conv_matches_float64(cuda_device, case):
    out = run_and_check(case, 2, cuda_device)
    N, co = case["N"], case.get("co", case["N"])
    if co < N:
        P = out["f32"].shape[0] - 8
        assert bool((out["f32"][:P, co:N] == 0).all()), "pad output channels must be exactly 0"
        hi, lo = out["split"][:P, co:N], out["split"][:P, N + co:2 * N]
        assert bool((hi == 0).all()) and bool((lo == 0).all()), "pad channels must be 0 in both halves"


def test_lo_mask_bit63_is_honoured(cuda_device):
    """ResNet layer4's 1x1 conv at cin 2048: a tap of 64 K blocks, the lo halves in blocks 32 .. 63.  Block 63 is
    filled with arbitrary values of magnitude 32 and given a W_lo of half an fp16 ulp, so that its W_lo pass moves the
    output far beyond the fp32 bar: the kernel must match the emulation that skips it."""
    case = CASES["resnet-1x1-c2048-9"]
    d = cl.build_case(case, 2, seed=13)
    f, vol = d["f"], d["vol"]
    assert (f["lo_mask"] >> 63) & 1 and f["k_per_tap"] == 64 * 64
    d["act"] = cl.ACT_NONE
    Kb = f["k_per_tap"]
    blk = slice(63 * 64, 64 * 64)
    g = torch.Generator().manual_seed(14)
    X = d["X"].clone()
    X[:, blk] = (torch.rand(X.shape[0], 64, generator=g) * 64 - 32).half()
    Wt = f["Wt"].clone()
    h = torch.exp2(-torch.randint(4, 7, (Wt.shape[0], 64), generator=g).double())
    h = h * torch.where(torch.rand(h.shape, generator=g) < 0.5, -1.0, 1.0)
    Wt[:, blk] = h.half()
    Wt[:, Kb + 63 * 64:Kb + 64 * 64] = (h * 0.98 * 2.0 ** -11).half()
    d["X"], d["f"] = X, dict(f, Wt=Wt)
    N, P = case["N"], vol.P
    D = launch(d, cuda_device, "f32", N, N)
    args = (d["X"].to(cuda_device), d["pitch"], vol, d["f"], d["bias"].to(cuda_device), d["scale"].to(cuda_device),
            d["act"])
    skip = cl.emulate(*args, lo_mask=True)
    full = cl.emulate(*args, lo_mask=False)
    check_f32(D[:P], skip, "resnet-1x1-c2048-9 block 63 arbitrary, lo_mask bit 63")
    apart = rel_l2(full, skip)
    print(f"emulation without lo_mask: rel-L2 {apart:.2e} from the one with it")
    assert apart > 10 * 2e-5, apart


# ------------------------------------------------------------- the engines' uploaded filters against the restatement
# Every conv of every depth as resnet.cu / r21d.cu uploaded it (vf_resnet_conv / vf_r21d_conv) must equal
# conv_layout.engine_filter on the same state-dict weights, bit for bit: W_hi | W_lo with the pad rows zero, lo_mask
# (bit 63 of layer4's 64-block taps included), the tap shifts, and the folded BatchNorm scale / bias (pad channels 0).
# The restated filters are tied to F.conv by test_conv_layout_cpu.py and to the kernel by the tests above, so an
# upload_conv that drops a lo column, a W_lo row or a mask bit fails here at any depth.

def _resnet_kinds(depth):
    """(conv key, BatchNorm key, conv_layout kind) in vf_resnet_conv's order: resnet.cu vf_resnet_create's walk."""
    from oracle import resnet_net
    bottleneck, layers = resnet_net.LAYERS[depth]
    out = [("conv1", "bn1", "stem")]
    cin = 64
    for L, nb in enumerate(layers):
        cout = (256 if bottleneck else 64) << L
        for b in range(nb):
            p, s2 = f"layer{L + 1}.{b}", b == 0 and L > 0
            if bottleneck:
                out += [(p + ".conv1", p + ".bn1", "same"), (p + ".conv2", p + ".bn2", "stride2" if s2 else "same"),
                        (p + ".conv3", p + ".bn3", "same")]
            else:
                out += [(p + ".conv1", p + ".bn1", "stride2" if s2 else "same"), (p + ".conv2", p + ".bn2", "same")]
            if s2 or (cin if b == 0 else cout) != cout:
                out.append((p + ".downsample.0", p + ".downsample.1", "same"))
        cin = cout
    return out


def _r21d_kinds():
    """The same for vf_r21d_conv: r21d.cu vf_r21d_create's walk."""
    out = [("stem.0", "stem.1", "stem"), ("stem.3", "stem.4", "temporal")]
    for L in range(4):
        for b in range(2):
            p, s2 = f"layer{L + 1}.{b}", b == 0 and L > 0
            out += [(p + ".conv1.0.0", p + ".conv1.0.1", "stride2" if s2 else "same"),
                    (p + ".conv1.0.3", p + ".conv1.1", "temporal2" if s2 else "temporal"),
                    (p + ".conv2.0.0", p + ".conv2.0.1", "same"), (p + ".conv2.0.3", p + ".conv2.1", "temporal")]
            if b == 0 and L > 0:
                out.append((p + ".downsample.0", p + ".downsample.1", "point"))
    return out


def _check_uploads(eng, sd, kinds, pad):
    vol = cl.Vol(1, 1, 1, 1, 0, 1, 0, 1, 0, 1)          # tap_off is not compared: the engine reports tap shifts
    masks64 = 0
    for i, (conv, bn, kind) in enumerate(kinds):
        got = eng.conv(i)
        w = sd[conv + ".weight"].double()
        co, ci = w.shape[:2]
        n_out = cl.pad8(co) if pad else co
        f = cl.engine_filter(kind, w, vol, ci_p=cl.pad8(ci) if pad else ci, n_out=n_out)
        what = f"{i} {conv} ({kind})"
        assert (got["n_out"], got["ntaps"], got["k_per_tap"]) == (n_out, f["ntaps"], f["k_per_tap"]), what
        assert got["shifts"] == f["shifts"], what
        assert got["lo_mask"] == f["lo_mask"], (what, hex(got["lo_mask"]), hex(f["lo_mask"]))
        assert torch.equal(got["w"].cpu(), f["Wt"]), what
        s = sd[bn + ".weight"].double() / torch.sqrt(sd[bn + ".running_var"].double() + 1e-5)
        sh = sd[bn + ".bias"].double() - sd[bn + ".running_mean"].double() * s
        zeros = torch.zeros(n_out - co, dtype=torch.float32)
        assert torch.equal(got["scale"].cpu(), torch.cat([s.float(), zeros])), what
        assert torch.equal(got["bias"].cpu(), torch.cat([sh.float(), zeros])), what
        masks64 += (got["lo_mask"] >> 63) & 1
    with pytest.raises(_vf_error(), match="outside"):
        eng.conv(len(kinds))
    return masks64


def _vf_error():
    from video_features_b200._lib import VfError
    return VfError


@pytest.mark.parametrize("depth", [18, 34, 50, 101, 152])
def test_resnet_uploads_match_the_restated_filters(cuda_device, depth):
    from oracle import resnet_net
    from video_features_b200.resnet_engine import ResNetEngine
    sd = resnet_net.stand_in_state_dict(depth)
    eng = ResNetEngine(sd, depth, 0, max_frames=1)
    kinds = _resnet_kinds(depth)
    n64 = _check_uploads(eng, sd, kinds, pad=False)
    # bottlenecks: layer4.0 conv2 (k_per_tap 4096) and the conv1 of layer4's later blocks (cin 2048) have 64 K blocks
    assert n64 == (3 if depth >= 50 else 0), n64
    eng.close()


def test_r21d_uploads_match_the_restated_filters(cuda_device):
    from oracle import r21d_net
    from video_features_b200.r21d_engine import R21DEngine
    sd = r21d_net.stand_in_state_dict()
    eng = R21DEngine(sd, 0, max_clips=1, max_T=1)
    _check_uploads(eng, sd, _r21d_kinds(), pad=True)
    eng.close()


def test_long_k_error_is_the_accumulation(cuda_device):
    """Where the fp32 error of a long-K conv comes from: layer4's stride-2 conv (4 taps of 64 K blocks, K = 16k with
    both weight passes) as one launch, and as four one-tap launches summed in float64.  The operands and the exact fp16
    products are the same; only the length of the accumulation chain differs.  A shorter chain cutting the error by
    more than half pins it on the accumulation, not on the operands or the layout."""
    case = CASES["resnet-3x3s2-c512-9"]
    d = cl.build_case(case, 2, seed=21)
    d["act"] = cl.ACT_NONE
    N, P, f = case["N"], d["vol"].P, d["f"]
    d["scale"], d["bias"] = torch.ones(N), torch.zeros(N)
    from test_conv_gemm_gpu import reference
    ref, keep = reference(d, cuda_device)
    whole = launch(d, cuda_device, "f32", N, N)[:P].double()
    kpt, Kb = f["k_per_tap"], f["ntaps"] * f["k_per_tap"]
    parts = torch.zeros_like(whole)
    for j in range(f["ntaps"]):
        Wj = torch.cat([f["Wt"][:, j * kpt:(j + 1) * kpt], f["Wt"][:, Kb + j * kpt:Kb + (j + 1) * kpt]], dim=1)
        dj = dict(d, f=dict(f, Wt=Wj.contiguous(), ntaps=1, tap_off=[f["tap_off"][j]]))
        parts += launch(dj, cuda_device, "f32", N, N)[:P].double()
    parts = parts * keep[:, None]
    e_whole, e_parts = rel_l2(whole, ref), rel_l2(parts, ref)
    print(f"K = 4 x 4096 in one chain: rel-L2 {e_whole:.2e}; four chains of 4096 summed in float64: {e_parts:.2e}")
    assert e_parts < 0.5 * e_whole, (e_whole, e_parts)

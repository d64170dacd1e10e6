"""wgmma GEMM (vf_gemm_f16 through the C ABI) against a plain fp32 torch reference of the same op."""
import pytest
import torch

from conftest import rel_l2

import video_features_b200  # noqa: F401  (registers torch.ops.vfeat)

pytestmark = pytest.mark.gpu


def _ref(a, b, bias, scale, act):
    y = a.float() @ b.float().t()
    if scale is not None:
        y = y * scale
    if bias is not None:
        y = y + bias
    if act == 1:
        y = y * torch.sigmoid(1.702 * y)
    elif act == 2:
        y = torch.relu(y)
    elif act == 3:
        y = torch.sigmoid(y)
    elif act == 4:
        y = torch.tanh(y)
    return y


CASES = [
    # M, N, K, bias, scale, act, out_f32           (tile: 128 rows x BN = 64 / 128 / 192 / 256 columns, the width
    #                                               that pads N least; one CTA per SM, tiles strided over the grid)
    (128, 256, 64, False, False, 0, True),
    (256, 256, 128, False, False, 0, True),
    (300, 256, 768, True, False, 0, True),
    (300, 128, 200, True, False, 0, True),       # K tail (zero-filled by TMA), BN=128
    (77, 64, 64, True, True, 2, False),          # BN=64, M tail, scale+relu, fp16 out
    (500, 96, 320, True, False, 0, True),        # N tail inside a 128-wide tile (clipped per element)
    (500, 200, 320, True, True, 2, False),       # N tail inside a 256-wide tile, fp16 out
    (1000, 40, 64, True, False, 0, False),       # narrow N (I3D-style channel counts)
    (1000, 8, 64, True, False, 0, True),         # N = 8 / 16 / 24: I3D branch_2.0 widths, one 64-wide tile
    (1000, 16, 200, True, True, 2, False),
    (700, 24, 136, True, False, 0, True),
    (1, 256, 768, True, False, 0, True),         # M = 1: one row of a 128-row tile
    (1, 96, 64, True, True, 1, False),
    (6000, 2304, 768, True, False, 0, False),    # ViT QKV
    (6000, 768, 768, True, False, 0, True),      # ViT out-proj
    (6000, 3072, 768, True, False, 1, False),    # ViT fc1 + QuickGELU
    (6000, 768, 3072, True, False, 0, True),     # ViT fc2
    (120, 512, 768, False, False, 0, True),      # final projection (one partial 128-row tile)
    (20000, 768, 768, True, False, 0, True),     # many tiles per CTA (persistent loop, barrier phase wrap)
    (3000, 192, 320, True, True, 2, False),      # one 192-wide tile (I3D / RAFT channel counts), fp16 out
    (3000, 160, 192, True, False, 0, True),      # 192-wide tile, clipped N, fp32 out
    (40000, 384, 256, True, False, 2, False),    # two 192-wide tiles per row block, many tiles per CTA
    (700, 288, 128, False, False, 0, True),      # 288 -> 2 x 192
    (11760, 768, 3072, False, False, 0, True),   # patch embedding
    (3000, 256, 384, True, True, 3, True),       # sigmoid (RAFT GRU z / r gates), fp32 out
    (3000, 128, 384, True, False, 4, True),      # tanh (RAFT GRU q), fp32 out
    (500, 192, 256, True, False, 3, False),      # sigmoid, fp16 out
]


@pytest.mark.parametrize("M,N,K,has_bias,has_scale,act,out_f32", CASES)
def test_gemm_matches_fp32_reference(cuda_device, M, N, K, has_bias, has_scale, act, out_f32):
    g = torch.Generator(device="cpu").manual_seed(M * 7 + N * 3 + K)
    a = (torch.randn(M, K, generator=g) * 0.5).half().to(cuda_device)
    b = (torch.randn(N, K, generator=g) * K ** -0.5).half().to(cuda_device)
    bias = torch.randn(N, generator=g).to(cuda_device) if has_bias else None
    scale = (1 + 0.1 * torch.randn(N, generator=g)).to(cuda_device) if has_scale else None
    out = torch.ops.vfeat.gemm_f16(a, b, bias, scale, act, out_f32)
    torch.cuda.synchronize()
    ref = _ref(a, b, bias, scale, act)
    assert out.shape == (M, N)
    assert torch.isfinite(out.float()).all()
    tol = 2e-5 if out_f32 else 1.5e-3     # fp32 accumulation-order noise / fp16 output rounding
    err = rel_l2(out.float(), ref)
    assert err < tol, f"rel L2 {err:.3e}"
    mx = float((out.float() - ref).abs().max() / ref.abs().max())
    assert mx < (1e-4 if out_f32 else 2e-3), f"max err {mx:.3e}"


def test_gemm_output_with_row_pitch_and_no_overrun(cuda_device):
    """D written through a wider pitch: the columns beyond N and the rows beyond M must stay untouched."""
    from video_features_b200._lib import check, lib
    M, N, K, ld = 200, 96, 128, 160
    g = torch.Generator().manual_seed(5)
    a = (torch.randn(M, K, generator=g) * 0.5).half().to(cuda_device)
    b = (torch.randn(N, K, generator=g) * 0.1).half().to(cuda_device)
    out = torch.full((M + 8, ld), 7.0, device=cuda_device)
    check(lib().vf_gemm_f16(a.data_ptr(), K, b.data_ptr(), K, M, N, K, out.data_ptr(), ld, 1, None, None, 0,
                            torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    ref = a.float() @ b.float().t()
    assert rel_l2(out[:M, :N], ref) < 2e-5
    assert bool((out[:M, N:] == 7.0).all()) and bool((out[M:] == 7.0).all())


def test_gemm_partial_n_tile_is_race_free(cuda_device):
    """N = 320 leaves the second 256-wide tile mostly empty: the slices right of N are skipped by the epilogue, which
    once let a staging buffer be rewritten while its TMA store was still reading it (intermittent)."""
    g = torch.Generator().manual_seed(9)
    a = (torch.randn(3000, 64, generator=g) * 0.5).half().to(cuda_device)
    b = (torch.randn(320, 64, generator=g) * 0.2).half().to(cuda_device)
    ref = a.float() @ b.float().t()
    for _ in range(40):
        out = torch.ops.vfeat.gemm_f16(a, b, None, None, 0, True)
        assert rel_l2(out, ref) < 2e-5
    b2 = (torch.randn(208, 64, generator=g) * 0.2).half().to(cuda_device)
    ref2 = a.float() @ b2.float().t()
    for _ in range(40):
        out = torch.ops.vfeat.gemm_f16(a, b2, None, None, 0, False)
        assert rel_l2(out.float(), ref2) < 1.5e-3


@pytest.mark.parametrize("M,N,K,act", [(700, 256, 320, 2), (1000, 96, 192, 0), (300, 192, 136, 2), (5000, 128, 648, 2)])
def test_gemm_split_output_is_a_hi_lo_pair(cuda_device, M, N, K, act):
    """vf_gemm_f16_split: hi half bit-equal to the plain fp16 output, lo half == fp16(v - hi) of the fp32 output,
    columns between / right of the two halves untouched (N = 96 / 192: the hi store's 64-wide box overlaps the lo
    half's columns and must be clipped at N, not at the row pitch)."""
    from video_features_b200 import _lib
    from video_features_b200.ops import _stream
    g = torch.Generator(device="cpu").manual_seed(M + N)
    a = (torch.randn(M, K, generator=g) * 0.5).half().to(cuda_device)
    b = (torch.randn(N, K, generator=g) * 0.1).half().to(cuda_device)
    bias = torch.randn(N, generator=g).to(cuda_device)
    plain16 = torch.ops.vfeat.gemm_f16(a, b, bias, None, act, False)
    plain32 = torch.ops.vfeat.gemm_f16(a, b, bias, None, act, True)
    off, ld = N + 8, 2 * N + 24
    out = torch.full((M, ld), 7.0, device=cuda_device, dtype=torch.float16)
    with torch.cuda.device(cuda_device):
        _lib.check(_lib.lib().vf_gemm_f16_split(a.data_ptr(), K, b.data_ptr(), K, M, N, K, out.data_ptr(), ld, off,
                                                bias.data_ptr(), None, act, _stream()))
    torch.cuda.synchronize()
    assert torch.equal(out[:, :N], plain16)
    lo = (plain32 - plain16.float()).half()
    assert torch.equal(out[:, off:off + N], lo)
    assert bool((out[:, N:off] == 7.0).all()) and bool((out[:, off + N:] == 7.0).all())
    assert rel_l2(out[:, :N].float() + out[:, off:off + N].float(), plain32) < 1e-6


def test_gemm_rejects_bad_arguments(cuda_device):
    from video_features_b200._lib import VfError
    a = torch.zeros(16, 60, dtype=torch.float16, device=cuda_device)   # K not a multiple of 8
    b = torch.zeros(64, 60, dtype=torch.float16, device=cuda_device)
    with pytest.raises(VfError):
        torch.ops.vfeat.gemm_f16(a, b, None, None, 0, True)


@pytest.mark.parametrize("M,N,K", [(300, 256, 768), (6000, 768, 768), (6000, 768, 3072), (77, 96, 200), (250, 768, 768)])
def test_gemm_accumulate_adds_into_fp32_output(cuda_device, M, N, K):
    """out += a @ b.T + bias (fp32 global reductions from the epilogue): twice in a row, against the fp32 reference of the same op; rows /
    columns outside M x N of a larger buffer stay untouched."""
    g = torch.Generator(device="cpu").manual_seed(M + N + K)
    a = (torch.randn(M, K, generator=g) * 0.5).half().to(cuda_device)
    b = (torch.randn(N, K, generator=g) * K ** -0.5).half().to(cuda_device)
    bias = torch.randn(N, generator=g).to(cuda_device)
    x0 = (torch.randn(M, N, generator=g) * 3).to(cuda_device)
    x = x0.clone()
    torch.ops.vfeat.gemm_f16_accumulate(x, a, b, bias, 0)
    torch.ops.vfeat.gemm_f16_accumulate(x, a, b, bias, 0)
    ref = x0 + 2 * _ref(a, b, bias, None, 0)
    assert rel_l2(x, ref) < 2e-6, rel_l2(x, ref)            # fp32 accumulate of fp16 products: only summation order differs


def _raw_gemm(a_ptr, lda, b_ptr, ldb, M, N, K, out, ldd, out_f32, bias, scale, act):
    from video_features_b200 import _lib
    with torch.cuda.device(out.device):
        _lib.check(_lib.lib().vf_gemm_f16(a_ptr, lda, b_ptr, ldb, M, N, K, out.data_ptr(), ldd, int(out_f32),
                                          None if bias is None else bias.data_ptr(),
                                          None if scale is None else scale.data_ptr(), act,
                                          torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()


@pytest.mark.parametrize("act", [3, 4])
def test_gemm_sigmoid_tanh_against_float64(cuda_device, act):
    """The fast-math sigmoid / tanh of the epilogue (__expf, __fdividef) on pre-activations spread over [-20, 20]:
    absolute error <= 5e-6 against float64 (measured on an H100 80GB HBM3: 1.0e-7 sigmoid, 2.0e-7 tanh).  The
    pre-activation is the bias (A = 0), so it is exact."""
    M, N, K = 128, 4096, 64
    a = torch.zeros(M, K, dtype=torch.float16, device=cuda_device)
    b = torch.zeros(N, K, dtype=torch.float16, device=cuda_device)
    v = torch.linspace(-20, 20, N, dtype=torch.float32, device=cuda_device)
    out = torch.ops.vfeat.gemm_f16(a, b, v, None, act, True)
    ref = torch.sigmoid(v.double()) if act == 3 else torch.tanh(v.double())
    err = float((out.double() - ref).abs().max())
    print(f"act {act}: max abs error {err:.2e} on [-20, 20]")
    assert err <= 5e-6


@pytest.mark.parametrize("act", [1, 3, 4])
def test_gemm_activations_saturate_without_nan(cuda_device, act):
    """Pre-activations of +-100 and +-1000, where exp(|v|) overflows fp32: sigmoid -> exactly 0 / 1, tanh -> exactly
    -1 / +1, QuickGELU -> v or 0 (never NaN: the overflowed exp gives inf and the division 0)."""
    v = torch.tensor([-1000, -100, 100, 1000] * 8, dtype=torch.float32, device=cuda_device)
    N, K = v.numel(), 64
    a = torch.zeros(16, K, dtype=torch.float16, device=cuda_device)
    b = torch.zeros(N, K, dtype=torch.float16, device=cuda_device)
    out = torch.ops.vfeat.gemm_f16(a, b, v, None, act, True)
    assert bool(torch.isfinite(out).all())
    neg, pos = out[:, v < 0], out[:, v > 0]
    if act == 3:
        assert bool((neg == 0).all()) and bool((pos == 1).all())
    elif act == 4:
        assert bool((neg == -1).all()) and bool((pos == 1).all())
    else:
        assert bool((neg == 0).all()) and torch.equal(pos, v[v > 0].expand_as(pos))


@pytest.mark.parametrize("M,N,K,lda,ldb,a_col,b_col", [(300, 96, 136, 200, 512, 8, 64), (1000, 256, 768, 1536, 1024, 768, 128),
                                                      (77, 24, 64, 72, 80, 8, 16)])
def test_gemm_reads_column_windows_of_wider_operands(cuda_device, M, N, K, lda, ldb, a_col, b_col):
    """lda > K and ldb > K: A and B are column windows of wider matrices (row pitch in elements, window start a
    multiple of 8); the columns around the window must not leak in."""
    g = torch.Generator().manual_seed(M + lda)
    aw = (torch.randn(M, lda, generator=g) * 0.5).half().to(cuda_device)
    bw = (torch.randn(N, ldb, generator=g) * K ** -0.5).half().to(cuda_device)
    bias = torch.randn(N, generator=g).to(cuda_device)
    out = torch.full((M, N), 5.0, device=cuda_device)
    _raw_gemm(aw.data_ptr() + 2 * a_col, lda, bw.data_ptr() + 2 * b_col, ldb, M, N, K, out, N, True, bias, None, 0)
    ref = _ref(aw[:, a_col:a_col + K], bw[:, b_col:b_col + K], bias, None, 0)
    assert rel_l2(out, ref) < 2e-5
    assert float((out - ref).abs().max() / ref.abs().max()) < 1e-4


@pytest.mark.parametrize("act", [2, 3])
def test_gemm_accumulate_with_scale_and_activation(cuda_device, act):
    """D += act(a @ b.T * scale + bias): the activation applies to the GEMM term only, before the add."""
    from video_features_b200 import _lib
    M, N, K = 500, 192, 320
    g = torch.Generator().manual_seed(act)
    a = (torch.randn(M, K, generator=g) * 0.5).half().to(cuda_device)
    b = (torch.randn(N, K, generator=g) * K ** -0.5).half().to(cuda_device)
    bias = torch.randn(N, generator=g).to(cuda_device)
    scale = (1 + 0.1 * torch.randn(N, generator=g)).to(cuda_device)
    x0 = (torch.randn(M, N, generator=g) * 3).to(cuda_device)
    x = x0.clone()
    with torch.cuda.device(cuda_device):
        _lib.check(_lib.lib().vf_gemm_f16_accumulate(a.data_ptr(), K, b.data_ptr(), K, M, N, K, x.data_ptr(), N,
                                                     bias.data_ptr(), scale.data_ptr(), act,
                                                     torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    ref = x0.double() + _ref(a, b, bias, scale, act).double()
    assert rel_l2(x, ref) < 2e-6, rel_l2(x, ref)
    assert float((x.double() - ref).abs().max()) < 1e-5 * float(ref.abs().max())

"""The split-fp16 ("pair") arithmetic the conv engines rely on, emulated on the CPU: fp16 operands, exact products, fp32
accumulation -- what a wgmma f16 MMA computes.  Pins the claims of DESIGN.md §2:
  * x = hi + lo with hi = fp16(x), lo = fp16(x - hi) carries ~22 mantissa bits;
  * hi.W_hi + lo.W_hi + hi.W_lo reproduces the fp32 product to ~1e-6 (the dropped lo.W_lo term is ~2^-22);
  * max() over pairs may compare hi + lo in fp32 (exact) and re-split (the pool kernels)."""
import numpy as np
import torch


def _split(x: torch.Tensor):
    hi = x.half()
    lo = (x - hi.float()).half()
    return hi, lo


def _mm16(a16: torch.Tensor, b16: torch.Tensor) -> torch.Tensor:
    """fp16 operands, exact products, wide accumulation (float64 here stands in for the fp32 accumulator)."""
    return a16.double() @ b16.double().t()


def test_pair_carries_about_22_bits():
    g = torch.Generator().manual_seed(0)
    x = torch.randn(100000, generator=g) * 3
    hi, lo = _split(x)
    big = x.abs() > 0.25                               # for smaller |x| the lo half is a fp16 subnormal: absolute error <= 2^-25
    err_single = ((hi.float() - x).abs() / x.abs())[big].max().item()
    err_pair = ((hi.float() + lo.float() - x).abs() / x.abs())[big].max().item()
    assert 1e-4 < err_single < 5e-4                    # 2^-11
    assert err_pair < 2.0 ** -20                       # ~2^-22 (lo is itself rounded to 11 bits)
    assert (hi.float() + lo.float() - x).abs().max().item() < 2.0 ** -20 * x.abs().max().item()
    assert (hi.float() + lo.float() - x)[~big].abs().max().item() <= 2.0 ** -24
    assert torch.equal(hi.float() + lo.float(), (hi.float() + lo.float()).float())   # the sum is exact in fp32


def test_three_term_product_matches_fp32():
    g = torch.Generator().manual_seed(1)
    a = torch.randn(256, 768, generator=g)
    w = torch.randn(192, 768, generator=g) * 0.05
    exact = a.double() @ w.double().t()
    rel = lambda y: float((y - exact).norm() / exact.norm())
    ah, al = _split(a)
    wh, wl = _split(w)
    single = _mm16(ah, wh)
    w_split = single + _mm16(ah, wl)                                  # hi/lo weights, single-fp16 activations (I3D 3x3x3 convs)
    three = w_split + _mm16(al, wh)                                   # pair activations: [hi | lo] rows x duplicated filter
    four = three + _mm16(al, wl)
    assert 2e-4 < rel(single) < 6e-4
    assert 1e-4 < rel(w_split) < rel(single)                          # activation rounding remains
    assert rel(three) < 2e-6 and rel(four) < 2e-6                      # fp32-class
    assert abs(rel(three) - rel(four)) < 1e-6                          # the fourth term is below the accumulator's resolution
    # the K-concatenated form the GEMM actually runs: A = [hi | lo], W = [w | w] (duplicated columns), hi and lo weight passes
    A = torch.cat([ah, al], 1)
    Wd_hi, Wd_lo = torch.cat([wh, wh], 1), torch.cat([wl, wl], 1)
    run = _mm16(A, Wd_hi) + _mm16(A[:, :768], Wd_lo[:, :768])          # W_lo pass skipped on the lo-only K blocks
    assert torch.allclose(run, three, rtol=0, atol=1e-9)


def test_max_over_pairs_is_exact():
    g = torch.Generator().manual_seed(2)
    x = torch.relu(torch.randn(27, 4096, generator=g))
    hi, lo = _split(x)
    v = hi.float() + lo.float()                         # what the pool kernels compare
    m = v.max(0).values
    mh, ml = _split(m)
    idx = v.argmax(0)
    # the re-split pair represents exactly the value of the winning input pair (at an exact tie between two fp16
    # neighbours the (hi, lo) representation may differ, the value does not)
    assert torch.equal(mh.float() + ml.float(), m)
    assert torch.equal(m, hi[idx, torch.arange(4096)].float() + lo[idx, torch.arange(4096)].float())
    assert np.all(m.numpy() >= 0)

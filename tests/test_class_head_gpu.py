"""The classifier-head kernel (vf_head_forward, csrc/class_head.cu) against float64 on the same fp32 inputs: logits,
softmax and top-k at every (K, C) the extractors use, tie order, and the ABI's argument checks."""
import ctypes as C

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

# one sequential fp32 FMA chain per logit over K <= 2048 terms: rounding grows like eps * sqrt(K) ~ 3e-6 relative.
# Each stage is held against float64 of ITS fp32 inputs: the logits against float64 of (feats, W, b), the softmax
# against float64 softmax of the kernel's own fp32 logits.  End to end, a logit's absolute error d moves its
# probability by a factor exp(d), so the softmax against float64 of (feats, W, b) is held to BAR * (1 + max |logit|).
BAR = 1e-5
SHAPES = [(K, Cc) for K in (512, 1024, 2048) for Cc in (400, 1000)]


def _inputs(n, K, Cc, seed):
    g = torch.Generator().manual_seed(seed)
    feats = torch.rand(n, K, generator=g) * torch.rand(n, 1, generator=g) * 2     # post-ReLU-like, rows of varied scale
    w = torch.randn(Cc, K, generator=g) * (1.0 / K ** 0.5) * 3
    b = torch.randn(Cc, generator=g) * 0.1
    return feats, w, b


def _float64(feats, w, b):
    lg = feats.double() @ w.double().T + b.double()
    return lg, torch.softmax(lg, dim=1)


def _row_rel(a, ref):
    a, ref = a.double().cpu(), ref.double().cpu()
    return ((a - ref).norm(dim=1) / ref.norm(dim=1)).max().item()


@pytest.mark.parametrize("K,Cc", SHAPES)
@pytest.mark.parametrize("n", [1, 7, 64, 65, 257])
def test_head_against_float64(cuda_device, K, Cc, n):
    from video_features_b200.class_head import ClassHead
    feats, w, b = _inputs(n, K, Cc, seed=K * 7 + Cc + n)
    head = ClassHead(w, b, 0)
    k = 8
    logits, probs, idx, tl, tp = head.forward(feats.to(cuda_device), k)
    torch.cuda.synchronize()
    lg64, p64 = _float64(feats, w, b)
    rl, rp = _row_rel(logits, lg64), _row_rel(probs, torch.softmax(logits.cpu().double(), dim=1))
    re2e, big = _row_rel(probs, p64), float(lg64.abs().max())
    print(f"K={K} C={Cc} n={n}: logits rel-L2 {rl:.2e}, softmax rel-L2 {rp:.2e} (end to end {re2e:.2e}, "
          f"max |logit| {big:.1f})")
    assert rl <= BAR and rp <= BAR and re2e <= BAR * (1 + big), (rl, rp, re2e)
    idx, tl, tp = idx.cpu().long(), tl.cpu(), tp.cpu()
    # the top-k values are the kernel's own logits / probabilities at the returned indices
    assert torch.equal(tl, logits.cpu().gather(1, idx)) and torch.equal(tp, probs.cpu().gather(1, idx))
    # ordered by probability, descending, equal probabilities by the lower index; nothing outside beats the k-th
    assert bool((tp[:, :-1] >= tp[:, 1:]).all())
    pc = probs.cpu()
    kth = tp[:, -1:]
    outside = pc.scatter(1, idx, -1.0)
    assert bool((outside <= kth).all())
    # the same indices as float64 wherever neighbouring probabilities are separated by more than the bar
    s64, i64 = torch.sort(p64, dim=1, descending=True)
    for r in range(n):
        for j in range(k):
            gap_prev = s64[r, j - 1] - s64[r, j] if j > 0 else float("inf")
            gap_next = s64[r, j] - s64[r, j + 1]
            if min(gap_prev, gap_next) > BAR * float(s64[r, 0]):
                assert int(idx[r, j]) == int(i64[r, j]), (r, j)
    head.close()


def test_ties_go_to_the_lower_class_index(cuda_device):
    from video_features_b200.class_head import ClassHead
    feats, w, b = _inputs(5, 512, 400, seed=3)
    w[:] = 0
    b[:] = 0
    b[[250, 17, 399, 3]] = 2.0                   # four equal winners, then 396 equal losers
    head = ClassHead(w, b, 0)
    _, probs, idx, tl, tp = head.forward(feats.to(cuda_device), 8)
    assert idx.cpu().tolist() == [[3, 17, 250, 399, 0, 1, 2, 4]] * 5
    assert bool((tl.cpu()[:, :4] == 2.0).all()) and bool((tl.cpu()[:, 4:] == 0.0).all())
    assert bool((tp.cpu()[:, :4] == tp.cpu()[0, 0]).all())
    # duplicated weight rows: identical FMA chains give bit-equal logits, resolved by index
    feats, w, b = _inputs(3, 1024, 1000, seed=4)
    w[700], b[700] = 1.0 / 1024, 50.0              # far above every other logit
    w[20], b[20] = w[700], b[700]
    head2 = ClassHead(w, b, 0)
    logits, _, idx, _, _ = head2.forward(feats.to(cuda_device), 2)
    assert torch.equal(logits[:, 20], logits[:, 700])
    assert idx.cpu().tolist() == [[20, 700]] * 3
    head.close()
    head2.close()


def test_softmax_is_max_subtracted(cuda_device):
    """Logits of 1e3 would overflow expf without the max subtraction."""
    from video_features_b200.class_head import ClassHead
    feats, w, b = _inputs(4, 512, 400, seed=5)
    b += 1000.0
    head = ClassHead(w, b, 0)
    logits, probs, _, _, _ = head.forward(feats.to(cuda_device), 5)
    assert torch.isfinite(probs).all()
    assert _row_rel(probs, torch.softmax(logits.cpu().double(), dim=1)) <= BAR
    head.close()


def test_non_finite_rows_keep_indices_in_range_and_follow_torch_sort(cuda_device):
    """A NaN or infinite feature makes the row's softmax all NaN, as in torch; the top-k still returns valid classes, in
    torch.sort(descending=True, stable=True)'s order (NaN above every number, then by index)."""
    from video_features_b200.class_head import ClassHead
    for Cc, K in ((400, 1024), (1000, 2048), (5, 512)):
        feats, w, b = _inputs(4, K, Cc, seed=Cc + 9)
        feats[1, 7] = float("nan")
        feats[2, 3] = float("inf")
        feats[3, :] = float("nan")
        w[0] = 0.0                     # class 0's logit is 0 * inf = NaN in row 2 only
        head = ClassHead(w, b, 0)
        k = 5
        logits, probs, idx, tl, tp = head.forward(feats.to(cuda_device), k)
        idx, tl, tp, lg, pr = idx.cpu().long(), tl.cpu(), tp.cpu(), logits.cpu(), probs.cpu()
        assert bool(((idx >= 0) & (idx < Cc)).all()), idx
        assert all(len(set(r)) == k for r in idx.tolist())
        ref = torch.softmax(lg, dim=1)                     # torch on the kernel's own logits
        assert torch.equal(torch.isnan(pr), torch.isnan(ref))
        assert bool(torch.isnan(pr[1:]).all()) and not bool(torch.isnan(pr[0]).any())
        order = torch.sort(pr, dim=1, descending=True, stable=True)[1][:, :k]
        assert torch.equal(idx, order) and idx[1:].tolist() == [[0, 1, 2, 3, 4]] * 3
        assert torch.allclose(tl, lg.gather(1, idx), rtol=0, atol=0, equal_nan=True)
        assert torch.allclose(tp, pr.gather(1, idx), rtol=0, atol=0, equal_nan=True)
        head.close()


def test_abi_rejects_bad_arguments(cuda_device):
    from video_features_b200._lib import VfError, check, lib
    L = lib()
    w = np.zeros((4, 8), np.float32)
    b = np.zeros(4, np.float32)
    h = C.c_void_p()
    for nc, nf in ((0, 8), (4, 0), (-1, 8)):
        assert L.vf_head_create(C.byref(h), w.ctypes.data, b.ctypes.data, nc, nf, 0) == 1
        assert b"head_create" in L.vf_last_error()
    assert L.vf_head_create(C.byref(h), None, b.ctypes.data, 4, 8, 0) == 1
    check(L.vf_head_create(C.byref(h), w.ctypes.data, b.ctypes.data, 4, 8, 0))
    nc, nf = C.c_int(), C.c_int()
    check(L.vf_head_info(h, C.byref(nc), C.byref(nf)))
    assert (nc.value, nf.value) == (4, 8)
    x = torch.zeros(3, 8, device=cuda_device)
    o = [torch.empty(3, 4, device=cuda_device) for _ in range(2)]
    t = [torch.empty(3, 8, device=cuda_device, dtype=torch.int32)] + [torch.empty(3, 8, device=cuda_device)] * 2

    def fwd(n=3, K=8, k=2, feats=x.data_ptr()):
        return L.vf_head_forward(h, feats, n, K, o[0].data_ptr(), o[1].data_ptr(), k, t[0].data_ptr(), t[1].data_ptr(),
                                 t[2].data_ptr(), None)
    check(fwd())
    for kw, text in ((dict(n=-1), b"rows"), (dict(n=16 * 65535 + 1), b"rows"), (dict(K=7), b"features"),
                     (dict(k=0), b"k = 0"), (dict(k=9), b"k = 9"), (dict(k=5), b"k = 5"), (dict(feats=None), b"null")):
        assert fwd(**kw) == 1, kw
        assert text in L.vf_last_error(), (kw, L.vf_last_error())
    assert fwd(n=0) == 0                             # nothing to do
    with pytest.raises(VfError):
        check(fwd(k=9))
    torch.cuda.synchronize()
    check(L.vf_head_destroy(h))

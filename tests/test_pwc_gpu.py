"""PWC-Net engine (seeded stand-in weights) against the float64 oracle: per-stage diagnostics, end-to-end flow at three
sizes, its input entries and call splits, and every uploaded conv read back against a CPU restatement.

The engine carries every GEMM operand as a split-fp16 pair (RAFT's scheme), so no operand class is declared rounded:
the float64 oracle is the reference computation itself."""
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

MAX_H, MAX_W = 436, 1024


def _rel(y, ref):
    return float((y.double() - ref.double()).norm() / ref.double().norm())


def _maxrel(y, ref):
    return float((y.double() - ref.double()).abs().max() / ref.double().abs().max())


@pytest.fixture(scope="module")
def sd():
    from oracle import pwc_net
    return pwc_net.stand_in_state_dict()


@pytest.fixture(scope="module")
def pwc(cuda_device, sd):
    from video_features_b200.pwc_engine import PWCEngine
    eng = PWCEngine(sd, 0, max_frames=5, max_h=MAX_H, max_w=MAX_W)
    yield eng
    eng.close()


def _frames(n, h, w, seed, shift):
    from oracle import raft_net
    return raft_net.synthetic_frames(n, h, w, seed=seed, shift=shift)


def _assert_masks_clear(st, rel=1e-4):
    """A warp mask value near the 0.999 threshold could flip under rounding, and a flipped pixel zeroes a whole feature
    vector: the comparisons below hold only for inputs without one.  The in-bounds weight sum moves by at most the error
    of the sample position, i.e. of the displacement dblBackward * upflow; at the 1e-4 relative flow bar of the stage
    test that is 1e-4 x the level's largest displacement.  (A fixed 1e-4 would reject every input at level 5: the
    stand-in's level-6 features are leaky(bias), constant over the image, so its level-5 displacements are ~0.01 px
    and the same border pixel sits 3e-5 from the threshold whatever the frames.)

    The threshold itself, and warps large enough to mask interior pixels, are tested in test_flow_motion_gpu.py, where a
    uniform displacement makes the raw mask a known function of its fractional part."""
    from oracle import pwc_net
    for l in (5, 4, 3, 2):
        tol = rel * float((st[f"upflow{l}"] * pwc_net.DBL_BACKWARD[l]).abs().max())
        near = int(((st[f"maskraw{l}"] - 0.999).abs() < tol).sum())
        assert near == 0, f"level {l}: {near} warp-mask values within {tol:.1e} of 0.999; choose another input"


def test_pwc_stages_vs_float64(pwc, sd, cuda_device):
    from oracle import pwc_net
    from video_features_b200 import pwc_engine as E
    x = _frames(3, 128, 160, seed=3, shift=(1.3, -0.7)).to(cuda_device)
    y = pwc.flow(x)
    sd64 = {k: v.to(cuda_device, torch.float64) for k, v in sd.items()}
    st = {}
    ref = pwc_net.forward(sd64, x[:-1].double(), x[1:].double(), torch.float64, stages=st)
    _assert_masks_clear(st)
    with torch.no_grad():
        pre = pwc_net.preprocess(x.double())
        feats = pwc_net.extractor(sd64, pre)
    for l in range(1, 6):
        f = pwc.debug_read(E.FEATURES, l)
        r = _rel(f, feats[l - 1])
        print(f"level {l} features rel-L2 {r:.2e}")
        assert r < 1e-5, (l, r)
    # Declared rounding: the checkpoint's level-6 extractor biases are <= 2.3e-7 and its weights <= 3e-14 (the stand-in
    # keeps that scale), so the level-6 features lie in fp16's subnormal range, where a split pair resolves 2^-24
    # absolute.  They feed only the level-6 cost volume (~1e-14), which the level-6 decoder multiplies by weights
    # <= 2e-16: the flow does not see them (asserted end to end below).
    err6 = float((pwc.debug_read(E.FEATURES, 6).double() - feats[5]).abs().max())
    print(f"level 6 features max-abs {err6:.2e} (max {float(feats[5].abs().max()):.2e})")
    assert err6 <= 2.0 ** -24, err6
    for l in range(6, 1, -1):
        f = pwc.debug_read(E.FEATURES, l).double()
        vol = pwc.debug_read(E.VOLUME, l)
        if l == 6:
            ref_vol = pwc_net._leaky(pwc_net.correlation(f[:-1], f[1:]))
        else:
            # the oracle fed the engine's OWN upsampled flow: upstream rounding cannot flip a 0.999 mask decision here
            upflow = pwc.debug_read(E.UPFLOW, l).double()
            warped, mask, raw = pwc_net.backward_warp(f[1:], upflow * pwc_net.DBL_BACKWARD[l])
            ref_vol = pwc_net._leaky(pwc_net.correlation(f[:-1], warped))
            clear = (raw - 0.999).abs() >= 1e-4
            emask = pwc.debug_read(E.MASK, l).double()
            assert torch.equal(emask[clear], mask[clear]), l
            # the transposed convs, fed the engine's coarser flow
            up = pwc_net._deconv(sd64, f"module{pwc_net.LEVEL_NAMES[l]}.moduleUpflow", pwc.debug_read(E.FLOW, l + 1).double())
            r = _rel(upflow, up)
            print(f"level {l} upflow rel-L2 {r:.2e}")
            assert r < 1e-5, (l, r)
            r = _rel(pwc.debug_read(E.UPFEAT, l), st[f"upfeat{l}"])
            print(f"level {l} upfeat vs oracle rel-L2 {r:.2e}")
            assert r < 1e-4, (l, r)
        if l == 6:                       # ~1e-14: below the split pair's 2^-24 resolution (see above)
            assert float((vol.double() - ref_vol).abs().max()) <= 2.0 ** -24
        else:
            # an fp32 sum of C products with cancellation (1.7e-5 measured at level 5); features with a lost lo half
            # (2^-11 relative) would put it near 1e-3
            r = _rel(vol, ref_vol)
            print(f"level {l} cost volume rel-L2 {r:.2e}")
            assert r < 1e-4, (l, r)
        r = _rel(pwc.debug_read(E.FLOW, l), st[f"flow{l}"])
        print(f"level {l} decoder flow vs oracle rel-L2 {r:.2e}")
        assert r < 1e-4, (l, r)
    r = _rel(pwc.debug_read(E.REFINE), st["refine"])
    print(f"refiner rel-L2 {r:.2e}")
    assert r < 1e-4
    assert _rel(y, ref) < 1e-4 and _maxrel(y, ref) < 1e-4


@pytest.mark.parametrize("h,w,n,seed", [(128, 160, 3, 5), (256, 341, 3, 5), (436, 1024, 2, 6)])
def test_pwc_flow_vs_float64(pwc, sd, cuda_device, h, w, n, seed):
    from oracle import pwc_net
    x = _frames(n, h, w, seed=seed, shift=(2.2, 1.1)).to(cuda_device)
    sd64 = {k: v.to(cuda_device, torch.float64) for k, v in sd.items()}
    st = {}
    ref = pwc_net.forward(sd64, x[:-1].double(), x[1:].double(), torch.float64, stages=st)
    _assert_masks_clear(st)
    y = pwc.flow(x)
    assert y.shape == (n - 1, 2, h, w) and y.dtype == torch.float32
    rel, mx = _rel(y, ref), _maxrel(y, ref)
    print(f"{h}x{w}: rel-L2 {rel:.2e}, max-abs / max {mx:.2e}, max |flow| {float(ref.abs().max()):.2f}")
    assert rel <= 1e-3 and mx <= 1e-3, (rel, mx)


def test_pwc_u8_entry_and_call_splits_are_bit_identical(pwc, cuda_device):
    x = _frames(5, 96, 200, seed=8, shift=(0.9, 0.4)).to(cuda_device)
    y = pwc.flow(x)
    u8 = x.permute(0, 2, 3, 1).contiguous().to(torch.uint8)
    assert torch.equal(pwc.flow(u8), y)
    parts = torch.cat([pwc.flow(x[0:3]), pwc.flow(x[2:4]), pwc.flow(x[3:5])])
    assert torch.equal(parts, y)


def test_pwc_refuses_bad_calls(pwc, cuda_device):
    from video_features_b200._lib import VfError
    x = torch.zeros((2, 3, 64, 1100), device=cuda_device)
    with pytest.raises(VfError, match="outside the workspace"):
        pwc.flow(x)
    with pytest.raises(VfError, match="frames outside"):
        pwc.flow(torch.zeros((6, 3, 64, 64), device=cuda_device))


# ---- conv read-back: the uploaded layout restated on the CPU
FEAT_C = [3, 16, 32, 64, 96, 128, 196]
NAMES = {1: "One", 2: "Two", 3: "Thr", 4: "Fou", 5: "Fiv", 6: "Six"}


def _r8(c):
    return (c + 7) // 8 * 8


def _layout(l):
    """decoder row of level l: slices c5, c4, c3, c2, c1, vol, f1, upflow, upfeat as (width, real channels, offset)"""
    w = [32, 64, 96, 128, 128, 88, _r8(FEAT_C[l]), 8, 8]
    r = [32, 64, 96, 128, 128, 81, FEAT_C[l], 2, 2]
    n = 9 if l < 6 else 6
    off, out = 0, []
    for j in range(n):
        out.append((w[j], r[j], off))
        off += 2 * w[j]
    return out, off


def _suffix(l, s0):
    """(hi, lo) columns, relative to the start of slice s0, of the reference channels of the suffix from s0"""
    sl, _ = _layout(l)
    base = sl[s0][2]
    return [(o - base + c, o - base + c + wd) for (wd, r, o) in sl[s0:] for c in range(r)]


def _conv3(sd, name, n_out, kpt, cols, dil=1):
    w = sd[name + ".weight"].double().numpy()
    co = w.shape[0]
    W = np.zeros((n_out, 9, kpt))
    for c, (hi, lo) in enumerate(cols):
        for t in range(9):
            W[:co, t, hi] = W[:co, t, lo] = w[:, c, t // 3, t % 3]
    shifts = [(0, (t // 3 - 1) * dil, (t % 3 - 1) * dil) for t in range(9)]
    b = np.zeros(n_out)
    b[:co] = sd[name + ".bias"].double().numpy()
    hi_cols = {h for h, _ in cols}
    return W, b, shifts, hi_cols


def _stride2(sd, name, n_out, ci8):
    w = sd[name + ".weight"].double().numpy()
    co, ci = w.shape[:2]
    pitch = 8 * ci8
    W = np.zeros((n_out, 2, 2 * pitch))
    hi_cols = set()
    for kh in range(3):
        for kw in range(3):
            a, ph, bq, pw = (kh + 1) // 2, (kh + 1) % 2, (kw + 1) // 2, (kw + 1) % 2
            for c in range(ci):
                k = bq * pitch + (ph * 2 + pw) * 2 * ci8 + c
                W[:co, a, k] = W[:co, a, k + ci8] = w[:, c, kh, kw]
                hi_cols.add(k)
    b = np.zeros(n_out)
    b[:co] = sd[name + ".bias"].double().numpy()
    return W, b, [(0, -1, -1), (0, 0, -1)], hi_cols


def _deconv(sd, name, kpt, cols):
    w = sd[name + ".weight"].double().numpy()          # [ci][2][4][4]
    W = np.zeros((8, 9, kpt))
    for c, (hi, lo) in enumerate(cols):
        for t in range(9):
            di, dj = t // 3 - 1, t % 3 - 1
            for py in range(2):
                for px in range(2):
                    ky, kx = py + 1 - 2 * di, px + 1 - 2 * dj
                    if 0 <= ky <= 3 and 0 <= kx <= 3:
                        for oc in range(2):
                            W[(py * 2 + px) * 2 + oc, t, hi] = W[(py * 2 + px) * 2 + oc, t, lo] = w[c, oc, ky, kx]
    b = np.array([float(sd[name + ".bias"][n % 2]) for n in range(8)])
    return W, b, [(0, t // 3 - 1, t % 3 - 1) for t in range(9)], {h for h, _ in cols}


def _expected_convs(sd):
    out = []
    for l in range(1, 7):
        p = f"moduleExtractor.module{NAMES[l]}."
        ci8, co8 = (8 if l == 1 else _r8(FEAT_C[l - 1])), _r8(FEAT_C[l])
        same = [(c, co8 + c) for c in range(FEAT_C[l])]
        out += [_stride2(sd, p + "0", co8, ci8), _conv3(sd, p + "2", co8, 2 * co8, same), _conv3(sd, p + "4", co8, 2 * co8, same)]
    for l in range(6, 1, -1):
        p = f"module{NAMES[l]}."
        sl, total = _layout(l)
        if l < 6:
            _, total_c = _layout(l + 1)
            out.append(_deconv(sd, p + "moduleUpflow", 16, [(0, 8), (1, 9)]))
            out.append(_deconv(sd, p + "moduleUpfeat", total_c, _suffix(l + 1, 0)))
        for k in range(6):
            s0 = 5 - k
            n_out = sl[4 - k][0] if k < 5 else 8
            out.append(_conv3(sd, p + f"module{NAMES[k + 1]}.0", n_out, total - sl[s0][2], _suffix(l, s0)))
    _, total2 = _layout(2)
    ch = [0, 128, 128, 128, 96, 64, 32, 2]
    for k, d in enumerate((1, 2, 4, 8, 16, 1, 1)):
        name = f"moduleRefiner.moduleMain.{2 * k}"
        if k == 0:
            out.append(_conv3(sd, name, 128, total2, _suffix(2, 0)))
        else:
            out.append(_conv3(sd, name, _r8(ch[k + 1]), 2 * ch[k], [(c, ch[k] + c) for c in range(ch[k])], d))
    return out


def _split(W, b):
    """per output row: scale by 2^e (largest |w| in [2^14, 2^15), e <= 126), then W_hi | W_lo; epilogue scale 2^-e"""
    n = W.shape[0]
    Wf = W.reshape(n, -1)
    hi = np.zeros(Wf.shape, np.float16)
    lo = np.zeros(Wf.shape, np.float16)
    scale = np.ones(n, np.float32)
    for o in range(n):
        row = Wf[o].astype(np.float32)
        m = float(np.abs(row).max())
        e = 0
        if m > 0:
            e = min(15 - math.frexp(m)[1], 126)
        wf = (row.astype(np.float64) * 2.0 ** e).astype(np.float32)
        h = wf.astype(np.float16)
        l_ = (wf - h.astype(np.float32)).astype(np.float16)
        nz = row != 0
        hi[o, nz], lo[o, nz] = h[nz], l_[nz]
        scale[o] = np.float32(2.0 ** -e)
    return np.concatenate([hi, lo], 1), scale, b.astype(np.float32)


def test_pwc_uploaded_convs_match_cpu_restatement(pwc, sd):
    expected = _expected_convs(sd)
    assert len(expected) == 63
    for i, (W, b, shifts, hi_cols) in enumerate(expected):
        got = pwc.conv(i)
        n_out, ntaps, kpt = W.shape
        assert (got["n_out"], got["ntaps"], got["k_per_tap"], got["nsplit"]) == (n_out, ntaps, kpt, 2), i
        assert got["shifts"] == shifts, i
        blocks = (kpt + 63) // 64
        mask = 0
        for kk in range(blocks):
            if not any(j in hi_cols for j in range(kk * 64, min((kk + 1) * 64, kpt))):
                mask |= 1 << kk
        assert got["lo_mask"] == mask, (i, hex(got["lo_mask"]), hex(mask))
        w, scale, bias = _split(W, b)
        assert np.array_equal(got["w"].cpu().numpy().view(np.int16), w.view(np.int16)), i
        assert np.array_equal(got["scale"].cpu().numpy(), scale), i
        assert np.array_equal(got["bias"].cpu().numpy(), bias), i
    # the checkpoint's near-zero level-6 weights keep their bits: the stand-in draws them at the trained scale
    ext6 = pwc.conv(15)
    assert float(ext6["scale"][:196].max()) < 2.0 ** -100

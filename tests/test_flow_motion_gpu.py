"""PWCEngine and RAFTEngine under real motion, against the float64 oracles.

The seeded stand-ins warp PWC's second frame by ~1 px and move RAFT's lookup centre by under half a cell, so the other
GPU tests only ever run warp_kernel, corr_lookup_kernel, coords_update_kernel and upsample_flow_kernel in their own
pixel's neighbourhood.  The state dicts of tests/flow_steering.py set the flow through the weights (a zero-weight conv
returns its bias): uniform PWC warps of 3 .. 20 px at each level, fractional, negative, whole-pixel and larger than the
map; warps whose border raw mask sits 5e-4 either side of the 0.999 threshold; spatially varying warps of 8 px; RAFT
steps that carry the lookup centre 3 .. 45 cells away and off the map; a 10x flow head; a saturated upsampling softmax.
test_flow_steering_cpu.py asserts in the oracle that each regime is reached and records what it separates.

Exact assertions: the steered convs as uploaded (an all-zero weight row: scale 1, no lo half), the uniform upflow and
low-res flow, every warp mask of a uniform warp, the border masks either side of the threshold.  Bars
(split_engine_bars.PWC_MOTION_BARS / RAFT_MOTION_BARS) carry their measured values; test_zz_report_measured prints
them (pytest -s)."""
import numpy as np
import pytest
import torch

import flow_steering as S
import split_engine_bars as bars
import test_i3d_raft_float64_gpu as T
import test_pwc_gpu as P
from oracle import pwc_net
from oracle import raft_net as R

pytestmark = pytest.mark.gpu

MEASURED = {}


def _note(key, *vals):
    old = MEASURED.get(key, (0.0,) * len(vals))
    MEASURED[key] = tuple(max(a, b) for a, b in zip(old, vals))


def _rel(y, ref):
    return float((y.double() - ref.double()).norm() / ref.double().norm())


def _maxrel(y, ref):
    return float((y.double() - ref.double()).abs().max() / ref.double().abs().max())


# ---------------------------------------------------------------------------------------------------------- PWC

@pytest.fixture(scope="module")
def pwc_sd():
    return pwc_net.stand_in_state_dict()


def _pwc_engine(sd, max_frames=3, max_h=256, max_w=384):
    from video_features_b200.pwc_engine import PWCEngine
    return PWCEngine(sd, 0, max_frames=max_frames, max_h=max_h, max_w=max_w)


def _pwc_frames(size, dev, n=3):
    return R.synthetic_frames(n, *size, **S.PWC_FRAMES[size]).to(dev)


def _upflow_conv(level):
    """Index of level `level`'s moduleUpflow in vf_pwc_conv's order: 18 extractor convs, 6 of level 6, then 8 per level."""
    return 24 + 8 * (5 - level)


def _assert_steered_conv(eng, sd, level):
    """The steered transposed conv as uploaded, bit for bit (test_pwc_gpu.py's restatement): every weight row is zero,
    which takes the m == 0 branch of the per-row power-of-two scaling (scale 1, hi = lo = 0) that no stand-in conv
    takes."""
    W, b, shifts, hi_cols = P._deconv(sd, f"module{pwc_net.LEVEL_NAMES[level]}.moduleUpflow", 16, [(0, 8), (1, 9)])
    got = eng.conv(_upflow_conv(level))
    w, scale, bias = P._split(W, b)
    assert (got["n_out"], got["ntaps"], got["k_per_tap"], got["nsplit"]) == (8, 9, 16, 2) and got["shifts"] == shifts
    assert not w.any() and np.array_equal(got["w"].cpu().numpy().view(np.int16), w.view(np.int16))
    assert np.array_equal(got["scale"].cpu().numpy(), np.ones(8, np.float32))
    assert np.array_equal(got["bias"].cpu().numpy(), bias)


def _pwc_check(name, eng, sd, x, uniform=None, must_reach_final=False):
    """Every decoder level of the engine's last flow(x) against float64.  Mask and cost volume are checked against the
    oracle's warp of the engine's OWN features and upsampled flow (upstream rounding cannot flip a mask there); the
    decoder flows and the final flow against the oracle's forward, down to the first level where the oracle has a raw
    mask value within reach of the threshold (_assert_masks_clear's criterion): below a flipped pixel the two
    computations differ by a whole feature vector.  uniform = (level, (dx, dy)): that level's upflow and mask are exact."""
    from video_features_b200 import pwc_engine as E
    dev = x.device
    y = eng.flow(x)
    assert torch.isfinite(y).all()
    sd64 = {k: v.to(dev, torch.float64) for k, v in sd.items()}
    st = {}
    with torch.no_grad():
        ref = pwc_net.forward(sd64, x[:-1].double(), x[1:].double(), torch.float64, stages=st)
    failures, comparable = [], True
    for l in (5, 4, 3, 2):
        dbl = pwc_net.DBL_BACKWARD[l]
        f = eng.debug_read(E.FEATURES, l).double()
        upflow = eng.debug_read(E.UPFLOW, l).double()
        emask = eng.debug_read(E.MASK, l).double()
        warped, mask, raw = pwc_net.backward_warp(f[1:], upflow * dbl)
        if uniform and uniform[0] == l:
            want = torch.tensor(uniform[1], dtype=torch.float64, device=dev).view(1, 2, 1, 1) / dbl
            assert torch.equal(upflow, want.expand_as(upflow)), (name, l)
            assert torch.equal(emask, mask) and torch.equal(emask, st[f"mask{l}"]), (name, l)
        else:
            clear = (raw - 0.999).abs() >= 1e-4
            # (the stand-in's level-5 border pixels sit 3e-5 from the threshold whatever the frames: 2 of 24 at 128x160)
            assert float(clear.double().mean()) > (0.99 if raw.numel() >= 1000 else 0.9), (name, l)
            assert torch.equal(emask[clear], mask[clear]), (name, l)
            reach = 1e-4 * float((st[f"upflow{l}"] * dbl).abs().max())
            comparable = comparable and int(((st[f"maskraw{l}"] - 0.999).abs() < reach).sum()) == 0
        vol, ref_vol = eng.debug_read(E.VOLUME, l), pwc_net._leaky(pwc_net.correlation(f[:-1], warped))
        if not ref_vol.any():                # every sample off the map: the volume is zero, not merely small
            assert not vol.any(), (name, l)
            r = 0.0
        else:
            r = _rel(vol, ref_vol)
        _note("pwc volume", r)
        if r >= bars.PWC_MOTION_BARS["volume"]:
            failures.append((name, l, "volume", r))
        line = f"{name} level {l}: masked {int((emask == 0).sum())}/{emask.numel()}, volume {r:.2e}"
        if comparable:
            r = _rel(eng.debug_read(E.FLOW, l), st[f"flow{l}"])
            _note("pwc decoder flow", r)
            line += f", flow vs oracle {r:.2e}"
            if r >= bars.PWC_MOTION_BARS["flow"]:
                failures.append((name, l, "flow", r))
        print(line)
    if comparable:
        e = (_rel(y, ref), _maxrel(y, ref))
        _note("pwc final flow", *e)
        print(f"{name} final flow: rel-L2 {e[0]:.2e}, max-abs/max {e[1]:.2e}, max |flow| {float(ref.abs().max()):.1f} px")
        if not bars.within(e, bars.PWC_MOTION_BARS["final"]):
            failures.append((name, "final", e))
    assert comparable or not must_reach_final, f"{name}: the oracle has a mask value at the threshold; choose another input"
    assert not failures, failures
    return st


@pytest.mark.parametrize("level", (5, 4, 3, 2))
def test_pwc_uniform_warps(cuda_device, pwc_sd, level):
    """One engine per displacement, 128x160 and 200x333 (working size 256x384)."""
    for d in S.PWC_UNIFORM[level]:
        sd, disp = S.pwc_uniform_warp(pwc_sd, level, *d)
        eng = _pwc_engine(sd)
        _assert_steered_conv(eng, sd, level)
        for size in ((128, 160), (200, 333)):
            st = _pwc_check(f"pwc uniform {disp[0]:+.2f},{disp[1]:+.2f} {size[0]}x{size[1]}", eng, sd,
                            _pwc_frames(size, cuda_device), (level, disp), must_reach_final=level == 2)
            mask = st[f"mask{level}"]
            assert 0 < int((mask == 0).sum()), "the warp masks nothing"
            if disp == (5.0, -5.0):          # whole pixels: mask 1 exactly where the source pixel is on the map
                h, w = mask.shape[2:]
                want = torch.zeros_like(mask)
                want[..., 5:, :max(w - 5, 0)] = 1
                assert torch.equal(eng.debug_read(6, level).double(), want)          # pwc_engine.MASK
        eng.close()


def test_pwc_mask_threshold(cuda_device, pwc_sd):
    """Level-2 warps of (+-f, 0) and (0, +-f): the border column / row has raw mask 1 - f = 0.9995 (kept) or 0.9985
    (masked), every other pixel 1.  The fp32 coordinate x + f (x <= 47) is 2e-6 from the float64 one, 250 times closer
    than the threshold: a mask compared with 0.99 or 0.9999, or a weight off by 1e-4, fails here."""
    from video_features_b200 import pwc_engine as E
    x = _pwc_frames((128, 160), cuda_device)
    for (dx, dy), border in S.PWC_THRESHOLD.items():
        sd, disp = S.pwc_uniform_warp(pwc_sd, 2, dx, dy)
        eng = _pwc_engine(sd, max_h=128, max_w=160)
        _pwc_check(f"pwc threshold {disp[0]:+.4f},{disp[1]:+.4f}", eng, sd, x, (2, disp), must_reach_final=True)
        mask = eng.debug_read(E.MASK, 2)
        want = torch.ones_like(mask)
        if dx:
            want[..., :, -1] = border
        else:
            want[..., 0, :] = border
        assert torch.equal(mask, want), (dx, dy)
        eng.close()


@pytest.mark.parametrize("name", list(S.PWC_VARYING))
def test_pwc_varying_warps(cuda_device, pwc_sd, name):
    sd = S.pwc_varying_warp(pwc_sd, S.PWC_VARYING[name])
    eng = _pwc_engine(sd, max_h=128, max_w=160)
    st = _pwc_check(f"pwc varying {name}", eng, sd, _pwc_frames((128, 160), cuda_device), must_reach_final=True)
    level = max(S.PWC_VARYING[name])
    r = S.warp_regime(st[f"maskraw{level}"].cpu(), (st[f"upflow{level}"] * pwc_net.DBL_BACKWARD[level]).cpu())
    print(name, r)
    assert r["all taps outside"] > 0 and r["masked interior"] > 0
    eng.close()


def test_pwc_smallest_map(cuda_device, pwc_sd):
    """40x50 frames: working size 64x64, level 6 is 1x1 and level 5 2x2."""
    x = _pwc_frames((40, 50), cuda_device)
    eng = _pwc_engine(pwc_sd, max_h=64, max_w=64)
    _pwc_check("pwc 40x50 stand-in", eng, pwc_sd, x, must_reach_final=True)
    eng.close()
    sd, disp = S.pwc_uniform_warp(pwc_sd, 3, 3.25, -2.5)
    eng = _pwc_engine(sd, max_h=64, max_w=64)
    _pwc_check("pwc 40x50 uniform level 3", eng, sd, x, (3, disp))
    eng.close()


def test_pwc_u8_entry_and_call_splits_under_a_masking_warp(cuda_device, pwc_sd):
    sd, _ = S.pwc_uniform_warp(pwc_sd, 2, -7.75, 3.25)
    eng = _pwc_engine(sd, max_frames=5)
    x = R.synthetic_frames(5, 96, 200, seed=8, shift=(0.9, 0.4)).to(cuda_device)
    y = eng.flow(x)
    assert torch.equal(eng.flow(x.permute(0, 2, 3, 1).contiguous().to(torch.uint8)), y)
    assert torch.equal(torch.cat([eng.flow(x[0:3]), eng.flow(x[2:4]), eng.flow(x[3:5])]), y)
    eng.close()


# --------------------------------------------------------------------------------------------------------- RAFT

@pytest.fixture(scope="module")
def raft_sd():
    from helpers import stand_in_state_dict
    return stand_in_state_dict("raft-sintel.pth")


def _raft_engine(sd):
    from video_features_b200.raft_engine import RAFTEngine
    return RAFTEngine(sd, 0, max_frames=2, max_h=200, max_w=200)


def _raft_check(key, name, eng, sd, size, iters, dev):
    bar = bars.RAFT_MOTION_BARS[key]
    xp = R.pad(R.synthetic_frames(2, *size, seed=size[0]).to(dev))
    ref = T._raft_ref(sd, xp, iters, declared_rounding=True)
    errs = T._raft_errors(name, eng, xp, iters, ref, record=False, bar=bar)
    for s, e in errs.items():
        _note(f"raft {key} {s}", *e)
    return errs, ref, [(name, s, e) for s, e in errs.items() if not bars.within(e, bar[s])]


def test_raft_uniform_steps(cuda_device, raft_sd):
    """Every iteration adds the flow head's bias (dyadic: the fp32 sums are exact), so the low-res flow is iters x
    (du, dv) exactly and the last lookup is centred (iters - 1) x (du, dv) from its query: up to 45 cells, off the
    map, whole level-0 windows off it.  The next iteration's GRU state covers the split pair written to hx / qx."""
    failures = []
    for (du, dv), iters in S.RAFT_UNIFORM:
        sd = S.raft_uniform_step(raft_sd, du, dv)
        eng = _raft_engine(sd)
        for size in ((128, 160), (200, 200)):
            errs, (up, st), f = _raft_check("uniform", f"raft uniform {du:+g},{dv:+g} x{iters} {size[0]}x{size[1]}",
                                            eng, sd, size, iters, cuda_device)
            failures += f
            low = eng.debug_read(3)
            want = torch.tensor([du, dv], device=cuda_device).view(1, 2, 1, 1) * iters
            assert torch.equal(low, want.expand_as(low)), float((low - want).abs().max())
            assert torch.isfinite(eng.debug_read(2)).all()
        eng.close()
    assert not failures, failures


def test_raft_varying_flow(cuda_device, raft_sd):
    sd = S.raft_varying_flow(raft_sd, S.RAFT_VARYING_GAIN)
    eng = _raft_engine(sd)
    failures = []
    for iters in (3, 20):
        for size in ((128, 160), (200, 200)):
            errs, (up, st), f = _raft_check(f"varying {iters}", f"raft varying it{iters} {size[0]}x{size[1]}", eng, sd,
                                            size, iters, cuda_device)
            failures += f
            print(f"    low-res flow max {float(st['lowres'][-1].abs().max()):.2f} cells")
    eng.close()
    assert not failures, failures


def test_raft_sharp_upsampling_mask(cuda_device, raft_sd):
    """Mask logits of +-60: most of the 9-way softmaxes are saturated."""
    sd = S.raft_sharp_mask(raft_sd, S.RAFT_SHARP_GAIN)
    eng = _raft_engine(sd)
    failures = []
    for size in ((128, 160), (200, 200)):
        errs, (up, st), f = _raft_check("sharp", f"raft sharp it3 {size[0]}x{size[1]}", eng, sd, size, 3, cuda_device)
        failures += f
        assert float(st["mask"].abs().max()) > 30
        assert torch.isfinite(eng.flow(R.pad(R.synthetic_frames(2, *size, seed=size[0]).to(cuda_device)), iters=3)).all()
    eng.close()
    assert not failures, failures


def test_zz_report_measured(cuda_device):
    """Prints the worst value per bar over the tests above (run in the same session)."""
    for k, v in sorted(MEASURED.items()):
        print(f"measured worst {k}: " + " / ".join(f"{x:.2e}" for x in v))

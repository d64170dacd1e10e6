"""The premise of test_flow_motion_gpu.py, in the float64 oracles alone (no GPU).

1. Regimes: the steered state dicts of flow_steering.py reach what they are named for -- PWC warps of 8 px and more
   at level 2, samples with all four taps off the map, masked interior pixels; RAFT lookup centres 3 and more cells from
   their query, off the map, with whole windows off it; saturated upsampling softmaxes -- and the stand-ins do not.  A
   later change to the stand-ins that empties the GPU tests fails here.
2. Separation: defective samplers (test code, next to the oracle's) run through the same oracles, and how far each lies
   above the bar the GPU tests hold the engine to, on the stand-in's small motion and on the steered inputs
   (split_engine_bars.SEPARATION_FLOW_MOTION).
"""
import pytest
import torch

import flow_steering as S
import split_engine_bars as bars
from oracle import pwc_net
from oracle import raft_net as R

PWC_BAR = {"volume": 1e-4, "flow": 1e-4, "final": (1e-4, 1e-4)}          # test_pwc_gpu.py's stages


@pytest.fixture(scope="module", autouse=True)
def _no_grad():
    with torch.no_grad():
        yield


@pytest.fixture(scope="module")
def pwc_sd():
    return {k: v.double() for k, v in pwc_net.stand_in_state_dict().items()}


@pytest.fixture(scope="module")
def raft_sd():
    from helpers import stand_in_state_dict
    return {k: v.double() for k, v in stand_in_state_dict("raft-sintel.pth").items()}


def _pwc(sd, size=(128, 160)):
    x = R.synthetic_frames(3, *size, **S.PWC_FRAMES[size]).double()
    st = {}
    y = pwc_net.forward(sd, x[:-1], x[1:], torch.float64, stages=st)
    return y, st


def _warp_regimes(st):
    return {l: S.warp_regime(st[f"maskraw{l}"], st[f"upflow{l}"] * pwc_net.DBL_BACKWARD[l]) for l in (5, 4, 3, 2)}


def _near_threshold(st, levels=(5, 4, 3, 2), rel=1e-4):
    """Raw mask values a 1e-4 relative error of the displacement could carry across 0.999 (test_pwc_gpu.py
    _assert_masks_clear)."""
    return sum(int(((st[f"maskraw{l}"] - 0.999).abs()
                    < rel * float((st[f"upflow{l}"] * pwc_net.DBL_BACKWARD[l]).abs().max())).sum()) for l in levels)


# ------------------------------------------------------------------------------------------------------ regimes

def test_pwc_stand_in_never_leaves_its_own_pixel(pwc_sd):
    """What the existing GPU tests' inputs exercise: at most ~1 px of warp, no sample fully outside, no masked interior
    pixel."""
    for size in ((128, 160), (200, 333)):
        for l, r in _warp_regimes(_pwc(pwc_sd, size)[1]).items():
            print(size, l, r)
            assert r["max displacement"] < 1.5 and r["all taps outside"] == 0 and r["masked interior"] == 0, (l, r)


@pytest.mark.parametrize("level", (5, 4, 3, 2))
def test_pwc_uniform_warps_reach_their_regime(pwc_sd, level):
    for size in ((128, 160), (200, 333)):
        for d in S.PWC_UNIFORM[level]:
            sd, disp = S.pwc_uniform_warp(pwc_sd, level, *d)
            st = _pwc(sd, size)[1]
            r = _warp_regimes(st)[level]
            print(size, level, disp, r)
            h, w = st[f"maskraw{level}"].shape[2:]
            assert max(abs(d[0] - disp[0]), abs(d[1] - disp[1])) < 0.01
            assert r["cell offsets"] == 1 and r["max displacement"] == max(abs(disp[0]), abs(disp[1]))
            assert torch.equal(st[f"upflow{level}"][:, 0], torch.full_like(st[f"upflow{level}"][:, 0],
                                                                           disp[0] / pwc_net.DBL_BACKWARD[level]))
            assert r["all taps outside"] > 0 and r["masked interior"] > 0, r
            # the mask of a uniform warp takes a few values far from 0.999: the engine's must equal it exactly
            raw = st[f"maskraw{level}"]
            assert float((raw - 0.999).abs().min()) > 1e-3
            if abs(disp[0]) >= w and abs(disp[1]) >= h:
                assert r["all taps outside"] == raw.numel()
    sd, _ = S.pwc_uniform_warp(pwc_sd, 2, -7.75, 3.25)
    r = _warp_regimes(_pwc(sd)[1])[2]
    assert r["all taps outside"] > 300 and r["masked interior"] > 300, r


def test_pwc_threshold_warps_bracket_0_999(pwc_sd):
    for (dx, dy), border in S.PWC_THRESHOLD.items():
        sd, disp = S.pwc_uniform_warp(pwc_sd, 2, dx, dy)
        st = _pwc(sd)[1]
        raw, mask = st["maskraw2"], st["mask2"]
        want = torch.ones_like(mask)
        if dx:
            want[..., :, -1] = border
        else:
            want[..., 0, :] = border
        assert torch.equal(mask, want), (dx, dy)
        edge = float(raw.min())
        # 5e-4 from the threshold: two hundred times the 2e-6 an fp32 coordinate of ~48 costs
        assert abs(abs(edge - 0.999) - 5e-4) < 2e-5, edge


def test_pwc_varying_warps_reach_their_regime(pwc_sd):
    want = {"level 2 x9": (2, 8.0), "level 4 x75": (4, 3.0)}
    for name, gains in S.PWC_VARYING.items():
        st = _pwc(S.pwc_varying_warp(pwc_sd, gains))[1]
        level, least = want[name]
        r = _warp_regimes(st)[level]
        print(name, r)
        assert r["max displacement"] >= least and r["all taps outside"] > 0 and r["masked interior"] > 0, r
        assert r["cell offsets"] >= 10, r
        assert _near_threshold(st) == 0


def test_pwc_smallest_map(pwc_sd):
    """40x50 frames: a 64x64 working size, level 6 is one pixel, level 5 2x2."""
    y, st = _pwc(pwc_sd, (40, 50))
    assert st["feats1"][5].shape[2:] == (1, 1) and st["maskraw5"].shape[2:] == (2, 2)
    assert torch.isfinite(y).all() and _near_threshold(st) == 0
    sd, _ = S.pwc_uniform_warp(pwc_sd, 3, 3.25, -2.5)
    y, st = _pwc(sd, (40, 50))
    assert torch.isfinite(y).all() and _warp_regimes(st)[3]["masked interior"] > 0


def _raft(sd, iters, size=(128, 160), **kw):
    x = R.pad(R.synthetic_frames(2, *size, seed=size[0])).double()
    return R.forward(sd, x[:-1], x[1:], iters, taps=True, declared_rounding=True, **kw)


def _last_centres(st):
    """coords1 of the last iteration's lookup."""
    low = st["lowres"]
    n, _, h, w = low[-1].shape
    ys, xs = torch.meshgrid(torch.arange(h), torch.arange(w), indexing="ij")
    prev = low[-2] if len(low) > 1 else torch.zeros_like(low[-1])
    return prev + torch.stack([xs, ys]).to(prev)


def test_raft_stand_in_stays_in_its_own_cell(raft_sd):
    for iters in (3, 20):
        r = S.lookup_regime(_last_centres(_raft(raft_sd, iters)[1]))
        print(iters, r)
        assert r["max offset"] < 0.5 and r["windows outside"] == 0, r


def test_raft_uniform_steps_reach_their_regime(raft_sd):
    seen = {"windows outside": 0, "max offset": 0.0}
    for (du, dv), iters in S.RAFT_UNIFORM:
        up, st = _raft(S.raft_uniform_step(raft_sd, du, dv), iters)
        want = torch.tensor([du, dv], dtype=torch.float64).view(1, 2, 1, 1) * iters
        assert torch.equal(st["lowres"][-1], want.expand_as(st["lowres"][-1]))        # dyadic steps: exact sums
        r = S.lookup_regime(_last_centres(st))
        print((du, dv), iters, r)
        assert r["cell offsets"] == 1 and r["centres outside"] > 0, r
        assert r["max offset"] == (iters - 1) * max(abs(du), abs(dv))
        seen = {k: max(v, r[k]) for k, v in seen.items()}
        assert torch.isfinite(up).all()
    assert seen["max offset"] >= 3 and seen["windows outside"] > 0, seen
    # (9, 7) x 5: every level-0 window is off the map, level 3 (2 x 2) still partly on it
    up, st = _raft(S.raft_uniform_step(raft_sd, 9.0, 7.0), 6)
    look = st["lookup"][-1]
    assert float(look[:, :81].abs().max()) == 0 and float(look[:, 243:].abs().max()) > 0


def test_raft_varying_flow_reaches_its_regime(raft_sd):
    up, st = _raft(S.raft_varying_flow(raft_sd, S.RAFT_VARYING_GAIN), 20)
    r = S.lookup_regime(_last_centres(st))
    print(r, float(st["lowres"][-1].abs().max()))
    assert r["max offset"] >= 2.5 and r["cell offsets"] >= 12 and r["centres outside"] > 0, r


def test_raft_sharp_mask_saturates_the_softmax(raft_sd):
    plain = _raft(raft_sd, 3)[1]["mask"]
    up, st = _raft(S.raft_sharp_mask(raft_sd, S.RAFT_SHARP_GAIN), 3)
    m = st["mask"]
    p = torch.softmax(m.view(-1, 9, 64, *m.shape[2:]), 1).amax(1)
    print(float(plain.abs().max()), float(m.abs().max()), float((p > 0.999).double().mean()))
    assert float(plain.abs().max()) < 5 and 30 < float(m.abs().max()) < 80
    assert float((p > 0.999).double().mean()) > 0.2 and torch.isfinite(up).all()
    # the mask head's last conv is a single-fp16 operand of the engine: the gained weights must stay in range
    assert float(S.raft_sharp_mask(raft_sd, S.RAFT_SHARP_GAIN)[S.RAFT_MASK2 + ".weight"].abs().max()) < 1000


# --------------------------------------------------------------------------------------------------- separation

def _trunc(t):
    return torch.trunc(t)


def _bilinear(img, x, y, floor=torch.floor, clamp=False):
    """img (B, C, H, W) sampled at pixel coordinates x, y (B, ...) -> (B, C, ...) and the in-bounds weight sum: zeros
    outside the map; `floor` = _trunc and `clamp` are the defects (int(x) for floorf(x); border clamp for zero padding)."""
    B, C, H, W = img.shape
    flat = img.reshape(B, C, H * W)
    shape = x.shape
    x, y = x.reshape(B, -1), y.reshape(B, -1)
    x0, y0 = floor(x), floor(y)
    ax, ay = x - x0, y - y0
    out, wsum = torch.zeros(B, C, x.shape[1], dtype=img.dtype), torch.zeros_like(x)
    for dy, dx in ((0, 0), (0, 1), (1, 0), (1, 1)):
        xi, yi = x0 + dx, y0 + dy
        wgt = (ax if dx else 1 - ax) * (ay if dy else 1 - ay)
        inside = (xi >= 0) & (xi <= W - 1) & (yi >= 0) & (yi <= H - 1)
        if clamp:
            inside = torch.ones_like(inside)
        idx = (yi.clamp(0, H - 1) * W + xi.clamp(0, W - 1)).long()
        wgt = torch.where(inside, wgt, torch.zeros_like(wgt))
        out = out + wgt[:, None] * flat.gather(2, idx[:, None].expand(-1, C, -1))
        wsum = wsum + wgt
    return out.view(B, C, *shape[1:]), wsum.view(B, 1, *shape[1:])


def _warp(floor=torch.floor, clamp=False, mask=">"):
    def backward_warp(x, flow, align_corners=True):
        n, _, h, w = flow.shape
        ys, xs = torch.meshgrid(torch.arange(h, dtype=flow.dtype), torch.arange(w, dtype=flow.dtype), indexing="ij")
        out, raw = _bilinear(x, xs + flow[:, 0], ys + flow[:, 1], floor, clamp)
        m = {">": raw > 0.999, ">=": raw >= 0.999, "none": torch.ones_like(raw, dtype=torch.bool)}[mask].to(x.dtype)
        return out * m, m, raw
    return backward_warp


def _warp_align_corners_false(x, flow, align_corners=True):
    return _ORACLE_WARP(x, flow, False)


_ORACLE_WARP = pwc_net.backward_warp
_ORACLE_DECONV = pwc_net._deconv
_ORACLE_MOTION = R.motion_encoder


def _deconv_upflow_hi_only(sd, name, x):
    """The upsampled flow kept as one fp16 value (the lo half of the engine's split pair lost)."""
    y = _ORACLE_DECONV(sd, name, x)
    return y.half().to(y.dtype) if name.endswith("moduleUpflow") else y


def _motion_flow_hi_only(sd, flow, corr):
    """The flow the motion encoder reads kept as one fp16 value (the lo half of the pair in hx / qx lost)."""
    return _ORACLE_MOTION(sd, flow.half().to(flow.dtype), corr)


PWC_DEFECTS = {"truncation for floor": _warp(floor=_trunc), "border clamp for zeros": _warp(clamp=True),
               "mask >= 0.999": _warp(mask=">="), "mask dropped": _warp(mask="none"),
               "align_corners=False": _warp_align_corners_false, "upflow pair's lo half lost": _ORACLE_WARP}


def _pwc_stage_errors(got, ref, levels, bar):
    """Worst rel-L2 over its bar among the stages the GPU test asserts (cost volume and decoder flow of `levels`, final
    flow)."""
    rel = lambda a, b: float((a - b).norm() / b.norm())
    return max([rel(got[1][f"{s}{l}"], ref[1][f"{s}{l}"]) / bar[k] for l in levels for s, k in (("vol", "volume"), ("flow", "flow"))]
               + [rel(got[0], ref[0]) / bar["final"][0]])


def test_pwc_defective_warps_are_separated_only_under_motion(pwc_sd, monkeypatch):
    inputs = {"small motion": (pwc_sd, (5, 4, 3, 2)),
              "uniform level 2": (S.pwc_uniform_warp(pwc_sd, 2, -7.75, 3.25)[0], (2,)),
              "varying level 2": (S.pwc_varying_warp(pwc_sd, S.PWC_VARYING["level 2 x9"]), (2,))}
    refs = {k: _pwc(sd) for k, (sd, _) in inputs.items()}
    monkeypatch.setattr(pwc_net, "backward_warp", _warp())
    for k, (sd, levels) in inputs.items():          # the test sampler without a defect is the oracle's
        assert _pwc_stage_errors(_pwc(sd), refs[k], levels, PWC_BAR) < 1e-8
    table = bars.SEPARATION_FLOW_MOTION["pwc"]
    assert set(table) == set(PWC_DEFECTS)
    failures = []
    for name, warp in PWC_DEFECTS.items():
        monkeypatch.setattr(pwc_net, "backward_warp", warp)
        monkeypatch.setattr(pwc_net, "_deconv", _deconv_upflow_hi_only if "lo half" in name else _ORACLE_DECONV)
        for k, (sd, levels) in inputs.items():
            x = _pwc_stage_errors(_pwc(sd), refs[k], levels, PWC_BAR if k == "small motion" else bars.PWC_MOTION_BARS)
            stated = table[name][k]
            print(f"pwc {name:<24s} {k:<16s} {x:10.3g}x the bar (stated {stated})")
            if stated == 0 and x >= 1:
                failures.append((name, k, x, "stated as not separated"))
            if stated and x < stated:
                failures.append((name, k, x, stated))
    assert not failures, failures


def _lookup(floor=torch.floor, clamp=False, transposed=True, floor_before_scale=False):
    def corr_lookup(pyr, coords, pixel_sampler=False):
        r = R.CORR_RADIUS
        b, _, h1, w1 = coords.shape
        d = torch.arange(-r, r + 1, dtype=coords.dtype)
        first, second = torch.meshgrid(d, d, indexing="ij")           # window axes 0 and 1
        ox, oy = (first, second) if transposed else (second, first)
        out = []
        for i in range(R.CORR_LEVELS):
            c = (torch.floor(coords) if floor_before_scale else coords) / 2 ** i
            x = c[:, 0].reshape(-1, 1, 1) + ox
            y = c[:, 1].reshape(-1, 1, 1) + oy
            out.append(_bilinear(pyr[i], x, y, floor, clamp)[0].view(b, h1, w1, -1))
        return torch.cat(out, -1).permute(0, 3, 1, 2).contiguous()
    return corr_lookup


RAFT_DEFECTS = {"truncation for floor": _lookup(floor=_trunc), "border clamp for zeros": _lookup(clamp=True),
                "window not transposed": _lookup(transposed=False),
                "level scaling after the floor": _lookup(floor_before_scale=True), "flow pair's lo half lost": _lookup()}


def test_raft_defective_lookups_are_separated_only_under_motion(raft_sd, monkeypatch):
    inputs = {"small motion": (raft_sd, 3),
              "uniform step": (S.raft_uniform_step(raft_sd, 2.25, 1.75), 3),
              "varying flow": (S.raft_varying_flow(raft_sd, S.RAFT_VARYING_GAIN), 20)}
    bar = {"small motion": bars.RAFT_BARS, "uniform step": bars.RAFT_MOTION_BARS["uniform"],
           "varying flow": bars.RAFT_MOTION_BARS["varying 20"]}
    stages = lambda r: {"lookup": r[1]["lookup"][-1], "net": r[1]["net"][-1], "flow_up": r[0]}
    refs = {k: stages(_raft(sd, it)) for k, (sd, it) in inputs.items()}
    monkeypatch.setattr(R, "corr_lookup", _lookup())
    for k, (sd, it) in inputs.items():
        got = stages(_raft(sd, it))
        assert all(bars.within(bars.row_errors(got[s], refs[k][s]), (1e-12, 1e-12)) for s in got), k
    table = bars.SEPARATION_FLOW_MOTION["raft"]
    assert set(table) == set(RAFT_DEFECTS)
    failures = []
    for name, lookup in RAFT_DEFECTS.items():
        monkeypatch.setattr(R, "corr_lookup", lookup)
        monkeypatch.setattr(R, "motion_encoder", _motion_flow_hi_only if "lo half" in name else _ORACLE_MOTION)
        for k, (sd, it) in inputs.items():
            got = stages(_raft(sd, it))
            # bars.beyond: rel-L2 or max-abs, whichever is further above its bar, at the worst stage
            x = max(e / b for s in got for e, b in zip(bars.row_errors(got[s], refs[k][s]), bar[k][s]))
            stated = table[name][k]
            print(f"raft {name:<30s} {k:<14s} {x:10.3g}x the bar (stated {stated})")
            if stated == 0 and x >= 1:
                failures.append((name, k, x, "stated as not separated"))
            if stated and x < stated:
                failures.append((name, k, x, stated))
    assert not failures, failures

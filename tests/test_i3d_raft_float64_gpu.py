"""I3DEngine and RAFTEngine against a float64 forward of the same network on the GPU, with the engine's declared
rounding (oracle/i3d_net.py, oracle/raft_net.py, declared_rounding=True): the operands the engine keeps as single fp16
are rounded to fp16 in the reference, every other operand stays float64.  What is left of the engine's error is its
fp32 accumulation and the split-fp16 pairs' ~22-bit operands, so a lost lo half, W_lo pass or lo_mask bit shows.

The fp32-oracle tests (test_i3d_gpu.py, test_raft_gpu.py) cannot see that: their bars (I3D 6e-4, RAFT 1e-4) are as
large as what one tensor class left in single fp16 costs (DESIGN.md §2 note 3).  Bars: tests/split_engine_bars.py.

I3D runs the checkpoint stand-ins at rgb T = 16, 11 (odd), one call of two stacks, and flow T = 12, and checks every
read_stage stage and the features.  RAFT runs the raft-sintel stand-in at 128x160 (3 frames), 200x200 (odd /8 map) and
270x480 after 1 and 3 iterations: fnet, cnet, the correlation pyramid, the last lookup, the GRU hidden state, the
low-res flow and flow_up; and flow_up after 20 iterations against a looser bar (the refinement amplifies rounding).
Controls through the public API: fp16-rounded conv weights (W_lo exactly zero), VF_I3D_FAST / VF_RAFT_FAST (every
weight single fp16) fail; VF_I3D_SINGLE=none passes the reference with no rounded weights; an fp16-rounded I3D input
gives the same bits (the stem input is single fp16, as declared).  At a padded side of 64 .. 127 px (a 1-pixel 4th
pyramid level, where the reference returns NaN) RAFT is compared with a float64 oracle whose sampler works in pixel
coordinates; under 64 px it rejects the frames.

test_zz_report_measured prints the worst row per stage over the session (pytest -s).
"""
import pytest
import torch

import split_engine_bars as bars
from oracle import i3d_net
from oracle import raft_net as R

pytestmark = pytest.mark.gpu

MEASURED = {}


def _f64(sd, dev):
    return {k: (v.double() if v.is_floating_point() else v).to(dev) for k, v in sd.items()}


def _fp16_weights(sd):
    """Conv weights (4-D / 5-D) rounded to fp16: the engine's W_lo is then exactly zero."""
    return {k: (v.half().float() if v.is_floating_point() and v.dim() >= 4 else v) for k, v in sd.items()}


def _compare(what, got, want, bar, record=True):
    assert got.shape == want.shape, (what, tuple(got.shape), tuple(want.shape))
    err = bars.row_errors(got, want)
    print(f"{what}: rel-L2 {err[0]:.2e}, max-abs/max {err[1]:.2e} (bar {bar[0]:.1e} / {bar[1]:.1e})")
    if record:
        key = what.split(" ")[0] + " " + what.split(" ")[-1]
        old = MEASURED.get(key, (0.0, 0.0))
        MEASURED[key] = (max(old[0], err[0]), max(old[1], err[1]))
    return err


def _failures(errs, bar):
    return [(s, e) for s, e in errs.items() if not bars.within(e, bar[s])]


# ---------------------------------------------------------------------------------------------------------- I3D

def _i3d_sd(modality):
    from helpers import checkpoint
    return torch.load(checkpoint(f"i3d_{modality}.pt"), map_location="cpu")


def _i3d_ref(sd, x, dev, **kw):
    with torch.no_grad():
        return i3d_net.forward_features(_f64(sd, dev), x.double().to(dev), return_stages=True, **kw)


def _i3d_errors(name, eng, y, ref, record=True):
    out, st = ref
    bar = bars.I3D_BARS[eng.modality]
    errs = {"features": _compare(f"{name} features", y, out, bar["features"], record)}
    for sid, s in enumerate(bars.I3D_STAGES[:-1]):
        errs[s] = _compare(f"{name} {s}", eng.read_stage(sid), st[s], bar[s], record)
    return errs


@pytest.mark.parametrize("modality,T,n", [("rgb", 16, 1), ("rgb", 11, 1), ("rgb", 16, 2), ("flow", 12, 1)])
def test_i3d_matches_float64(cuda_device, modality, T, n):
    from video_features_b200.i3d_engine import I3DEngine
    sd = _i3d_sd(modality)
    cin = 3 if modality == "rgb" else 2
    x = (torch.rand(n, cin, T, 224, 224, generator=torch.Generator().manual_seed(40 + T)) * 2 - 1).to(cuda_device)
    eng = I3DEngine(sd, modality, 0, max_stacks=n, max_T=16)
    y = eng(x)
    name = f"i3d-{modality}-T{T}x{n}"
    errs = _i3d_errors(name, eng, y, _i3d_ref(sd, x, cuda_device, declared_rounding=True))
    _i3d_errors(f"{name} (vs plain float64)", eng, y, _i3d_ref(sd, x, cuda_device), record=False)
    eng.close()
    assert not _failures(errs, bars.I3D_BARS[modality])


def test_i3d_controls(cuda_device, monkeypatch):
    """fp16 weights: the 2c stage (the first with split weights: the stem's are single fp16) fails tenfold against the
    declared reference of the original weights and passes against that of the rounded ones.  VF_I3D_FAST=1 fails;
    VF_I3D_SINGLE=none passes the reference with no fp16 weights; an fp16-rounded input gives the same bits."""
    from video_features_b200.i3d_engine import I3DEngine
    sd = _i3d_sd("rgb")
    x = (torch.rand(1, 3, 12, 224, 224, generator=torch.Generator().manual_seed(9)) * 2 - 1).to(cuda_device)
    ref = _i3d_ref(sd, x, cuda_device, declared_rounding=True)
    bar = bars.I3D_BARS["rgb"]

    sd16 = _fp16_weights(sd)
    eng = I3DEngine(sd16, "rgb", 0, max_stacks=1, max_T=16)
    y = eng(x)
    lost = _i3d_errors("i3d fp16-weights vs original", eng, y, ref, False)
    kept = _i3d_errors("i3d fp16-weights vs rounded", eng, y, _i3d_ref(sd16, x, cuda_device, declared_rounding=True),
                       False)
    eng.close()
    assert bars.beyond(lost["2c"], bar["2c"], 10), lost["2c"]
    assert bars.beyond(lost["features"], bar["features"]), lost["features"]
    assert not _failures(kept, bar), kept

    monkeypatch.setenv("VF_I3D_FAST", "1")
    eng = I3DEngine(sd, "rgb", 0, max_stacks=1, max_T=16)
    fast = _i3d_errors("i3d VF_I3D_FAST=1", eng, eng(x), ref, False)
    eng.close()
    monkeypatch.delenv("VF_I3D_FAST")
    assert bars.beyond(fast["2c"], bar["2c"], 10), fast["2c"]

    monkeypatch.setenv("VF_I3D_SINGLE", "none")
    eng = I3DEngine(sd, "rgb", 0, max_stacks=1, max_T=16)
    y = eng(x)
    none = _i3d_errors("i3d VF_I3D_SINGLE=none", eng, y, _i3d_ref(sd, x, cuda_device, declared_rounding=True,
                                                                   fp16_units=()), False)
    stem_lost = _i3d_errors("i3d VF_I3D_SINGLE=none vs fp16 stem weights", eng, y, ref, False)["1a"]
    assert torch.equal(eng(x.half().float()), y)       # the stem input is single fp16
    eng.close()
    monkeypatch.delenv("VF_I3D_SINGLE")
    assert not _failures(none, bar), none
    assert bars.beyond(stem_lost, bar["1a"], 10), stem_lost


def test_i3d_read_stage_follows_the_last_call(cuda_device):
    """read_stage describes the last call also when it replays a cached graph: one clip, two clips, one clip again
    (stages 2 and 3 sit at offsets that depend on the clip count)."""
    from video_features_b200.i3d_engine import I3DEngine
    sd = i3d_net.synthetic_state_dict("rgb", 4)
    g = torch.Generator().manual_seed(12)
    x1 = (torch.rand(1, 3, 12, 224, 224, generator=g) * 2 - 1).to(cuda_device)
    x2 = (torch.rand(2, 3, 12, 224, 224, generator=g) * 2 - 1).to(cuda_device)
    eng = I3DEngine(sd, "rgb", 0, max_stacks=2, max_T=16)
    eng(x1)
    first = [eng.read_stage(i).clone() for i in range(5)]
    eng(x2)
    assert all(eng.read_stage(i).shape[0] == 2 for i in range(5))
    eng(x1)
    again = [eng.read_stage(i) for i in range(5)]
    eng.close()
    for i, (a, b) in enumerate(zip(first, again)):
        assert a.shape == b.shape and torch.equal(a, b), i


# --------------------------------------------------------------------------------------------------------- RAFT

@pytest.fixture(scope="module")
def raft(cuda_device):
    from helpers import stand_in_state_dict
    from video_features_b200.raft_engine import RAFTEngine
    sd = stand_in_state_dict("raft-sintel.pth")
    eng = RAFTEngine(sd, 0, max_frames=3, max_h=272, max_w=480)
    yield sd, eng
    eng.close()


def _pyramid(rows, pyr):
    """The engine's pyramid rows (vf_raft_debug_read 5: per pair and /8 position, level 0 at column 0, level l >= 1 at
    P8 + the sizes of the levels l' in 1 .. l-1; the columns between are padding) and the oracle's pyramid, both as
    (pairs, P, level 0 | level 1 | level 2 | level 3)."""
    n, P = rows.shape[:2]
    got, want, off = [], [], 0
    for lv, p in enumerate(pyr):
        hw = p.shape[-2] * p.shape[-1]
        got.append(rows[:, :, 0, off:off + hw])
        want.append(p.reshape(n, P, hw))
        off = (P + 7) // 8 * 8 if lv == 0 else off + hw
    return torch.cat(got, -1), torch.cat(want, -1)


def _raft_errors(name, eng, xp, iters, ref, record=True, bar=bars.RAFT_BARS):
    """Runs the engine on padded frames xp and compares every debug_read tensor and flow_up with ref (flow_up, taps)."""
    y = eng.flow(xp, iters=iters, unpad=False)
    up, st = ref
    n = xp.shape[0] - 1
    f = st["fnet"]
    got = {s: eng.debug_read(i) for s, i in (("fnet", 0), ("cnet", 1), ("net", 2), ("lowres", 3), ("lookup", 4))}
    want = {"fnet": torch.cat([f[:n], f[-1:]]), "cnet": st["cnet"], "net": st["net"][-1], "lowres": st["lowres"][-1],
            "lookup": st["lookup"][-1]}
    got["pyramid"], want["pyramid"] = _pyramid(eng.debug_read(5), st["pyramid"])
    errs = {s: _compare(f"{name} {s}", got[s], want[s], bar[s], record) for s in bars.RAFT_STAGES[:-1]}
    errs["flow_up"] = _compare(f"{name} flow_up", y, up, bar["flow_up"], record)
    return errs


def _raft_ref(sd, xp, iters, **kw):
    dev = xp.device
    x = xp.double()
    with torch.no_grad():
        return R.forward(_f64(sd, dev), x[:-1], x[1:], iters, taps=True, **kw)


@pytest.mark.parametrize("h,w,n", [(128, 160, 3), (200, 200, 2), (270, 480, 2)])
def test_raft_matches_float64(raft, cuda_device, h, w, n):
    sd, eng = raft
    xp = R.pad(R.synthetic_frames(n, h, w, seed=h).to(cuda_device))
    failures = []
    for iters in (1, 3):
        errs = _raft_errors(f"raft-{h}x{w}-it{iters}", eng, xp, iters, _raft_ref(sd, xp, iters, declared_rounding=True))
        failures += [(iters, s, e) for s, e in _failures(errs, bars.RAFT_BARS)]
    y = eng.flow(xp, iters=20, unpad=False)
    up = _raft_ref(sd, xp, 20, declared_rounding=True)[0]
    e20 = _compare(f"raft-{h}x{w}-it20 flow_up20", y, up, bars.RAFT_BAR_20_ITERS)
    _compare(f"raft-{h}x{w}-it20 (vs plain float64) flow_up20", y, _raft_ref(sd, xp, 20)[0], bars.RAFT_BAR_20_ITERS,
             False)
    assert not failures, failures
    assert bars.within(e20, bars.RAFT_BAR_20_ITERS), e20


@pytest.mark.parametrize("h,w", [(96, 128), (64, 120)])
def test_raft_one_pixel_pyramid_level(raft, cuda_device, h, w):
    """Padded 96x128 (level 3 is 1x2) and 64x120 (1x1): the reference returns NaN there (its sampler divides by H - 1
    = 0); the engine's lookup samples the integer neighbourhood with zeros outside the map, which is what the
    pixel-coordinate sampler computes."""
    sd, eng = raft
    xp = R.pad(R.synthetic_frames(3, h, w, seed=h).to(cuda_device))
    assert tuple(xp.shape[-2:]) == (h, w)
    failures = []
    for iters in (1, 3):
        errs = _raft_errors(f"raft-{h}x{w}-it{iters}", eng, xp, iters,
                            _raft_ref(sd, xp, iters, declared_rounding=True, pixel_sampler=True))
        failures += [(iters, s, e) for s, e in _failures(errs, bars.RAFT_BARS)]
    assert not failures, failures


def test_raft_rejects_frames_under_64_px(raft, cuda_device):
    """Under 64 padded px the 4th pyramid level would have no rows (the reference's avg_pool2d raises)."""
    from video_features_b200._lib import VfError
    sd, eng = raft
    for h, w in ((56, 128), (128, 40)):
        with pytest.raises(VfError, match="under 64 px"):
            eng.flow(R.synthetic_frames(2, h, w, seed=1).to(cuda_device), iters=1)


def test_raft_controls(cuda_device, monkeypatch):
    """fp16 weights fail fnet's bar tenfold against the declared reference of the original weights and pass against
    that of the rounded ones; VF_RAFT_FAST=1 fails."""
    from helpers import stand_in_state_dict
    from video_features_b200.raft_engine import RAFTEngine
    sd = stand_in_state_dict("raft-sintel.pth")
    xp = R.pad(R.synthetic_frames(2, 128, 160, seed=21).to(cuda_device))
    ref = _raft_ref(sd, xp, 1, declared_rounding=True)

    sd16 = _fp16_weights(sd)
    eng = RAFTEngine(sd16, 0, max_frames=2, max_h=128, max_w=160)
    lost = _raft_errors("raft fp16-weights vs original", eng, xp, 1, ref, False)
    kept = _raft_errors("raft fp16-weights vs rounded", eng, xp, 1, _raft_ref(sd16, xp, 1, declared_rounding=True),
                        False)
    eng.close()
    assert bars.beyond(lost["fnet"], bars.RAFT_BARS["fnet"], 10), lost["fnet"]
    assert bars.beyond(lost["flow_up"], bars.RAFT_BARS["flow_up"]), lost["flow_up"]
    assert not _failures(kept, bars.RAFT_BARS), kept

    monkeypatch.setenv("VF_RAFT_FAST", "1")
    eng = RAFTEngine(sd, 0, max_frames=2, max_h=128, max_w=160)
    fast = _raft_errors("raft VF_RAFT_FAST=1", eng, xp, 1, ref, False)
    eng.close()
    assert bars.beyond(fast["fnet"], bars.RAFT_BARS["fnet"], 10), fast["fnet"]


def test_zz_report_measured(cuda_device):
    """Prints the worst row per run and stage over the tests above (run in the same session)."""
    for k, (rel, mx) in sorted(MEASURED.items()):
        print(f"measured worst {k}: rel-L2 {rel:.2e}, max-abs/max {mx:.2e}")

"""The I3D and S3D Mixed blocks branch by branch, and the pool and head kernels both trunks share, against float64.

Every Mixed block of I3D (rgb and flow stand-ins) and S3D runs on its own through the engines' debug entries (the
trunk's own buffers and kernels) on a split-fp16 pair input: the float64 trunk's real input to that block, and a
synthetic non-negative input with about half its elements exactly zero, at T = 1, 2, 3, 8 and one or three clips.  The
input is canonical (hi = fp16(v), lo = fp16(v - hi)) and the reference reads exactly hi + lo, so what is left of the
difference is the block's own arithmetic.  Each of the four branch slices of the concat output is compared on its own
(worst clip, rel-L2 and max-abs / max): S3D against plain float64, I3D against float64 with its declared rounding.  A
lo half lost in one branch's store, conv input or W_lo pass is smaller than the stage bars past Mixed 3c, but tenfold
or more above these (test_inception_block_bars_cpu.py).  Every border row of the output must be exactly zero: the next
block reads it as padding.

Controls: one split conv's weights pre-rounded to fp16 fail that branch's bar and leave the other three bit-identical;
I3D's declared single-fp16 units pre-rounded change no bit; an input whose lo half is dropped fails every branch.

Pools: every pool call of both trunks, at even and odd extents, plus small-C cases on either side of every dispatch
condition, bit for bit against the float64 max of hi + lo re-split (the max of exact sums is exact); the kernel that ran
is asserted.  Head: the (2,7,7) average pool and temporal mean against float64.

Bars: tests/inception_block_bars.py.  test_zz_report_measured prints the worst values of the session (pytest -s)."""
import pytest
import torch
import torch.nn.functional as F

import inception_block_bars as ib
import split_engine_bars as bars
from oracle import i3d_net, s3d_net

pytestmark = pytest.mark.gpu

MEASURED = {}          # (engine, block, branch) -> worst (rel-L2, max-abs / max)
PATHS = {}             # pool case -> VF_POOL_* kernel that ran
HEAD = {}              # head case -> (rel-L2, max-abs / max)
SHARES = {}            # (engine, defect kind) -> largest |defect_share| of I3D branches 1, 2 over the session
S3D_KEYS = tuple(s3d_net.MIXED)                 # features index of block b
I3D_KEYS = tuple(i3d_net.MIXED)                 # mixed_3b .. mixed_5c
SHAPES = [(1, 1), (2, 3), (3, 1), (8, 3)]       # (T, n) of the synthetic inputs


def _f64(sd, dev):
    return {k: (v.double() if v.is_floating_point() else v).to(dev) for k, v in sd.items()}


def _fp16_weight(sd, key):
    out = dict(sd)
    out[key] = sd[key].half().to(sd[key].dtype)
    return out


# ---- pair volumes
def split(v):
    """float64 NCTHW -> (hi, lo) fp16, canonical: hi = fp16(v), lo = fp16(v - hi)."""
    hi = v.half()
    return hi, (v - hi.double()).half()


def to_pairs(v):
    """float64 (n, C, T, S, S) -> (its exact hi + lo value, the fp16 pair volume (n, T + 2, S + 2, S + 2, 2C) with a
    zero border)."""
    hi, lo = split(v)
    n, c, t, s, _ = v.shape
    x = torch.zeros(n, t + 2, s + 2, s + 2, 2 * c, dtype=torch.float16, device=v.device)
    x[:, 1:-1, 1:-1, 1:-1, :c] = hi.permute(0, 2, 3, 4, 1)
    x[:, 1:-1, 1:-1, 1:-1, c:] = lo.permute(0, 2, 3, 4, 1)
    return hi.double() + lo.double(), x


def from_pairs(y, c):
    """Pair volume (n, T + 2, S + 2, S + 2, 2c) -> float64 (n, c, T, S, S) of hi + lo over the valid region."""
    inner = y[:, 1:-1, 1:-1, 1:-1].double()
    return (inner[..., :c] + inner[..., c:]).permute(0, 4, 1, 2, 3)


def border_nonzero(y):
    """Number of nonzero halves in the border rows of a pair volume."""
    m = torch.ones(y.shape[:4], dtype=torch.bool, device=y.device)
    m[:, 1:-1, 1:-1, 1:-1] = False
    return int((y[m].view(torch.int16) != 0).sum())


def slices(block):
    widths = ib.WIDTHS[block][1:]
    edges = [0]
    for w in widths:
        edges.append(edges[-1] + w)
    return [(edges[j], edges[j + 1]) for j in range(4)]


def synthetic(block, T, n, seed, dev):
    """Non-negative, about half exactly zero, O(1): a post-ReLU-like block input."""
    g = torch.Generator().manual_seed(seed)
    S, cin = ib.SIDE[block], ib.WIDTHS[block][0]
    return torch.relu(torch.randn(n, cin, T, S, S, generator=g, dtype=torch.float64)).to(dev)


def branch_errors(y, ref, block):
    """[(rel-L2, max-abs / max)] of the four branch slices, worst clip, y the engine's pair volume."""
    got = from_pairs(y, ref.shape[1])
    return [bars.row_errors(got[:, a:b], ref[:, a:b]) for a, b in slices(block)]


def record(engine, block, errs):
    for j, e in enumerate(errs):
        old = MEASURED.get((engine, block, j), (0.0, 0.0))
        MEASURED[(engine, block, j)] = (max(old[0], e[0]), max(old[1], e[1]))


# ---- engines and references
@pytest.fixture(scope="module")
def s3d(cuda_device):
    from video_features_b200.s3d_engine import S3DEngine
    sd = s3d_net.stand_in_state_dict()
    eng = S3DEngine(sd, 0, max_clips=3, max_T=16)
    yield sd, eng
    eng.close()


def _i3d_sd(modality):
    from oracle.stand_in import state_dict
    return state_dict(f"i3d_{modality}.pt")


@pytest.fixture(scope="module", params=["rgb", "flow"])
def i3d(request, cuda_device):
    from video_features_b200.i3d_engine import I3DEngine
    sd = _i3d_sd(request.param)
    eng = I3DEngine(sd, request.param, 0, max_stacks=3, max_T=16)
    yield request.param, sd, eng
    eng.close()


def s3d_ref(sd64, block, x):
    with torch.no_grad():
        return s3d_net.mixed_block(sd64, S3D_KEYS[block], x)


def i3d_ref(sd64, block, x, **kw):
    return i3d_net.mixed_block(sd64, I3D_KEYS[block], x, declared_rounding=True, **kw)


def i3d_directions(m, j):
    """The defects of I3D branch j (1 or 2) of block m that its bars do not separate: the fp16 weights of each of its
    split units (a lost W_lo pass), the fp16 pair input of its 1x1x1 reducer (a lost lo half read or lo_mask bit), its
    store's lost lo half."""
    names = i3d_net.unit_names()
    declared = {names[u] for u in i3d_net.DECLARED_FP16_UNITS}
    return ([("w", f"branch_{j}.{k}") for k in (0, 1) if f"{m}.branch_{j}.{k}" not in declared]
            + [("x", f"branch_{j}.0"), ("store", j)])


def _check_block(name, engine, block, eng_fn, ref_fn, v):
    """Runs one block on v (float64 NCTHW) and returns the failures (branch bar or border)."""
    xv, x = to_pairs(v)
    y = eng_fn(block, x)
    ref = ref_fn(block, xv)
    errs = branch_errors(y, ref, block)
    record(engine, block, errs)
    bar = ib.BARS[engine][block]
    fails = []
    for j, e in enumerate(errs):
        print(f"{name} block {block} branch {j}: rel-L2 {e[0]:.2e}, max-abs/max {e[1]:.2e} "
              f"(bar {bar[j][0]:.1e} / {bar[j][1]:.1e})")
        if not bars.within(e, bar[j]):
            fails.append((name, block, j, e))
    if engine.startswith("i3d"):
        # branches 1 and 2: their bars hold the declared-fp16 flips, so the engine must carry at most SHARE[0] of the
        # direction of each defect those bars do not separate (split weights, the reducer's pair input, the store)
        got = from_pairs(y, ref.shape[1])
        m = I3D_KEYS[block]
        for j in (1, 2):
            a, b = slices(block)[j]
            for d in i3d_directions(m, j):
                if d[0] == "store":
                    ref_d = ref[:, a:b].half().double()
                else:
                    kw = {"fp16_weights" if d[0] == "w" else "fp16_inputs": (f"{m}.{d[1]}",)}
                    ref_d = ref_fn(block, xv, **kw)[:, a:b]
                share = bars.defect_share(got[:, a:b], ref[:, a:b], ref_d)
                key = (engine, d[0])
                SHARES[key] = max(SHARES.get(key, 0.0), abs(share))
                if abs(share) > ib.SHARE[0]:
                    fails.append((name, block, j, d, "share", share))
    nz = border_nonzero(y)
    if nz:
        fails.append((name, block, "border", nz))
    return fails


@pytest.fixture(scope="module")
def s3d_real(s3d, cuda_device):
    """(float64 weights, the float64 trunk's input to every Mixed block) for one 13-frame clip, computed once."""
    sd64 = _f64(s3d[0], cuda_device)
    x = s3d_net.calibration_clips(seed=21, n=1, T=13).double().to(cuda_device)
    with torch.no_grad():
        return sd64, s3d_net.mixed_inputs(sd64, x)


@pytest.fixture(scope="module")
def i3d_real(i3d, cuda_device):
    """(float64 weights, T, the declared-rounding float64 trunk's input to every Mixed block), computed once per
    modality: rgb T = 16, flow T = 12."""
    modality, sd, _ = i3d
    sd64 = _f64(sd, cuda_device)
    cin, T = (3, 16) if modality == "rgb" else (2, 12)
    g = torch.Generator().manual_seed(31 + T)
    x = (torch.rand(1, cin, T, 224, 224, generator=g, dtype=torch.float64) * 2 - 1).to(cuda_device)
    return sd64, T, i3d_net.mixed_inputs(sd64, x, declared_rounding=True)


@pytest.mark.parametrize("block", range(9))
def test_s3d_block_matches_float64(s3d, s3d_real, cuda_device, block):
    eng = s3d[1]
    sd64, real = s3d_real

    def ref(b, v, **kw):
        return s3d_ref(sd64, b, v)
    fails = _check_block("s3d real T=13", "s3d", block, eng.debug_mixed, ref, real[block])
    for T, n in SHAPES:
        v = synthetic(block, T, n, 100 * block + T, cuda_device)
        fails += _check_block(f"s3d synthetic T={T} n={n}", "s3d", block, eng.debug_mixed, ref, v)
    assert not fails, fails


@pytest.mark.parametrize("block", range(9))
def test_i3d_block_matches_float64(i3d, i3d_real, cuda_device, block):
    modality, _, eng = i3d
    sd64, T, real = i3d_real
    engine = f"i3d-{modality}"

    def ref(b, v, **kw):
        return i3d_ref(sd64, b, v, **kw)
    fails = _check_block(f"{engine} real T={T}", engine, block, eng.debug_mixed, ref, real[block])
    for Tb, n in SHAPES:
        v = synthetic(block, Tb, n, 100 * block + Tb + 7, cuda_device)
        fails += _check_block(f"{engine} synthetic T={Tb} n={n}", engine, block, eng.debug_mixed, ref, v)
    assert not fails, fails


# ---- controls
def _control_input(block, dev):
    return synthetic(block, 3, 1, 7000 + block, dev)


def test_s3d_control_fp16_weights_of_one_conv(s3d, cuda_device):
    """features.12 (Mixed 4f) branch1's temporal conv with fp16 weights (its W_lo pass multiplies zeros): branch 1
    fails its bar by the factor the bars file names; branches 0, 2 and 3 are bit-identical to the intact engine's."""
    from video_features_b200.s3d_engine import S3DEngine
    sd, eng = s3d
    block, branch, key = ib.S3D_CONTROL
    bad = S3DEngine(_fp16_weight(sd, key), 0, max_clips=1, max_T=16)
    xv, x = to_pairs(_control_input(block, cuda_device))
    y, y_bad = eng.debug_mixed(block, x), bad.debug_mixed(block, x)
    bad.close()
    errs = branch_errors(y_bad, s3d_ref(_f64(sd, cuda_device), block, xv), block)
    bar = ib.BARS["s3d"][block][branch]
    print(f"s3d control {key}: rel-L2 {errs[branch][0]:.2e} ({errs[branch][0] / bar[0]:.1f}x bar), max-abs/max "
          f"{errs[branch][1]:.2e} ({errs[branch][1] / bar[1]:.1f}x bar)")
    assert bars.beyond(errs[branch], bar, ib.CONTROL_FACTOR["s3d"]), errs[branch]
    ctot = sum(ib.WIDTHS[block][1:])
    for j, (a, b) in enumerate(slices(block)):
        if j != branch:
            for off in (0, ctot):
                assert torch.equal(y[..., off + a:off + b], y_bad[..., off + a:off + b]), (j, off)


def test_i3d_control_fp16_weights(cuda_device, monkeypatch):
    """I3D rgb: the weights of a split unit (mixed_4f branch_0) pre-rounded to fp16 fail branch 0 by the factor the
    bars file names and leave the other branches bit-identical; those of mixed_4f branch_1.1 show as a defect_share of
    their own direction that the intact engine does not carry; the four declared single-fp16 units (5, 7, 11, 13)
    pre-rounded change no bit of blocks 0 and 1; VF_I3D_SINGLE=none passes the reference without fp16 weights."""
    from video_features_b200.i3d_engine import I3DEngine
    sd = _i3d_sd("rgb")
    sd64 = _f64(sd, cuda_device)
    eng = I3DEngine(sd, "rgb", 0, max_stacks=1, max_T=16)
    block, branch, unit = ib.I3D_CONTROL
    name = i3d_net.unit_names()[unit]
    bad = I3DEngine(_fp16_weight(sd, f"{name}.conv3d.weight"), "rgb", 0, max_stacks=1, max_T=16)
    xv, x = to_pairs(_control_input(block, cuda_device))
    y, y_bad = eng.debug_mixed(block, x), bad.debug_mixed(block, x)
    bad.close()
    errs = branch_errors(y_bad, i3d_ref(sd64, block, xv), block)
    bar = ib.BARS["i3d-rgb"][block][branch]
    print(f"i3d control {name}: rel-L2 {errs[branch][0]:.2e} ({errs[branch][0] / bar[0]:.1f}x bar), max-abs/max "
          f"{errs[branch][1]:.2e} ({errs[branch][1] / bar[1]:.1f}x bar)")
    assert bars.beyond(errs[branch], bar, ib.CONTROL_FACTOR["i3d"]), errs[branch]
    ctot = sum(ib.WIDTHS[block][1:])
    for j, (a, b) in enumerate(slices(block)):
        if j != branch:
            for off in (0, ctot):
                assert torch.equal(y[..., off + a:off + b], y_bad[..., off + a:off + b]), (j, off)
    # split units of branches 1 and 2 (under those bars): their fp16 weights show as a share of their own direction,
    # the intact engine carries none of it
    for block, branch, unit in ib.I3D_SHARE_CONTROLS:
        name = i3d_net.unit_names()[unit]
        bad = I3DEngine(_fp16_weight(sd, f"{name}.conv3d.weight"), "rgb", 0, max_stacks=1, max_T=16)
        xv, x = to_pairs(_control_input(block, cuda_device))
        a, b = slices(block)[branch]
        ref = i3d_ref(sd64, block, xv)[:, a:b]
        ref_defect = i3d_ref(sd64, block, xv, fp16_weights=(name,))[:, a:b]
        ctot = sum(ib.WIDTHS[block][1:])
        y_bad = from_pairs(bad.debug_mixed(block, x), ctot)[:, a:b]
        share_ok = bars.defect_share(from_pairs(eng.debug_mixed(block, x), ctot)[:, a:b], ref, ref_defect)
        share_bad = bars.defect_share(y_bad, ref, ref_defect)
        err_bad = bars.row_errors(y_bad, ref)
        bar = ib.BARS["i3d-rgb"][block][branch]
        bad.close()
        print(f"i3d control {name}: defect_share intact {share_ok:+.3f}, with fp16 weights {share_bad:+.3f} "
              f"(rel-L2 {err_bad[0] / bar[0]:.1f}x, max-abs {err_bad[1] / bar[1]:.1f}x its bar)")
        assert abs(share_ok) <= ib.SHARE[0] and share_bad >= ib.SHARE[1], (name, share_ok, share_bad)
    # the declared set, block by block
    sd_decl = sd
    for u in i3d_net.DECLARED_FP16_UNITS[1:]:
        sd_decl = _fp16_weight(sd_decl, f"{i3d_net.unit_names()[u]}.conv3d.weight")
    decl = I3DEngine(sd_decl, "rgb", 0, max_stacks=1, max_T=16)
    for b in (0, 1):
        _, xb = to_pairs(_control_input(b, cuda_device))
        assert torch.equal(eng.debug_mixed(b, xb), decl.debug_mixed(b, xb)), b
    decl.close()
    # VF_I3D_SINGLE=none: every unit split; the reference then rounds no weight
    monkeypatch.setenv("VF_I3D_SINGLE", "none")
    none = I3DEngine(sd, "rgb", 0, max_stacks=1, max_T=16)
    monkeypatch.delenv("VF_I3D_SINGLE")
    xv0, x0 = to_pairs(_control_input(0, cuda_device))
    errs = branch_errors(none.debug_mixed(0, x0), i3d_ref(sd64, 0, xv0, fp16_units=()), 0)
    none.close()
    eng.close()
    print(f"i3d VF_I3D_SINGLE=none block 0: {errs}")
    assert all(bars.within(e, ib.BARS["i3d-rgb"][0][j]) for j, e in enumerate(errs)), errs


@pytest.mark.parametrize("engine", ["s3d", "i3d-rgb"])
def test_control_lo_half_dropped(s3d, cuda_device, engine):
    """The input's lo half zeroed, against the reference of hi + lo: every branch fails its bar."""
    from video_features_b200.i3d_engine import I3DEngine
    sd, eng = s3d
    if engine == "i3d-rgb":
        sd = _i3d_sd("rgb")
        eng = I3DEngine(sd, "rgb", 0, max_stacks=1, max_T=16)
    sd64 = _f64(sd, cuda_device)
    for block in (0, 6, 8):
        xv, x = to_pairs(_control_input(block, cuda_device))
        cin = ib.WIDTHS[block][0]
        x[..., cin:] = 0
        y = eng.debug_mixed(block, x)
        ref = s3d_ref(sd64, block, xv) if engine == "s3d" else i3d_ref(sd64, block, xv)
        errs = branch_errors(y, ref, block)
        print(f"{engine} lo half dropped, block {block}: " + ", ".join(f"{e[0]:.1e} / {e[1]:.1e}" for e in errs))
        assert all(bars.beyond(e, ib.BARS[engine][block][j]) for j, e in enumerate(errs)), (block, errs)
    if engine == "i3d-rgb":
        eng.close()


def test_read_stage_fails_after_a_debug_block(s3d, cuda_device):
    """The debug entries run on the buffers read_stage reads: after one, read_stage fails until the next forward."""
    from video_features_b200._lib import VfError
    from video_features_b200.i3d_engine import I3DEngine
    sd, eng = s3d
    x = s3d_net.calibration_clips(seed=3, n=1, T=13).to(cuda_device)
    _, xb = to_pairs(_control_input(0, cuda_device))
    eng.forward_f32(x)
    before = eng.read_stage(2).clone()
    eng.debug_mixed(0, xb)
    with pytest.raises(VfError) as e:
        eng.read_stage(2)
    assert e.value.code == 1
    eng.forward_f32(x)
    assert torch.equal(eng.read_stage(2), before)
    ieng = I3DEngine(_i3d_sd("rgb"), "rgb", 0, max_stacks=1, max_T=12)
    xi = torch.rand(1, 3, 12, 224, 224, device=cuda_device) * 2 - 1
    ieng(xi)
    first = [ieng.read_stage(s).clone() for s in range(5)]
    ieng.debug_mixed(0, xb)
    for s in range(5):
        with pytest.raises(VfError) as e:
            ieng.read_stage(s)
        assert e.value.code == 1
    ieng(xi)
    assert all(torch.equal(ieng.read_stage(s), first[s]) for s in range(5))
    # more rows than the workspace holds: refused before any launch
    with pytest.raises(VfError, match="workspace"):
        ieng.debug_mixed(0, torch.zeros(2, 9, 30, 30, 384, dtype=torch.float16, device=cuda_device))
    with pytest.raises(VfError, match="workspace"):
        eng.debug_mixed(0, torch.zeros(10, 10, 30, 30, 384, dtype=torch.float16, device=cuda_device))
    ieng.close()


# ---- pools, bit for bit
def bordered(n, T, S, b=1):
    return (n, T + 2 * b, S + 2 * b, S + 2 * b, b, T + b, b, S + b, b, S + b)


def _pool_input(vol, C, seed, dev):
    """Pair rows of the volume vol: hi from a few fp16 values (exact ties, ties in hi), lo of either sign within half
    an fp16 ulp of hi or zero, about a third of the elements exactly zero; zero outside the valid region."""
    g = torch.Generator().manual_seed(seed)
    n, Tp, Hp, Wp, t0, t1, h0, h1, w0, w1 = vol
    shape = (n, C, t1 - t0, h1 - h0, w1 - w0)
    hi = torch.tensor([0.0, 0.5, 1.0, 1.25, 3.0, 7.5], dtype=torch.float64)[torch.randint(0, 6, shape, generator=g)]
    hi = torch.where(torch.rand(shape, generator=g) < 0.5, hi, torch.rand(shape, generator=g, dtype=torch.float64) * 8)
    hi = hi.half().double()
    ulp = torch.where(hi > 0, 2.0 ** (torch.floor(torch.log2(hi.clamp(min=1e-3))) - 10), torch.zeros_like(hi))
    lo = (torch.randint(-4, 5, shape, generator=g).double() / 8 * ulp * torch.rand(shape, generator=g,
                                                                                    dtype=torch.float64).gt(0.3))
    lo = lo.half().double()
    v = (hi + lo).float().double()            # the fp32 sum the kernel forms
    x = torch.zeros(n, Tp, Hp, Wp, 2 * C, dtype=torch.float16)
    x[:, t0:t1, h0:h1, w0:w1, :C] = hi.half().permute(0, 2, 3, 4, 1)
    x[:, t0:t1, h0:h1, w0:w1, C:] = lo.half().permute(0, 2, 3, 4, 1)
    return v.to(dev), x.to(dev)


def _expected(m, vol_out, C):
    """float64 pooled values (n, C, To, Ho, Wo) -> the pair volume of vol_out, split in fp32 as the kernels do."""
    n, Tp, Hp, Wp, t0, t1, h0, h1, w0, w1 = vol_out
    assert tuple(m.shape[2:]) == (t1 - t0, h1 - h0, w1 - w0), (tuple(m.shape), vol_out)
    f = m.float()
    hi = f.half()
    lo = (f - hi.float()).half()
    y = torch.zeros(n, Tp, Hp, Wp, 2 * C, dtype=torch.float16, device=m.device)
    y[:, t0:t1, h0:h1, w0:w1, :C] = hi.permute(0, 2, 3, 4, 1)
    y[:, t0:t1, h0:h1, w0:w1, C:] = lo.permute(0, 2, 3, 4, 1)
    return y


def _i3d_pool(k, s):
    return lambda v: i3d_net.maxpool(v, k, s)


def _torch_pool(k, s, p):
    return lambda v: F.max_pool3d(v, k, s, p)


# (name, C, vol_in, vol_out, k, s, p, float64 reference, expected kernel)
G, FA, S3 = 0, 1, 2
POOL_CASES = [
    # I3D: maxPool3d_2a / 3a (fixed windows inside the border), 4a at even / odd T1, 5a at even / odd T2
    ("i3d 2a", 64, (1, 6, 115, 115, 1, 4, 1, 113, 1, 113), bordered(1, 3, 56), (1, 3, 3), (1, 2, 2), (0, 0, 0),
     _i3d_pool((1, 3, 3), (1, 2, 2)), FA),
    ("i3d 3a", 192, bordered(2, 3, 56), bordered(2, 3, 28), (1, 3, 3), (1, 2, 2), (0, 0, 0),
     _i3d_pool((1, 3, 3), (1, 2, 2)), FA),
    ("i3d 4a T1=4", 480, bordered(1, 4, 28), bordered(1, 2, 14), (3, 3, 3), (2, 2, 2), (0, 0, 0),
     _i3d_pool((3, 3, 3), (2, 2, 2)), FA),
    ("i3d 4a T1=5", 480, bordered(1, 5, 28), bordered(1, 3, 14), (3, 3, 3), (2, 2, 2), (0, 0, 0),
     _i3d_pool((3, 3, 3), (2, 2, 2)), G),
    ("i3d 5a T2=2", 832, bordered(2, 2, 14), bordered(2, 1, 7), (2, 2, 2), (2, 2, 2), (0, 0, 0),
     _i3d_pool((2, 2, 2), (2, 2, 2)), FA),
    ("i3d 5a T2=3", 832, bordered(1, 3, 14), bordered(1, 2, 7), (2, 2, 2), (2, 2, 2), (0, 0, 0),
     _i3d_pool((2, 2, 2), (2, 2, 2)), FA),
    # the Mixed blocks' branch-3 pool (both trunks), 28 / 14 / 7
    ("mixed 3x3x3 C=192", 192, bordered(1, 1, 28), bordered(1, 1, 28), (3, 3, 3), (1, 1, 1), (1, 1, 1),
     _torch_pool(3, 1, 1), S3),
    ("mixed 3x3x3 C=480", 480, bordered(2, 3, 14), bordered(2, 3, 14), (3, 3, 3), (1, 1, 1), (1, 1, 1),
     _torch_pool(3, 1, 1), S3),
    ("mixed 3x3x3 C=832", 832, bordered(1, 2, 7), bordered(1, 2, 7), (3, 3, 3), (1, 1, 1), (1, 1, 1),
     _torch_pool(3, 1, 1), S3),
    # S3D: features.1 from the stem's volume, features.4, features.7 at even / odd T1, features.13 at even / odd T2
    ("s3d features.1", 64, (1, 6, 115, 115, 2, 5, 2, 114, 2, 114), bordered(1, 3, 56), (1, 3, 3), (1, 2, 2),
     (0, 1, 1), _torch_pool((1, 3, 3), (1, 2, 2), (0, 1, 1)), G),
    ("s3d features.4", 192, bordered(1, 2, 56), bordered(1, 2, 28), (1, 3, 3), (1, 2, 2), (0, 1, 1),
     _torch_pool((1, 3, 3), (1, 2, 2), (0, 1, 1)), G),
    ("s3d features.7 T1=4", 480, bordered(1, 4, 28), bordered(1, 2, 14), (3, 3, 3), (2, 2, 2), (1, 1, 1),
     _torch_pool(3, 2, 1), G),
    ("s3d features.7 T1=7", 480, bordered(1, 7, 28), bordered(1, 4, 14), (3, 3, 3), (2, 2, 2), (1, 1, 1),
     _torch_pool(3, 2, 1), G),
    ("s3d features.13 T2=4", 832, bordered(1, 4, 14), bordered(1, 2, 7), (2, 2, 2), (2, 2, 2), (0, 0, 0),
     _torch_pool(2, 2, 0), FA),
    ("s3d features.13 T2=5", 832, bordered(2, 5, 14), bordered(2, 2, 7), (2, 2, 2), (2, 2, 2), (0, 0, 0),
     _torch_pool(2, 2, 0), FA),
    # C = 8, the other side of each dispatch condition
    ("3x3x3/1 without a border", 8, (1, 3, 5, 6, 0, 3, 0, 5, 0, 6), (1, 3, 5, 6, 0, 3, 0, 5, 0, 6), (3, 3, 3),
     (1, 1, 1), (1, 1, 1), _torch_pool(3, 1, 1), G),
    ("3x3x3/1 onto another geometry", 8, bordered(1, 3, 6), bordered(1, 3, 6, 2), (3, 3, 3), (1, 1, 1), (1, 1, 1),
     _torch_pool(3, 1, 1), G),
    ("3x3x3/1 C=8 odd sides", 8, (2, 5, 9, 7, 1, 4, 1, 8, 1, 6), (2, 5, 9, 7, 1, 4, 1, 8, 1, 6), (3, 3, 3), (1, 1, 1),
     (1, 1, 1), _torch_pool(3, 1, 1), S3),
    ("2x2x2/2 C=8", 8, bordered(1, 4, 6), bordered(1, 2, 3), (2, 2, 2), (2, 2, 2), (0, 0, 0), _torch_pool(2, 2, 0), FA),
    ("window without a fast kernel", 8, bordered(1, 4, 9), bordered(1, 3, 4), (2, 3, 3), (1, 2, 2), (0, 0, 0),
     _torch_pool((2, 3, 3), (1, 2, 2), 0), G),
    ("1x3x3/1x2x2 past the border", 8, bordered(1, 2, 9), bordered(1, 2, 5), (1, 3, 3), (1, 2, 2), (0, 0, 0),
     _i3d_pool((1, 3, 3), (1, 2, 2)), G),
]


@pytest.mark.parametrize("case", POOL_CASES, ids=[c[0] for c in POOL_CASES])
def test_pool_bit_exact(cuda_device, case):
    from video_features_b200._lib import debug_maxpool3d
    name, C, vi, vo, k, s, p, ref_fn, want_path = case
    v, x = _pool_input(vi, C, sum(map(ord, name)), cuda_device)
    y, path = debug_maxpool3d(x, vi, vo, C, k, s, p)
    PATHS[name] = path
    want = _expected(ref_fn(v), vo, C)
    diff = int((y.view(torch.int16) != want.view(torch.int16)).sum())
    print(f"pool {name}: kernel {path}, {diff} differing halves of {y.numel()}")
    assert path == want_path, (name, path)
    assert diff == 0, (name, diff)


def test_pool_paths_cover_every_kernel():
    """Run after the pool cases: all three kernels ran, and each dispatch condition went both ways (the cases above
    name which side each one takes)."""
    if len(PATHS) < len(POOL_CASES):
        pytest.skip("the pool cases did not all run in this session")
    assert set(PATHS.values()) == {G, FA, S3}, PATHS


# ---- head
@pytest.mark.parametrize("T3,n,C", [(2, 1, 1024), (3, 5, 832), (8, 1, 832), (32, 5, 1024), (2, 5, 832)])
def test_head_matches_float64(cuda_device, T3, n, C):
    from video_features_b200._lib import debug_i3d_head
    vol = bordered(n, T3, 7)
    g = torch.Generator().manual_seed(T3 * 10 + n)
    v = torch.relu(torch.randn(n, C, T3, 7, 7, generator=g, dtype=torch.float64)).to(cuda_device)
    xv, x = to_pairs(v)
    y = debug_i3d_head(x, vol, C)
    ref = F.avg_pool3d(xv, (2, 7, 7), 1).mean(dim=(2, 3, 4))
    err = bars.row_errors(y, ref)
    HEAD[(T3, n, C)] = err
    print(f"head T3={T3} n={n} C={C}: rel-L2 {err[0]:.2e}, max-abs/max {err[1]:.2e}")
    assert bars.within(err, ib.HEAD_BAR), err


def test_zz_report_measured(cuda_device):
    """Prints the worst values per engine, block and branch over the session (pytest -s), and the pool kernels."""
    for (engine, block, j), (rel, mx) in sorted(MEASURED.items()):
        print(f"measured worst {engine} block {block} branch {j}: rel-L2 {rel:.2e}, max-abs/max {mx:.2e}")
    print("measured dict:", {k: (float(f"{v[0]:.3g}"), float(f"{v[1]:.3g}")) for k, v in sorted(MEASURED.items())})
    for name, path in PATHS.items():
        print(f"pool {name}: kernel {('general', 'fast', 'same3')[path]}")
    for (engine, kind), share in sorted(SHARES.items()):
        print(f"measured largest |defect_share| {engine} branches 1, 2, {kind} directions: {share:.3f}")
    if HEAD:
        print(f"measured worst head: rel-L2 {max(e[0] for e in HEAD.values()):.2e}, "
              f"max-abs/max {max(e[1] for e in HEAD.values()):.2e}")

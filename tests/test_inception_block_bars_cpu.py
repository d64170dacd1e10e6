"""The per-branch bars of the Mixed blocks (tests/inception_block_bars.py) tell the split-fp16 scheme from a lost lo half
inside one branch, and the oracle's block pieces compose to its whole trunk.

A float64 emulation of one block per spatial size (3b, 4f, 5c) of S3D and of I3D (rgb stand-in) on the real input of
the float64 trunk: the engine's split scheme carries every conv operand and every stored branch output to ~22 bits
(emulated as fp32 values; I3D keeps its declared single-fp16 operands).  Against the float64 block of the same input
the all-split block must stay tenfold under every branch's bar; one conv's weights or input, or one branch's stored
output, in single fp16 must exceed that branch's bar by the factor inception_block_bars.SEPARATION names.  I3D's
branches 1 and 2 are the exception: their bars hold the 1-ulp flips of the single-fp16 reducer outputs and do not
separate a lost lo half there, so those defects are told apart by split_engine_bars.defect_share, with the flips
modelled by computing the block's convolutions in fp32."""
import pytest
import torch
import torch.nn.functional as F

import inception_block_bars as ib
import split_engine_bars as bars
from oracle import i3d_net, s3d_net

BLOCKS = (0, 6, 8)          # 3b (28 x 28), 4f (14 x 14), 5c (7 x 7)


def _rnd(t, how):
    if how == "fp16":
        return t.half().double()
    return t.float().double() if how == "split" else t


def _cna(sd, p, x, how_x, how_w, pad=0):
    w = _rnd(sd[p + ".0.weight"], how_w)
    y = F.conv3d(_rnd(x, how_x), w, padding=pad)
    y = F.batch_norm(y, sd[p + ".1.running_mean"], sd[p + ".1.running_var"], sd[p + ".1.weight"], sd[p + ".1.bias"],
                     False, 0.0, s3d_net.EPS)
    return F.relu(y)


S3D_CONVS = ("b0", "b1a", "b1s", "b1t", "b2a", "b2s", "b2t", "b3")
S3D_BRANCH = {"b0": 0, "b1a": 1, "b1s": 1, "b1t": 1, "b2a": 2, "b2s": 2, "b2t": 2, "b3": 3}


def s3d_block(sd, i, x, defect=None):
    """SepInceptionBlock3D features[i] with every operand and branch store split (fp32), except defect: ("w" | "x",
    conv) rounds that conv's weights / input to fp16, ("store", branch) that branch's output."""
    p = f"features.{i}"

    def how(kind, conv):
        return "fp16" if defect == (kind, conv) else "split"

    def conv(name, key, x, pad=0):
        return _cna(sd, key, x, how("x", name), how("w", name), pad)

    def sep(pre, key, x):
        x = conv(pre + "s", key + ".0", x, (0, 1, 1))
        return conv(pre + "t", key + ".1", _rnd(x, "split"), (1, 0, 0))

    b = [conv("b0", p + ".branch0", x),
         sep("b1", p + ".branch1.1", _rnd(conv("b1a", p + ".branch1.0", x), "split")),
         sep("b2", p + ".branch2.1", _rnd(conv("b2a", p + ".branch2.0", x), "split")),
         conv("b3", p + ".branch3.1", F.max_pool3d(x, 3, 1, 1))]
    return torch.cat([_rnd(y, "fp16" if defect == ("store", j) else "split") for j, y in enumerate(b)], 1)


I3D_UNITS = ("branch_0", "branch_1.0", "branch_1.1", "branch_2.0", "branch_2.1", "branch_3.1")
I3D_BRANCH = {"branch_0": 0, "branch_1.0": 1, "branch_1.1": 1, "branch_2.0": 2, "branch_2.1": 2, "branch_3.1": 3}


def i3d_block(sd, m, x, defect=None, f32=False):
    """I3D Mixed block m with the engine's scheme: the declared single-fp16 operands rounded, every other operand and
    every branch store split (fp32); defect as for s3d_block (("w", unit) only for units whose weights are split).
    f32: the convolutions computed in fp32 (the accumulation-error proxy), so that the fp16 rounding of branch_1.0 /
    2.0's output flips elements near a rounding boundary as the engine's does; otherwise in float64."""
    names = i3d_net.unit_names()
    declared_w = {names[u] for u in i3d_net.DECLARED_FP16_UNITS}

    def unit(u, x, k):
        name = f"{m}.{u}"
        how_x = "fp16" if u in ("branch_1.1", "branch_2.1") or defect == ("x", u) else "split"
        how_w = "fp16" if name in declared_w or defect == ("w", u) else "split"
        w, xr = _rnd(sd[f"{name}.conv3d.weight"], how_w), _rnd(x, how_x)
        if f32:
            y = F.conv3d(xr.float(), w.float(), padding=k // 2).double()
        else:
            y = F.conv3d(xr, w, padding=k // 2)
        y = F.batch_norm(y, sd[f"{name}.batch3d.running_mean"], sd[f"{name}.batch3d.running_var"],
                         sd[f"{name}.batch3d.weight"], sd[f"{name}.batch3d.bias"], False, 0.0, i3d_net.BN_EPS)
        return F.relu(y)

    b = [unit("branch_0", x, 1), unit("branch_1.1", unit("branch_1.0", x, 1), 3),
         unit("branch_2.1", unit("branch_2.0", x, 1), 3), unit("branch_3.1", F.max_pool3d(x, 3, 1, 1), 1)]
    return torch.cat([_rnd(y, "fp16" if defect == ("store", j) else "split") for j, y in enumerate(b)], 1)


def i3d_directions(m, j):
    """The defects of I3D branch j (1 or 2) that its bars do not separate: the fp16 weights of each of its split units,
    the fp16 (lo half lost) pair input of its 1x1x1 reducer, its store."""
    names = i3d_net.unit_names()
    declared = {names[u] for u in i3d_net.DECLARED_FP16_UNITS}
    return ([("w", f"branch_{j}.{k}") for k in (0, 1) if f"{m}.branch_{j}.{k}" not in declared]
            + [("x", f"branch_{j}.0"), ("store", j)])


def _branch_errors(y, ref, block):
    out, a = [], 0
    for w in ib.WIDTHS[block][1:]:
        out.append(bars.row_errors(y[:, a:a + w], ref[:, a:a + w]))
        a += w
    return out


def _canonical(v):
    hi = v.half()
    return hi.double() + (v - hi.double()).half().double()


@pytest.fixture(scope="module")
def s3d_inputs():
    torch.set_grad_enabled(False)
    sd = {k: v.double() for k, v in s3d_net.stand_in_state_dict().items()}
    x = s3d_net.calibration_clips(seed=7, n=1, T=13).double()
    return sd, [_canonical(v) for v in s3d_net.mixed_inputs(sd, x)]


@pytest.fixture(scope="module")
def i3d_inputs():
    from oracle.stand_in import state_dict
    torch.set_grad_enabled(False)
    sd = {k: v.double() for k, v in state_dict("i3d_rgb.pt").items()}
    x = torch.rand(1, 3, 10, 224, 224, generator=torch.Generator().manual_seed(5), dtype=torch.float64) * 2 - 1
    return sd, [_canonical(v) for v in i3d_net.mixed_inputs(sd, x, declared_rounding=True)]


def _report(engine, block, what, errs):
    bar = ib.BARS[engine][block]
    print(f"{engine} block {block} {what:<12s} " + "  ".join(
        f"b{j} {e[0]:.1e} ({e[0] / bar[j][0]:5.1f}x) / {e[1]:.1e} ({e[1] / bar[j][1]:5.1f}x)" for j, e in enumerate(errs)))


def _factor(err, bar):
    """How far err lies above bar: the larger of its rel-L2 and max-abs ratios (bars.beyond)."""
    return max(err[0] / bar[0], err[1] / bar[1])


@pytest.mark.parametrize("block", BLOCKS)
def test_s3d_block_bars_separate_a_lost_lo_half(s3d_inputs, block):
    sd, ins = s3d_inputs
    key = tuple(s3d_net.MIXED)[block]
    x = ins[block]
    ref = s3d_net.mixed_block(sd, key, x)
    bar = ib.BARS["s3d"][block]
    failures = []
    errs = _branch_errors(s3d_block(sd, key, x), ref, block)
    _report("s3d", block, "all split", errs)
    failures += [("all split", j, e) for j, e in enumerate(errs) if not bars.within(e, bar[j], 0.1)]
    least = []
    for d in [(k, c) for k in ("w", "x") for c in S3D_CONVS] + [("store", j) for j in range(4)]:
        j = S3D_BRANCH[d[1]] if d[0] != "store" else d[1]
        e = _branch_errors(s3d_block(sd, key, x, d), ref, block)
        _report("s3d", block, f"{d[0]} {d[1]}", e)
        least.append((_factor(e[j], bar[j]), d))
    print(f"s3d block {block}: least separation {min(least)}")
    f = ib.SEPARATION["s3d"][block]
    failures += [(d, f"{g:.1f}x, not {f}x over the bar") for g, d in least if g < f]
    assert not failures, failures


@pytest.mark.parametrize("block", BLOCKS)
def test_i3d_block_bars_separate_a_lost_lo_half(i3d_inputs, block):
    """Branches 0 and 3 by the bars.  Branches 1 and 2, whose bars hold the declared-fp16 flips, by defect_share along
    each defect's direction (its float64 reference minus the intact one): with the flips modelled (fp32 convolutions),
    the all-split block carries at most SHARE[0] of it, and the block with that defect at least SHARE[1]."""
    sd, ins = i3d_inputs
    m = tuple(i3d_net.MIXED)[block]
    x = ins[block]
    ref = i3d_net.mixed_block(sd, m, x, declared_rounding=True)
    bar = ib.BARS["i3d-rgb"][block]
    failures = []
    errs = _branch_errors(i3d_block(sd, m, x), ref, block)
    _report("i3d-rgb", block, "all split", errs)
    failures += [("all split", j, e) for j, e in enumerate(errs) if j in (0, 3) and not bars.within(e, bar[j], 0.1)]
    least = []
    for d in [(k, u) for k in ("w", "x") for u in ("branch_0", "branch_3.1")] + [("store", 0), ("store", 3)]:
        j = I3D_BRANCH[d[1]] if d[0] != "store" else d[1]
        e = _branch_errors(i3d_block(sd, m, x, d), ref, block)
        _report("i3d-rgb", block, f"{d[0]} {d[1]}", e)
        least.append((_factor(e[j], bar[j]), d))
    print(f"i3d-rgb block {block}: least separation (branches 0, 3) {min(least)}")
    f = ib.SEPARATION["i3d"][block]
    failures += [(d, f"{g:.1f}x, not {f}x over the bar") for g, d in least if g < f]
    split32 = i3d_block(sd, m, x, f32=True)
    _report("i3d-rgb", block, "fp32 convs", _branch_errors(split32, ref, block))
    edges = [0]
    for w in ib.WIDTHS[block][1:]:
        edges.append(edges[-1] + w)
    for j in (1, 2):
        a, b = edges[j], edges[j + 1]
        for d in i3d_directions(m, j):
            if d[0] == "store":
                ref_d = ref[:, a:b].half().double()
            else:
                kw = {"fp16_weights" if d[0] == "w" else "fp16_inputs": (f"{m}.{d[1]}",)}
                ref_d = i3d_net.mixed_block(sd, m, x, declared_rounding=True, **kw)[:, a:b]
            ok = bars.defect_share(split32[:, a:b], ref[:, a:b], ref_d)
            bad = bars.defect_share(i3d_block(sd, m, x, d, f32=True)[:, a:b], ref[:, a:b], ref_d)
            print(f"i3d-rgb block {block} branch {j} {d[0]} {d[1]}: defect_share all split {ok:+.3f}, "
                  f"with the defect {bad:+.3f}")
            if abs(ok) > ib.SHARE[0] or bad < ib.SHARE[1]:
                failures.append((j, d, ok, bad))
    assert not failures, failures


def test_s3d_blocks_and_pools_compose_to_the_trunk(s3d_inputs):
    """mixed_inputs + mixed_block + the trunk's pools give forward's taps exactly (112 x 112, two clips)."""
    sd = s3d_inputs[0]
    x = s3d_net.calibration_clips(seed=2, n=2, T=13).double()[..., :112, :112]
    _, taps = s3d_net.features(sd, x, taps=True)
    ins = s3d_net.mixed_inputs(sd, x)
    keys = tuple(s3d_net.MIXED)
    outs = [s3d_net.mixed_block(sd, k, v) for k, v in zip(keys, ins)]
    assert torch.equal(outs[1], taps["mixed_3c"]) and torch.equal(outs[6], taps["mixed_4f"])
    assert torch.equal(outs[8], taps["mixed_5c"])
    assert torch.equal(F.max_pool3d(outs[1], 3, 2, 1), ins[2]) and torch.equal(F.max_pool3d(outs[6], 2, 2, 0), ins[7])
    for b in (0, 2, 3, 4, 5, 7):
        assert torch.equal(outs[b], ins[b + 1]), b


@pytest.mark.parametrize("declared", [False, True])
def test_i3d_blocks_and_pools_compose_to_the_trunk(i3d_inputs, declared):
    """mixed_inputs + mixed_block + maxpool give forward_features' stages exactly, with and without the declared
    rounding."""
    sd = i3d_inputs[0]
    x = torch.rand(1, 3, 10, 224, 224, generator=torch.Generator().manual_seed(9), dtype=torch.float64) * 2 - 1
    _, st = i3d_net.forward_features(sd, x, return_stages=True, declared_rounding=declared)
    ins = i3d_net.mixed_inputs(sd, x, declared_rounding=declared)
    outs = [i3d_net.mixed_block(sd, m, v, declared_rounding=declared) for m, v in zip(i3d_net.MIXED, ins)]
    assert torch.equal(outs[1], st["3c"]) and torch.equal(outs[6], st["4f"]) and torch.equal(outs[8], st["5c"])
    assert torch.equal(i3d_net.maxpool(outs[1], (3, 3, 3), (2, 2, 2)), ins[2])
    assert torch.equal(i3d_net.maxpool(outs[6], (2, 2, 2), (2, 2, 2)), ins[7])
    for b in (0, 2, 3, 4, 5, 7):
        assert torch.equal(outs[b], ins[b + 1]), b

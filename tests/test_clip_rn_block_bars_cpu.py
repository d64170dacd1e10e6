"""The premise of tests/clip_rn_block_bars.py, in a CPU float64 emulation: a lo half lost anywhere inside one CLIP ResNet
Bottleneck lies far above the block bars the GPU test holds the engine to.

Four blocks per tower, on the float64 trunk's real input to them (one calibration frame): layer1.0 (the stem's
AvgPool2d fused into its convs), layer2.0 (stride 2: the pool fused into conv3 and the downsample), and one identity
block each of layer3 and layer4 (x.1).  The emulated block models every split pair exactly as the engine forms it,
hi = fp16(v), lo = fp16(v - hi) with subnormal lo halves included, for the weights and for every stored activation
(conv1's and conv2's outputs, the branch, the shortcut, the block output); the convolutions themselves are exact.  One
defect at a time leaves one operand in single fp16: the weights of conv1, conv2, conv3 or the downsample; the input of
each of them; the branch store; the block output store.  Each defect is compared, against the float64 block with the
original weights, on the part the GPU test checks it by (convs 1 .. 3 and the branch store: the branch; the
downsample: the shortcut; the output store: the output), and must exceed that part's bar by SEPARATION.

The intact emulation's own distance from float64 is the cost of the pair representation alone (mostly the weights'
subnormal lo halves); it is asserted to stay under a third of every bar (PAIR_SHARE)."""
import functools

import pytest
import torch

import clip_rn_block_bars as rb
import split_engine_bars as bars
from oracle import clip_resnet

def chosen_blocks(cfg):
    """layer1.0, layer2.0, layer3.1, layer4.1."""
    L = cfg["layers"]
    return (0, L[0], L[0] + L[1] + 1, L[0] + L[1] + L[2] + 1)


@functools.lru_cache(maxsize=None)
def _inputs(name):
    sd = {k: v.double() for k, v in clip_resnet.stand_in_state_dict(name).items()}
    cfg = clip_resnet.config(sd)
    x = clip_resnet.calibration_images(cfg["n_px"], seed=7, n=1).double()
    with torch.no_grad():
        ins = clip_resnet.block_inputs(sd, x, cfg)
    return sd, cfg, {i: rb.pair(ins[i]) for i in chosen_blocks(cfg)}


def separations(name):
    """{(block, defect): (factor over the bar, error)} and {(block, part): the intact emulation's error / its bar}."""
    sd, cfg, ins = _inputs(name)
    sep, share = {}, {}
    with torch.no_grad():
        for i, x in ins.items():
            ref = dict(zip(rb.PARTS, clip_resnet.block(sd, cfg, i, x)))
            bar = rb.BLOCK[name][clip_resnet.blocks(cfg)[i][2]]
            clean = rb.emulated_block(sd, cfg, i, x)
            for part in rb.PARTS:
                e = bars.row_errors(clean[part], ref[part])
                share[(i, part)] = max(e[0] / bar[part][0], e[1] / bar[part][1])
            for d in rb.DEFECTS:
                if d[1] == "downsample.0" and not rb.has_downsample(sd, cfg, i):
                    continue
                part = rb.PART[d[1]]
                e = bars.row_errors(rb.emulated_block(sd, cfg, i, x, d)[part], ref[part])
                sep[(i, d)] = (max(e[0] / bar[part][0], e[1] / bar[part][1]), e)
    return sep, share


@pytest.mark.parametrize("name", list(clip_resnet.TOWERS))
def test_every_single_fp16_defect_exceeds_its_bar(name):
    sep, share = separations(name)
    for (i, d), (f, e) in sorted(sep.items()):
        print(f"{name} block {i} {d[0]} {d[1]}: {f:.1f}x its {rb.PART[d[1]]} bar (rel-L2 {e[0]:.2e}, max-abs {e[1]:.2e})")
    for (i, part), s in sorted(share.items()):
        print(f"{name} block {i} {part}: the exact-pair emulation sits at {s:.3f} of the bar")
    _, cfg, _ = _inputs(name)
    low = {k: v[0] for k, v in sep.items() if v[0] < rb.SEPARATION[name][clip_resnet.blocks(cfg)[k[0]][2]]}
    assert not low, low
    assert max(share.values()) <= rb.PAIR_SHARE, share


def test_lo_halves_of_the_weights_are_mostly_subnormal():
    """The premise of the exact pair model: |w| < 0.125 puts lo = fp16(w - hi) among fp16's subnormals."""
    sd = clip_resnet.stand_in_state_dict("RN50")
    w = sd["visual.layer4.0.conv2.weight"].float()
    hi = w.half()
    lo = (w - hi.float()).half()
    sub = ((lo != 0) & (lo.abs() < 2.0 ** -14)).double().mean().item()
    rel = ((hi.double() + lo.double() - w.double()).norm() / w.double().norm()).item()
    print(f"layer4.0.conv2: {sub:.1%} of the lo halves subnormal, pair vs fp32 weight rel-L2 {rel:.1e}")
    assert sub > 0.9 and 1e-7 < rel < 1e-5
